"""CPU: the host side of the grid decode — the settings -> decode parameter conversion of model_output_to_notes_grid /
predict_grid against the arithmetic of model_output_to_notes (_decode) and predict, and the chunking of
bp_decode_grid_chunk_params against the workspace budget documented in include/bp_b200.h."""
import numpy as np
import pytest

from basic_pitch_b200 import note_creation as nc
from basic_pitch_b200.constants import AUDIO_SAMPLE_RATE, FFT_HOP

HZ = [None, 1.0, 27.5, 30.0, 100.0, 440.0, 1000.0, 4186.0, 4500.0, 20000.0]
BUDGET = 2 << 30  # bytes per chunk, include/bp_b200.h (bp_decode_grid_chunk_params)


def test_predict_names_convert_like_predict():
    for ms in (0.0, 11.6, 50.0, 127.7, 128.0, 1000.0):
        for lo_hz in HZ:
            for hi_hz in HZ:
                s = dict(onset_threshold=0.4, frame_threshold=0.2, minimum_note_length=ms, minimum_frequency=lo_hz,
                         maximum_frequency=hi_hz, multiple_pitch_bends=True, melodia_trick=False, midi_tempo=90)
                d, midi = nc.grid_setting(s, predict_names=True)
                # predict: inference.py (min_note_len, frequency_to_column_range) and transcribe_arrays' defaults
                lo, hi = nc.frequency_to_column_range(lo_hz, hi_hz)
                assert d == dict(onset_thresh=0.4, frame_thresh=0.2,
                                 min_note_len=int(np.round(ms / 1000 * (AUDIO_SAMPLE_RATE / FFT_HOP))), energy_tol=11,
                                 infer_onsets=True, melodia_trick=False, include_pitch_bends=True, min_pitch_idx=lo,
                                 max_pitch_idx=hi), s
                assert midi == dict(multiple_pitch_bends=True, midi_tempo=90)
    d, midi = nc.grid_setting({}, predict_names=True)
    assert (d["onset_thresh"], d["frame_thresh"], d["min_note_len"], d["min_pitch_idx"], d["max_pitch_idx"]) == (0.5, 0.3, 11, 0, 88)
    assert d["melodia_trick"] and midi == dict(multiple_pitch_bends=False, midi_tempo=120)


def test_notes_names_convert_like_decode():
    for lo_hz in HZ:
        for hi_hz in HZ:
            s = dict(onset_thresh=0.6, frame_thresh=0.1, min_note_len=7, min_freq=lo_hz, max_freq=hi_hz,
                     infer_onsets=False, include_pitch_bends=False)
            d, midi = nc.grid_setting(s)
            lo, hi = nc.frequency_to_column_range(lo_hz, hi_hz, 88)  # what _decode passes to decode_arrays
            assert d == dict(onset_thresh=0.6, frame_thresh=0.1, min_note_len=7, energy_tol=nc.ENERGY_TOLERANCE,
                             infer_onsets=False, melodia_trick=True, include_pitch_bends=False, min_pitch_idx=lo,
                             max_pitch_idx=hi), s
            assert midi == dict(multiple_pitch_bends=False, midi_tempo=120)
    # out-of-range limits follow NumPy's slice rules, as the reference's constrain_frequency does
    assert nc.grid_setting(dict(onset_thresh=0.5, frame_thresh=0.3, min_freq=20000.0))[0]["min_pitch_idx"] == 88
    # 1 Hz is column -57: m[:, -57:] = 0 zeroes from column 88 - 57 on
    assert nc.grid_setting(dict(onset_thresh=0.5, frame_thresh=0.3, max_freq=1.0))[0]["max_pitch_idx"] == 31


def test_unknown_or_missing_names_raise():
    with pytest.raises(TypeError):
        nc.grid_setting(dict(onset_threshold=0.5), predict_names=False)
    with pytest.raises(TypeError):
        nc.grid_setting(dict(onset_thresh=0.5), predict_names=True)
    with pytest.raises(TypeError):
        nc.grid_setting(dict(onset_thresh=0.5))  # frame_thresh is required, as in model_output_to_notes


def _workspace(total_frames, n_files):
    """Bytes per setting of a chunk, the formula of include/bp_b200.h."""
    f, c = total_frames, 88 * total_frames
    return 4 * c + 4 * (c // 32 + 2) + 8 * 88 * (f // 256 + n_files + 1) + 12 * min(c, 8 * f + 64 * n_files) + 16 * n_files + 64


def test_chunk_params_bounded_by_the_budget():
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    for n_files in (1, 3, 64, 1250, 20000):
        prev = None
        for total in (0, 1, 100, 15_503, 100_000, 1_076_250, 10**7, 10**9):
            if total < n_files and total:
                continue
            c = int(lib.bp_decode_grid_chunk_params(total, n_files))
            assert c >= 1, (total, n_files)
            assert c == 1 or c * _workspace(total, n_files) <= BUDGET, (total, n_files, c)
            assert c == 65535 or (c + 1) * _workspace(total, n_files) > BUDGET, (total, n_files, c)
            if prev is not None:
                assert c <= prev, (total, n_files, c, prev)
            prev = c
    # the shapes of tools/decode_grid_profile.py: one 180 s clip takes 256 settings in one chunk; the bench workload
    # (1 250 x 10 s) needs several chunks for 16
    assert lib.bp_decode_grid_chunk_params(15_503, 1) >= 256
    assert lib.bp_decode_grid_chunk_params(1250 * 861, 1250) < 16
