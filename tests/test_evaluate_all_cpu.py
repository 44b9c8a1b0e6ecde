"""CPU: the host side of bp_evaluate_* — bp_evaluate_chunk_params against the formula include/bp_b200.h documents, and
the request Model.evaluate packs (no GPU: the request is built and read back, nothing is launched)."""
import ctypes as C
import itertools

import numpy as np
import pytest

from basic_pitch_b200 import _lib
from basic_pitch_b200.inference import Model


class _NoDevice(Model):
    """A Model without a device: just enough for the request packing."""

    def __init__(self):
        self._lib = _lib.load()


NOTE_FAMS = ("notes", "onset_offset", "pairs", "frames", "bent_frames", "note_melody", "flat_note_melody")


def _grid_bytes(F, n):
    C_ = 88 * F
    cand = C_ // 32 + 2
    blk = F // 256 + n + 1
    return 4 * C_ + 4 * cand + 8 * 88 * blk + 12 * min(C_, 8 * F + 64 * n) + 16 * n + 64


def _expected(F, n, fams, R, K, V):
    S = min(88 * F, 8 * F + 64 * n)
    per = _grid_bytes(F, n)
    extra = dict(notes=8 * R + 16 * S, onset_offset=24 * R + 16 * S + 8 * n, pairs=8 * R + 28 * S, frames=16 * V + 8 * K,
                 bent_frames=16 * V + 8 * K + 4)
    per += sum(extra[f] for f in fams if f in extra)
    if {"note_melody", "flat_note_melody"} & set(fams):
        per += 16 * F
    return max(1, min(65535, (2 << 30) // per))


def _refs(n, notes_per_file, frames_per_file, values_per_frame):
    nrefs = [(np.tile([[0.1, 0.5]], (notes_per_file, 1)), np.full(notes_per_file, 220.0))] * n
    t = np.arange(frames_per_file) * 0.01
    mp = [(t, [np.full(values_per_frame, 220.0)] * frames_per_file)] * n
    mel = [(t, np.full(frames_per_file, 220.0))] * n
    return nrefs, mp, mel


def test_chunk_params_follow_the_documented_formula():
    m = _NoDevice()
    lib = m._lib
    for F, n in ((0, 1), (100, 1), (3_000, 2), (200_000, 40), (2_000_000, 1250), (40_000_000, 3)):
        assert lib.bp_evaluate_chunk_params(F, n, None) == lib.bp_decode_grid_chunk_params(F, n)
        nrefs, mp, mel = _refs(n, 7, 11, 3)
        R, K, V = 7 * n, 11 * n, 33 * n
        for k in (1, 2, 7):
            for fams in itertools.combinations(NOTE_FAMS, k):
                got = m.evaluate_chunk_params(F, fams, [dict()], note_refs=nrefs, multipitch_refs=mp, f0_refs=mel)
                assert got == _expected(F, n, fams, R, K, V), (F, n, fams)
    # the posteriorgram families run their own chunks: they leave the decode chunk as it is
    nrefs, mp, mel = _refs(2, 7, 11, 3)
    sal = dict(settings=[dict(threshold=0.3)], references=mp)
    assert m.evaluate_chunk_params(5000, ["salience"], salience=sal, f0_refs=mel) == lib.bp_decode_grid_chunk_params(5000, 2)


def test_request_packing():
    from basic_pitch_b200 import evaluate

    m = _NoDevice()
    nrefs, mp, mel = _refs(2, 3, 5, 2)
    sal = dict(settings=[dict(threshold=0.3), dict(threshold=0.4, peak_picking=False)], kind="note", references=mp)
    mel_spec = dict(settings=[dict(threshold=0.5)], references=mel)
    req, keep, out = m._eval_request(2, Model.EVAL_FAMILIES, [dict(), dict(min_note_len=3)], note_refs=nrefs,
                                     multipitch_refs=mp, f0_refs=mel, salience=sal, melody=mel_spec, window=0.25,
                                     cent_tolerance=30.0, onset_tolerance=0.07)
    assert req.n_params == 2 and req.n_salience == 2 and req.n_melody == 1
    assert req.salience_gram == 1 and req.melody_gram == 0
    assert req.window == 0.25 and req.salience_window == 0.25 and req.cent_tolerance == 30.0 and req.melody_tolerance == 30.0
    params = C.cast(req.params, C.POINTER(_lib.DecodeParams))
    assert params[1].min_note_len == 3 and params[0].include_pitch_bends == 1
    score = C.cast(req.score, C.POINTER(_lib.ScoreParams))[0]
    assert score.onset_tolerance == 0.07 and score.pitch_tolerance == 50.0
    assert req.est_log2_hz == evaluate.EST_LOG2_HZ.ctypes.data
    assert req.est_midi == evaluate.EST_MIDI.ctypes.data and req.bin_midi and req.bin_cent and req.melody_cent
    sp = C.cast(req.salience_params, C.POINTER(_lib.SalienceParams))
    assert sp[1].peak_pick == 0 and sp[1].threshold == 0.4 and sp[0].bin_hi == 88
    for name, shape in (("notes", (2, 2, 4)), ("onset_offset", (2, 2, 4)), ("frames", (2, 2, 7)), ("bent_frames", (2, 2, 7)),
                        ("note_melody", (2, 2, 7)), ("flat_note_melody", (2, 2, 7)), ("salience", (2, 2, 7)),
                        ("melody", (1, 2, 7))):
        assert out[name].shape == shape, name
    assert req.notes_counts == out["notes"].ctypes.data
    assert req.pair_match == out["pairs"][0].ctypes.data and not req.pair_notes
    # only what is asked for is set
    req, keep, out = m._eval_request(2, ["frames"], [dict()], multipitch_refs=mp)
    assert set(out) == {"frames"} and not req.notes_counts and not req.note_refs and not req.salience_counts
    with pytest.raises(ValueError, match="unknown famil"):
        m._eval_request(2, ["frame"], [dict()])
    with pytest.raises(ValueError, match="f0 references are required"):
        m._eval_request(2, ["note_melody"], [dict()])
    with pytest.raises(ValueError, match="2 files but 1 note references"):
        m._eval_request(2, ["notes"], [dict()], note_refs=nrefs[:1])
