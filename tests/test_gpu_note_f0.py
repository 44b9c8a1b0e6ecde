"""GPU: decoded notes with their pitch bends scored as multi-f0 and single-f0 estimates on the device
(bp_score_bent_frames_grid_*, bp_score_note_melody_grid_*: csrc/score_frames.cu, csrc/score_melody.cu, csrc/api.cu) and
their Python entry points (Model.score_frames_grid(contours=...), Model.score_note_melody_grid,
inference.evaluate_frames_grid(pitch_bends=True), inference.evaluate_note_melody_grid).

Every count must equal oracle/multipitch_ref.py / oracle/melody_ref.py applied to evaluate.note_frames_to_multipitch /
evaluate.note_frames_to_melody of the notes and bends Model.decode_grid (bp_decode_grid_host) returns for the same
inputs and setting."""
import ctypes as C

import numpy as np
import pytest

from oracle import melody_ref as melr
from tests import postsets
from tests.test_gpu_decode_edges import _kw, _set
from tests.test_gpu_decode_grid import _model_grid
from tests.test_gpu_frame_score import _oracle, _times, _vals
from tests.test_gpu_melody import HOP_58, _notes_f0
from tests.test_gpu_score import _hz

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def edges(golden_dir):
    return dict(np.load(golden_dir / "decode_edges.npz"))


def _bends(r):
    bo, b = r["bend_off"], r["bends"]
    return [b[bo[j] : bo[j + 1]] for j in range(len(r["start"]))]


def _mp_oracle(res, lens, refs, window=0.5):
    from basic_pitch_b200.evaluate import multipitch_values, note_frames_to_multipitch

    rv = [_vals(r) for r in refs]
    out = np.zeros((len(res), len(lens), 7), np.int64)
    for k, per in enumerate(res):
        for i, r in enumerate(per):
            et, ef = note_frames_to_multipitch(r["start"], r["end"], r["pitch"], _bends(r), lens[i])
            out[k, i] = _oracle(rv[i][0], rv[i][1], et, [multipitch_values(f) for f in ef], window)
    return out


def _mel_oracle(res, notes, refs, tol=50.0):
    from basic_pitch_b200.evaluate import note_frames_to_melody

    out = np.zeros((len(res), len(notes), 7), np.int64)
    for k, per in enumerate(res):
        for i, r in enumerate(per):
            et, f0 = note_frames_to_melody(r["start"], r["end"], r["pitch"], _bends(r), notes[i])
            out[k, i] = melr.counts(refs[i][0], refs[i][1], et, f0, tol)
    return out


def _base_times(name, T, rng):
    """Reference times of a file of T model frames: the model frames themselves, vocadito's 256 / 44100 s hop, or a
    jittered 10 ms grid."""
    dur = max(T * 256 / 22050, 0.5)
    if name == "identity":
        return _times(T)
    if name == "hop58":
        return np.arange(1, int(dur / HOP_58)) * HOP_58
    t = np.arange(0, dur, 0.01)
    return np.maximum(np.sort(np.round(t + rng.uniform(-0.004, 0.004, len(t)), 5)), 0.0)


def _check_grid(model, notes, onsets, contours, settings, mp_refs, mel_refs, res=None):
    """Both grids against the oracle on the host definitions of bp_decode_grid_host's notes and bends."""
    if res is None:
        res = model.decode_grid(notes, onsets, contours, settings)
    lens = [a.shape[0] for a in notes]
    exp_mp = _mp_oracle(res, lens, mp_refs)
    np.testing.assert_array_equal(model.score_frames_grid(notes, onsets, settings, mp_refs, contours=contours), exp_mp)
    exp_mel = _mel_oracle(res, notes, mel_refs)
    np.testing.assert_array_equal(model.score_note_melody_grid(notes, onsets, contours, settings, mel_refs), exp_mel)
    return res, exp_mp, exp_mel


# ------------------------------------------------------------------------------------------------ model output
@pytest.fixture(scope="module")
def model_case(model, golden_dir):
    """The vocadito clip, two synth melody lines, random notes, dense chords and an empty clip, with their note
    annotations (multi-pitch references) and f0 functions (melody references)."""
    from basic_pitch_b200 import synth

    z = np.load(golden_dir / "vocadito10.npz")
    voc = (np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"]))
    rnd = synth.random_notes_events(5.0, 930, 5.0)
    chords = synth.dense_chords_events(3.0)

    def from_f0(f):
        return lambda t: [np.array([x]) if x > 0 else np.zeros(0) for x in f(t)]

    def from_notes(n):
        from basic_pitch_b200.evaluate import notes_to_multipitch

        return lambda t: notes_to_multipitch(n[0], n[1], t)

    items = [(z["audio22k"].astype(np.float32), from_notes(voc), lambda t: _notes_f0(voc, t))]
    for sec, seed in ((6.0, 41), (8.0, 42)):
        f = lambda t, sec=sec, seed=seed: synth.melody_f0(sec, seed, t)  # noqa: E731
        items.append((synth.melody_clip(sec, seed), from_f0(f), f))
    items.append((synth.random_notes_clip(5.0, 930, 5.0), from_notes(rnd), lambda t: _notes_f0(rnd, t)))
    items.append((synth.dense_chords_clip(3.0, seed=931), from_notes(chords), lambda t: _notes_f0(chords, t)))
    items.append((np.zeros(0, np.float32), lambda t: [np.array([220.0])] * len(t), lambda t: np.full(len(t), 220.0)))
    outs = model.run_inference_arrays([c for c, _, _ in items])
    return items, outs


def test_grid_counts_equal_the_oracle_on_model_output(model, model_case):
    """48 settings (bends on and off, thresholds, ranges, min_note_len, infer / melodia) on three reference time bases."""
    items, outs = model_case
    notes, onsets, contours = ([o[k] for o in outs] for k in ("note", "onset", "contour"))
    settings = _model_grid()
    assert len(settings) >= 48 and {s["include_pitch_bends"] for s in settings} == {True, False}
    res = model.decode_grid(notes, onsets, contours, settings)
    rng = np.random.default_rng(31)
    for base in ("identity", "hop58", "jitter"):
        ts = [_base_times(base, a.shape[0], rng) for a in notes]
        mp_refs = [(t, mp(t)) for t, (_, mp, _) in zip(ts, items)]
        mel_refs = [(t, f0(t)) for t, (_, _, f0) in zip(ts, items)]
        _, exp_mp, exp_mel = _check_grid(model, notes, onsets, contours, settings, mp_refs, mel_refs, res)
        assert exp_mp[..., 2].sum() > 1000 and exp_mel[..., 4].sum() > 1000, base
        assert (exp_mel[:, 5, 2] == 0).all()  # the empty clip is unvoiced throughout
    # the bends matter: the same settings without bends score differently somewhere
    flat = [{**s, "include_pitch_bends": False} for s in settings]
    assert not np.array_equal(model.score_note_melody_grid(notes, onsets, contours, flat, mel_refs),
                              model.score_note_melody_grid(notes, onsets, contours, settings, mel_refs))


def test_device_on_a_caller_stream_equals_host(model, model_case):
    import torch

    from basic_pitch_b200.evaluate import bent_bins

    items, outs = model_case
    notes, onsets, contours = ([o[k] for o in outs] for k in ("note", "onset", "contour"))
    settings = _model_grid()[::5]
    ts = [_base_times("hop58", a.shape[0], None) for a in notes]
    mp_refs = [(t, mp(t)) for t, (_, mp, _) in zip(ts, items)]
    mel_refs = [(t, f0(t)) for t, (_, _, f0) in zip(ts, items)]
    dev = f"cuda:{model.device}"
    d = [torch.from_numpy(np.ascontiguousarray(np.concatenate(x), np.float32)).to(dev) for x in (notes, onsets, contours)]
    foff = np.cumsum([0] + [a.shape[0] for a in notes]).astype(np.int64)
    ps = model._grid_params(settings)
    _, midi, chroma, cents = bent_bins()
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    mp_set, keep_mp = model._multipitch_set(mp_refs, "references")
    mel_set, keep_mel = model._melody_set(mel_refs, "references")
    got_mp = np.full((len(settings), len(notes), 7), -1, np.int64)
    got_mel = np.full((len(settings), len(notes), 7), -1, np.int64)
    with torch.cuda.stream(stream):
        model._lib.bp_score_bent_frames_grid_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                                    foff.ctypes.data, len(notes), ps, len(settings), C.byref(mp_set),
                                                    0.5, midi.ctypes.data, chroma.ctypes.data, got_mp.ctypes.data,
                                                    stream.cuda_stream)
        model._lib.bp_score_note_melody_grid_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(),
                                                    foff.ctypes.data, len(notes), ps, len(settings), C.byref(mel_set),
                                                    50.0, cents.ctypes.data, got_mel.ctypes.data, stream.cuda_stream)
    assert got_mp.tobytes() == model.score_frames_grid(notes, onsets, settings, mp_refs, contours=contours).tobytes()
    assert got_mel.tobytes() == model.score_note_melody_grid(notes, onsets, contours, settings, mel_refs).tobytes()


# ------------------------------------------------------------------------------------------------ adversarial decodes
@pytest.mark.parametrize("name", postsets.NAMES)
def test_adversarial_sets(model, edges, name):
    """The pinned sets of tests/postsets.py under their grids, bends alternately on and off, plus a setting with
    energy_tol 2^31 - 1 (same-pitch overlaps); pitch_edges drives keys 0 and 263.  References at the model frames and
    at 10 ms, from each file's first decode with notes dropped and shifted."""
    from basic_pitch_b200.evaluate import note_frames_to_multipitch

    files, grid = _set(edges, name)
    notes, onsets, contours = ([f[k] for f in files] for k in range(3))
    settings = [{**_kw(p), "include_pitch_bends": j % 2 == 0} for j, p in enumerate(grid)]
    settings.append({**_kw(grid[0]), "energy_tol": 2**31 - 1, "include_pitch_bends": True})
    res = model.decode_grid(notes, onsets, contours, settings)
    lens = [a.shape[0] for a in notes]
    rng = np.random.default_rng(8)
    for hop in (None, 0.01):
        mp_refs, mel_refs = [], []
        for i in range(len(files)):
            r = res[0][i]
            t = _times(lens[i] + 1)
            iv = np.stack([t[r["start"]], t[r["end"]]], 1) if len(r["start"]) else np.zeros((0, 2))
            p = np.asarray(r["pitch"], np.float64) + rng.choice([0, 0, 0, 1 / 3, -1 / 3, 1, 12, 0.5], len(r["pitch"]))
            keep = rng.random(len(p)) < 0.85
            times = t[: lens[i]] if hop is None else np.arange(0, lens[i] * 256 / 22050 + 0.05, hop)
            ref = (iv[keep], _hz(p[keep]))
            from basic_pitch_b200.evaluate import notes_to_multipitch

            mp_refs.append((times, notes_to_multipitch(ref[0], ref[1], times)))
            mel_refs.append((times, _notes_f0(ref, times)))
        _check_grid(model, notes, onsets, contours, settings, mp_refs, mel_refs, res)
    if name == "pitch_edges":
        keys = set()
        for per in res:
            for i, r in enumerate(per):
                _, ef = note_frames_to_multipitch(r["start"], r["end"], r["pitch"], _bends(r), lens[i])
                keys |= {round(float(f), 6) for fr in ef for f in fr}
        from basic_pitch_b200.evaluate import BENT_HZ

        assert round(float(BENT_HZ[0]), 6) in keys and round(float(BENT_HZ[263]), 6) in keys


# ------------------------------------------------------------------------------------------------ bends off
def test_bends_off_with_a_null_contour_equals_the_plain_grid(model, edges):
    from basic_pitch_b200 import _lib
    from basic_pitch_b200.evaluate import EST_CHROMA, EST_MIDI, bent_bins

    files, grid = _set(edges, "ties")
    notes = np.ascontiguousarray(np.concatenate([f[0] for f in files]))
    onsets = np.ascontiguousarray(np.concatenate([f[1] for f in files]))
    foff = np.cumsum([0] + [f[0].shape[0] for f in files]).astype(np.int64)
    settings = [{**_kw(p), "include_pitch_bends": False} for p in grid]
    ps = model._grid_params(settings)
    refs = [(_times(f[0].shape[0])[::3], [np.array([261.6, 440.0])] * len(_times(f[0].shape[0])[::3])) for f in files]
    ms, keep = model._multipitch_set(refs, "references")
    _, midi, chroma, _ = bent_bins()
    a = np.full((len(settings), len(files), 7), -1, np.int64)
    b = a.copy()
    model._lib.bp_score_bent_frames_grid_host(model.handle, notes.ctypes.data, onsets.ctypes.data, None,
                                              foff.ctypes.data, len(files), ps, len(settings), C.byref(ms), 0.5,
                                              midi.ctypes.data, chroma.ctypes.data, a.ctypes.data)
    model._lib.bp_score_frames_grid_host(model.handle, notes.ctypes.data, onsets.ctypes.data, foff.ctypes.data,
                                         len(files), ps, len(settings), C.byref(ms), 0.5, EST_MIDI.ctypes.data,
                                         EST_CHROMA.ctypes.data, b.ctypes.data)
    assert a.tobytes() == b.tobytes() and a[..., 1].sum() > 0
    with pytest.raises(_lib.BpError, match=r"null contour posteriorgram, but decode params\[0\] has include_pitch_bends"):
        model._lib.bp_score_bent_frames_grid_host(model.handle, notes.ctypes.data, onsets.ctypes.data, None,
                                                  foff.ctypes.data, len(files), model._grid_params([dict()]), 1,
                                                  C.byref(ms), 0.5, midi.ctypes.data, chroma.ctypes.data, a.ctypes.data)


# ------------------------------------------------------------------------------------------------ chunks, launches
def test_forced_multi_chunk_call_equals_single_setting_calls(model, edges):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    base = []
    for name in ("ties", "long_notes", "nan_file", "runs"):
        base += _set(edges, name)[0]
    files = []
    while sum(f[0].shape[0] for f in files) < 120_000:
        files += base
    notes, onsets, contours = ([f[k] for f in files] for k in range(3))
    lens = [a.shape[0] for a in notes]
    chunk = int(lib.bp_decode_grid_chunk_params(sum(lens), len(files)))
    distinct = [dict(onset_thresh=0.5, frame_thresh=0.3), dict(frame_thresh=0.05, min_note_len=0, infer_onsets=False),
                dict(onset_thresh=0.95, min_note_len=1, energy_tol=64, include_pitch_bends=False),
                dict(onset_thresh=0.0, melodia_trick=False), dict(min_pitch_idx=20, max_pitch_idx=70)]
    settings = [distinct[k % len(distinct)] for k in range(chunk + 3)]
    n_chunks = -(-len(settings) // chunk)
    assert n_chunks >= 2, chunk
    mp_refs = [(np.arange(0, n * 256 / 22050, 0.01), None) for n in lens]
    mp_refs = [(t, [np.array([261.63, 392.0])] * len(t)) for t, _ in mp_refs]
    mel_refs = [(t, np.where(np.arange(len(t)) % 7 == 0, 0.0, 261.63)) for t, _ in mp_refs]
    for call, refs, per_chunk in ((lambda s, r: model.score_frames_grid(notes, onsets, s, r, contours=contours), mp_refs, 6),
                                  (lambda s, r: model.score_note_melody_grid(notes, onsets, contours, s, r), mel_refs, 7)):
        before = model.launch_count
        got = call(settings, refs)
        assert model.launch_count - before == per_chunk * n_chunks
        for j, s in enumerate(distinct):
            before = model.launch_count
            one = call([s], refs)[0]
            assert model.launch_count - before == per_chunk
            for k in range(j, len(settings), len(distinct)):
                np.testing.assert_array_equal(got[k], one, err_msg=f"setting {k}")
        assert got[..., 2].sum() > 0
    # a small grid: the decode's three launches + 3 (bent frames) or + 4 (note melody) whatever the number of settings
    small, _ = _set(edges, "nan_file")
    sn, so, sc = ([f[k] for f in small] for k in range(3))
    srefs_mp = [(np.array([0.1, 0.2]), [np.array([261.6]), np.array([])])] * len(small)
    srefs_mel = [(np.array([0.1, 0.2]), np.array([261.6, 0.0]))] * len(small)
    for p in (1, 64):
        ss = [distinct[k % len(distinct)] for k in range(p)]
        before = model.launch_count
        model.score_frames_grid(sn, so, ss, srefs_mp, contours=sc)
        assert model.launch_count - before == 6
        before = model.launch_count
        model.score_note_melody_grid(sn, so, sc, ss, srefs_mel)
        assert model.launch_count - before == 7
    before = model.launch_count
    assert model.score_note_melody_grid(sn, so, sc, [], srefs_mel).shape == (0, len(small), 7)
    assert model.score_frames_grid([], [], [dict()], [], contours=[]).shape == (1, 0, 7)
    assert model.launch_count == before


# ------------------------------------------------------------------------------------------------ invalid input
def test_invalid_inputs_are_rejected_by_name_without_a_launch(model):
    from basic_pitch_b200 import _lib
    from basic_pitch_b200.evaluate import bent_bins

    T = 6
    notes = np.zeros((3 * T, 88), np.float32)
    onsets = notes.copy()
    contour = np.zeros((3 * T, 264), np.float32)
    foff = np.array([0, T, 2 * T, 3 * T], np.int64)
    _, midi, chroma, cents = bent_bins()
    mp_good = [(np.array([0.0, 0.01]), [np.array([220.0]), np.zeros(0)])] * 3
    mel_good = [(np.array([0.0, 0.1]), np.array([220.0, 0.0]))] * 3
    ok = [dict(), dict(include_pitch_bends=False)]
    out = np.zeros((2, 3, 7), np.int64)
    before = model.launch_count

    def mp(settings=ok, refs=mp_good, c=contour, tm=midi, tc=chroma, window=0.5):
        ms, keep = model._multipitch_set(refs, "references")
        model._lib.bp_score_bent_frames_grid_host(model.handle, notes.ctypes.data, onsets.ctypes.data,
                                                  None if c is None else c.ctypes.data, foff.ctypes.data, 3,
                                                  model._grid_params(settings), len(settings), C.byref(ms), window,
                                                  tm.ctypes.data, tc.ctypes.data, out.ctypes.data)

    def mel(settings=ok, refs=mel_good, c=contour, tab=cents, tol=50.0):
        ms, keep = model._melody_set(refs, "references")
        model._lib.bp_score_note_melody_grid_host(model.handle, notes.ctypes.data, onsets.ctypes.data,
                                                  None if c is None else c.ctypes.data, foff.ctypes.data, 3,
                                                  model._grid_params(settings), len(settings), C.byref(ms), tol,
                                                  tab.ctypes.data, out.ctypes.data)

    def at(a, k, v):
        a = a.copy()
        a[k] = v
        return a

    cases = [
        (lambda: mp(c=None), r"bp_score_bent_frames_grid_host: null contour posteriorgram, but decode params\[0\] has"),
        (lambda: mel(settings=[dict(include_pitch_bends=False), dict()], c=None), r"decode params\[1\] has include_pitch_bends"),
        (lambda: mp(tm=at(midi, 17, 0.0)), "bin table entry 17: midi decreases"),
        (lambda: mp(tc=at(chroma, 5, 12.0)), r"bin table entry 5: chroma outside \[0, 12\)"),
        (lambda: mp(tm=at(midi, 263, np.nan)), "bin table entry 263: non-finite midi"),
        (lambda: mel(tab=at(cents, 0, 0.0)), "bin table entry 0: cents must be > 0"),
        (lambda: mel(tab=at(cents, 17, 0.0)), "bin table entry 17: cents decrease"),
        (lambda: mel(tab=at(cents, 9, np.inf)), "bin table entry 9: non-finite cents"),
        (lambda: mp(refs=[mp_good[0], (np.array([0.0, -0.1]), [np.zeros(0)] * 2), mp_good[0]]),
         "references file 1 frame 1: time < 0"),
        (lambda: mel(refs=[mel_good[0], mel_good[0], (np.array([0.1, 0.05]), np.array([1.0, 1.0]))]),
         "references file 2 frame 1: time decreases"),
        (lambda: mel(tol=0.0), "cent_tolerance must be finite and > 0"),
        (lambda: mp(window=-1.0), "window must be finite and >= 0"),
        (lambda: mp(settings=[dict(), dict(energy_tol=0)]), r"decode params\[1\]: energy_tol must be >= 1"),
        (lambda: mel(settings=[dict(min_note_len=-1)]), r"decode params\[0\]: min_note_len must be >= 0"),
    ]
    for call, msg in cases:
        with pytest.raises(_lib.BpError, match=msg) as e:
            call()
        assert e.value.code == _lib.BP_E_INVALID
    with pytest.raises(ValueError, match="pitch bends need the contour"):
        model.score_note_melody_grid([notes], [onsets], None, [dict()], mel_good[:1])
    assert model.launch_count == before


# ------------------------------------------------------------------------------------------------ Python entry points
def test_evaluate_entry_points_on_arrays_and_a_wav_path(model, golden_dir, tmp_path):
    from scipy.io import wavfile

    from basic_pitch_b200 import inference, synth
    from basic_pitch_b200.audio_io import load_audio_device
    from basic_pitch_b200.evaluate import MELODY_KEYS, frame_scores, melody_scores, notes_to_multipitch
    from basic_pitch_b200.note_creation import grid_setting

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    wav = tmp_path / "vocadito_10.wav"
    wavfile.write(wav, int(zp["sample_rate"]), zp["pcm"])
    z = np.load(golden_dir / "vocadito10.npz")
    voc = (np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"]))
    clip = synth.melody_clip(6.0, 51)
    t_voc = np.arange(1, int(9.5 / HOP_58)) * HOP_58
    t_mel = np.arange(0, 6.0, 0.01)
    f_mel = synth.melody_f0(6.0, 51, t_mel)
    mel_refs = [(t_voc, _notes_f0(voc, t_voc)), (t_mel, f_mel)]
    mp_refs = [(t_voc, notes_to_multipitch(voc[0], voc[1], t_voc)),
               (t_mel, [np.array([f]) if f > 0 else np.zeros(0) for f in f_mel])]
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2, minimum_note_length=58.0),
                dict(minimum_frequency=150.0, maximum_frequency=700.0), dict(melodia_trick=False)]
    audio, _ = load_audio_device(wav, model)
    outs = model.run_inference_arrays([audio, clip])
    notes, onsets, contours = ([o[k] for o in outs] for k in ("note", "onset", "contour"))
    decode = [grid_setting(s, predict_names=True)[0] for s in settings]
    assert all(d["include_pitch_bends"] for d in decode)
    res = model.decode_grid(notes, onsets, contours, decode)
    lens = [a.shape[0] for a in notes]
    for src in ([wav, clip], [audio, clip]):
        counts, scores = inference.evaluate_frames_grid(src, mp_refs, settings, model, pitch_bends=True)
        np.testing.assert_array_equal(counts, _mp_oracle(res, lens, mp_refs))
        ref_scores = frame_scores(counts)
        for k in ("precision", "recall", "accuracy", "chroma_precision"):
            np.testing.assert_array_equal(scores[k], ref_scores[k])
        plain, _ = inference.evaluate_frames_grid(src, mp_refs, settings, model)
        np.testing.assert_array_equal(plain, model.score_frames_grid(notes, onsets, decode, mp_refs))
        counts, scores = inference.evaluate_note_melody_grid(src, mel_refs, settings, model)
        np.testing.assert_array_equal(counts, _mel_oracle(res, notes, mel_refs))
        ref_scores = melody_scores(counts)
        for k in MELODY_KEYS.values():
            np.testing.assert_array_equal(scores[k], ref_scores[k])
            np.testing.assert_array_equal(scores["mean"][k], ref_scores["mean"][k])
    assert scores["raw_pitch_accuracy"][0, 1] > 0.5, scores["raw_pitch_accuracy"]
    flat = [{**d, "include_pitch_bends": False} for d in decode]
    counts, _ = inference.evaluate_note_melody_grid([audio, clip], mel_refs, settings, model, pitch_bends=False,
                                                    cent_tolerance=25.0)
    np.testing.assert_array_equal(counts, _mel_oracle(model.decode_grid(notes, onsets, None, flat), notes, mel_refs, 25.0))
