"""GPU: frame-level multi-pitch scoring on the device (csrc/score_frames.cu, the frame half of csrc/api.cu's scoring)
and its Python entry points (Model.score_frames_grid, Model.score_multipitch, inference.evaluate_frames_grid).

Every count must equal oracle/multipitch_ref.py (mir_eval.multipitch restated in NumPy, SciPy's interp1d and maximum
matching) applied to the piano roll of the notes Model.decode_grid gives for the same (setting, file)."""
import ctypes as C

import numpy as np
import pytest

from oracle import multipitch_ref as mr
from tests import postsets
from tests.test_gpu_decode_edges import _fixture_file, _kw, _set
from tests.test_gpu_decode_grid import _model_grid
from tests.test_gpu_score import _annotated_clips, _hz

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def edges(golden_dir):
    return dict(np.load(golden_dir / "decode_edges.npz"))


def _times(n):
    from basic_pitch_b200 import _lib

    t = np.zeros(n)
    _lib.load().bp_frame_times(n, t.ctypes.data)
    return t


def _est_values(res, T):
    """Decode arrays of one file -> its estimate series as (midi, chroma) per frame: the piano roll at the model frames."""
    from basic_pitch_b200.evaluate import EST_CHROMA, EST_MIDI

    roll = np.zeros((T, 128), np.int64)
    for a, b, p in zip(res["start"], res["end"], res["pitch"]):
        roll[a:b, p] += 1
    return _times(T), [(np.repeat(EST_MIDI, r), np.repeat(EST_CHROMA, r)) for r in roll]


_memo = {}


def _tp(rm, rc, em, ec, window):
    key = (rm.tobytes(), rc.tobytes(), em.tobytes(), ec.tobytes(), window)
    if key not in _memo:
        _memo[key] = (mr.max_matching(mr.hit_matrix(rm, em, window, False)),
                      mr.max_matching(mr.hit_matrix(rc, ec, window, True)))
    return _memo[key]


def _oracle(ref_t, ref_vals, est_t, est_vals, window=0.5):
    """mr.counts_values with the per-frame matchings memoised (sustained notes repeat the same frame many times)."""
    idx = mr.resample_index(est_t, ref_t)
    out = np.zeros(7, np.int64)
    empty = (np.zeros(0), np.zeros(0))
    for k, (rm, rc) in enumerate(ref_vals):
        em, ec = est_vals[idx[k]] if idx[k] >= 0 else empty
        r, e = len(rm), len(em)
        tp = _tp(np.asarray(rm), np.asarray(rc), em, ec, window) if r and e else (0, 0)
        out += [r, e, tp[0], tp[1], min(r, e), max(r - e, 0), max(e - r, 0)]
    return out


def _vals(series):
    from basic_pitch_b200.evaluate import multipitch_values

    t, freqs = series
    return np.asarray(t, np.float64), [multipitch_values(np.asarray(f, np.float64)) for f in freqs]


def _oracle_grid(grid_res, lens, refs, window=0.5):
    out = np.zeros((len(grid_res), len(lens), 7), np.int64)
    rv = [_vals(r) for r in refs]
    for k, per in enumerate(grid_res):
        for i, res in enumerate(per):
            et, ev = _est_values(res, lens[i])
            out[k, i] = _oracle(rv[i][0], rv[i][1], et, ev, window)
    return out


def _series_from_notes(refs, times):
    from basic_pitch_b200.evaluate import notes_to_multipitch

    return (times, notes_to_multipitch(refs[0], refs[1], times))


# ------------------------------------------------------------------------------------------------ model output, grid
def test_grid_counts_equal_the_oracle_on_model_output(model, golden_dir):
    """Nine annotated clips under 48 settings, references at the model frames, 10 ms, 5 ms, 23 ms and jittered hops:
    bp_score_frames_grid_host and bp_score_frames_grid_device on a caller stream equal the oracle."""
    import torch

    from basic_pitch_b200.evaluate import EST_CHROMA, EST_MIDI

    from basic_pitch_b200 import synth

    clips, notes_refs = _annotated_clips(golden_dir)
    clips.append(synth.dense_chords_clip(4.0, seed=920))
    notes_refs.append(synth.dense_chords_events(4.0))
    outs = model.run_inference_arrays(clips)
    notes, onsets = [o["note"] for o in outs], [o["onset"] for o in outs]
    lens = [a.shape[0] for a in notes]
    settings = _model_grid()
    assert len(settings) >= 48 and len(clips) >= 9
    res = model.decode_grid(notes, onsets, None, [{**s, "include_pitch_bends": False} for s in settings])
    rng = np.random.default_rng(12)
    hops = {"model": None, "10ms": 0.01, "5ms": 0.005, "23ms": 0.023, "jitter": -1}
    for name, hop in hops.items():
        refs = []
        for i, nr in enumerate(notes_refs):
            dur = max(lens[i] * 256 / 22050, 0.5)
            if hop is None:
                t = _times(lens[i])
            elif hop > 0:
                t = np.arange(0, dur, hop)
            else:
                t = np.sort(np.round(np.arange(0, dur, 0.01) + rng.uniform(-0.004, 0.004, len(np.arange(0, dur, 0.01))), 5))
                t = np.maximum(t, 0.0)
            refs.append(_series_from_notes(nr, t))
        sel = settings if name in ("model", "10ms") else settings[::4]
        rsel = res if name in ("model", "10ms") else res[::4]
        exp = _oracle_grid(rsel, lens, refs)
        got = model.score_frames_grid(notes, onsets, sel, refs)
        np.testing.assert_array_equal(got, exp, err_msg=name)
        assert exp[..., 2].sum() > 1000 and exp[..., 3].sum() >= exp[..., 2].sum(), name
        if name == "model":
            foff = np.cumsum([0] + lens).astype(np.int64)
            dev = f"cuda:{model.device}"
            d = [torch.from_numpy(np.ascontiguousarray(np.concatenate(x))).to(dev) for x in (notes, onsets)]
            stream = torch.cuda.Stream(device=dev)
            torch.cuda.synchronize(dev)
            ps = model._grid_params(settings)
            ms, keep = model._multipitch_set(refs, "references")
            got = np.full((len(settings), len(clips), 7), -1, np.int64)
            with torch.cuda.stream(stream):
                model._lib.bp_score_frames_grid_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), foff.ctypes.data,
                                                       len(clips), ps, len(settings), C.byref(ms), 0.5,
                                                       EST_MIDI.ctypes.data, EST_CHROMA.ctypes.data, got.ctypes.data,
                                                       stream.cuda_stream)
            np.testing.assert_array_equal(got, exp)
            for w in (0.0, 1.0, 6.0):
                np.testing.assert_array_equal(model.score_frames_grid(notes, onsets, settings[:6], refs, window=w),
                                              _oracle_grid(res[:6], lens, refs, w), err_msg=str(w))


def test_golden_vocadito_scores_perfectly_against_its_own_events(model, golden_dir):
    z = np.load(golden_dir / "vocadito10.npz")
    T = z["gold_note"].shape[0]
    t = _times(T + 1)
    start, end = np.asarray(z["gold_events/start"]), np.asarray(z["gold_events/end"])
    # the events' times are the model frame times of their frames
    s_idx, e_idx = np.searchsorted(t, start), np.searchsorted(t, end)
    assert (t[s_idx] == start).all() and (t[e_idx] == end).all()
    ref = _series_from_notes((np.stack([start, end], 1), _hz(z["gold_events/pitch"])), t[:T])
    counts = model.score_frames_grid([z["gold_note"]], [z["gold_onset"]], [dict()], [ref])
    n = sum(len(f) for f in ref[1])
    assert n > 100
    assert counts.tolist() == [[[n, n, n, n, n, 0, 0]]]


# ------------------------------------------------------------------------------------------------ adversarial decodes
@pytest.mark.parametrize("name", postsets.NAMES)
def test_adversarial_sets(model, edges, name):
    """The pinned sets of tests/postsets.py under their grids (lengths has files of 0, 1 and 2 frames; crowded reruns a
    chunk for its slots; several carry overlapping notes of one pitch): references at the model frames and at 10 ms,
    made from each file's first decode with notes dropped, shifted a semitone or an octave."""
    files, grid = _set(edges, name)
    notes, onsets = [f[0] for f in files], [f[1] for f in files]
    lens = [a.shape[0] for a in notes]
    rng = np.random.default_rng(7)
    res = [[_fixture_file(edges, f"{name}/p{j}", i) for i in range(len(files))] for j in range(len(grid))]
    settings = [_kw(p) for p in grid]
    multi = 0
    for hop in (None, 0.01):
        refs = []
        for i in range(len(files)):
            r = res[0][i]
            t = _times(lens[i] + 1)
            iv = np.stack([t[r["start"]], t[r["end"]]], 1) if len(r["start"]) else np.zeros((0, 2))
            p = np.asarray(r["pitch"], np.float64) + rng.choice([0, 0, 0, 1, 12, -12, 0.5], len(r["pitch"]))
            keep = rng.random(len(p)) < 0.85
            times = t[: lens[i]] if hop is None else np.arange(0, lens[i] * 256 / 22050 + 0.05, hop)
            refs.append(_series_from_notes((iv[keep], _hz(p[keep])), times))
        exp = _oracle_grid(res, lens, refs)
        got = model.score_frames_grid(notes, onsets, settings, refs)
        np.testing.assert_array_equal(got, exp, err_msg=str(hop))
    for per in res:
        for i, r in enumerate(per):
            roll = np.zeros((max(lens[i], 1), 128), np.int64)
            for a, b, p in zip(r["start"], r["end"], r["pitch"]):
                roll[a:b, p] += 1
            multi = max(multi, roll.max())
    if name in ("ties", "runs", "nan_file", "lengths"):
        assert multi > 1, name  # the roll carries multiplicities above 1


# ------------------------------------------------------------------------------------------------ explicit series
def _mp(model, items, window):
    """bp_score_multipitch_host on items [(ref_t, ref_vals, est_t, est_vals)] with (midi, chroma) given as bits."""
    from basic_pitch_b200 import _lib

    def ms(sets):
        f_off = np.cumsum([0] + [len(t) for t, _ in sets]).astype(np.int64)
        vals = [v for _, vs in sets for v in vs]
        v_off = np.cumsum([0] + [len(m) for m, _ in vals]).astype(np.int64)
        cat = lambda xs: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), np.float64)
        arrs = (f_off, cat([t for t, _ in sets]), v_off, cat([m for m, _ in vals]), cat([c for _, c in vals]))
        s = _lib.MultipitchSet()
        s.frame_off, s.time_s, s.value_off, s.midi, s.chroma = (a.ctypes.data for a in arrs)
        return s, arrs

    r, kr = ms([(a, b) for a, b, _, _ in items])
    e, ke = ms([(c, d) for _, _, c, d in items])
    out = np.full((len(items), 7), -1, np.int64)
    model._lib.bp_score_multipitch_host(model.handle, C.byref(e), C.byref(r), len(items), float(window), out.ctypes.data)
    return out


def _rand_vals(rng, n_frames, max_vals, spread):
    out = []
    for _ in range(n_frames):
        k = rng.integers(0, max_vals + 1)
        m = 60.0 + rng.integers(-spread, spread + 1, k) + rng.choice([0.0, 0.5, -0.5, 0.25, 1e-12, 11.999999], k)
        out.append((m, np.mod(np.mod(m, 12), 12)))
    return out


def test_score_multipitch_random_and_adversarial(model):
    rng = np.random.default_rng(21)
    items = []
    for hop_r, hop_e in ((0.01, 0.01), (0.01, 0.0116), (0.005, 0.023)):
        tr, te = np.arange(40) * hop_r, np.arange(35) * hop_e
        items.append((tr, _rand_vals(rng, 40, 6, 14), te, _rand_vals(rng, 35, 6, 14)))
    # frames of several hundred values, dense pitch sets: augmenting paths through many groups
    t = np.arange(4) * 0.01
    items.append((t, _rand_vals(rng, 4, 400, 30), t, _rand_vals(rng, 4, 300, 30)))
    # chroma wrap: 11.8 against 0.2, values just below 12 against 0
    wrap = (np.array([59.8, 71.99999999999999, 47.9]), np.mod(np.array([59.8, 71.99999999999999, 47.9]), 12))
    zero = (np.array([72.2, 60.0, 36.1]), np.mod(np.array([72.2, 60.0, 36.1]), 12))
    items.append((t[:1], [wrap], t[:1], [zero]))
    items.append((t[:1], [zero], t[:1], [wrap]))
    # duplicates, empty frames on either side, an empty series
    dup = (np.full(5, 60.0), np.zeros(5))
    two = (dup[0][:2], dup[1][:2])
    items.append((t[:3], [dup, (np.zeros(0), np.zeros(0)), dup], t[:3], [two, two, (np.zeros(0), np.zeros(0))]))
    items.append((t, _rand_vals(rng, 4, 3, 3), np.zeros(0), []))
    items.append((np.zeros(0), [], t, _rand_vals(rng, 4, 3, 3)))
    for window in (0.0, 0.25, 0.5, 5.5, 12.0):
        got = _mp(model, items, window)
        for q, it in enumerate(items):
            assert got[q].tolist() == mr.counts_values(*it, window=window), (q, window)
    assert _mp(model, items[3:4], 0.5)[0, 2] > 200


def test_score_multipitch_item_of_a_million_frames(model):
    rng = np.random.default_rng(6)
    K = 1_000_000
    tr = np.arange(K) * 0.01
    te = np.arange(int(K * 0.01 / 0.0116)) * 0.0116
    vocab = [(np.zeros(0), np.zeros(0))] + [
        (m, np.mod(np.mod(m, 12), 12)) for m in (np.array([60.0]), np.array([60.0, 64.0]), np.array([48.0, 60.4, 67.0]),
                                                 np.array([72.6]), np.array([60.0, 60.0]))]
    ref_vals = [vocab[k] for k in rng.integers(0, len(vocab), K)]
    est_vals = [vocab[k] for k in rng.integers(0, len(vocab), len(te))]
    got = _mp(model, [(tr, ref_vals, te, est_vals)], 0.5)
    exp = _oracle(tr, ref_vals, te, est_vals)
    assert got[0].tolist() == exp.tolist()
    assert 0 < got[0, 2] < got[0, 3] < got[0, 0]


# ------------------------------------------------------------------------------------------------ chunks, launches, errors
def test_chunked_grid_and_launch_counts(model, edges):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    base = []
    for name in ("ties", "long_notes", "nan_file", "runs", "crowded"):
        base += _set(edges, name)[0]
    files = []
    while sum(f[0].shape[0] for f in files) < 120_000:
        files += base
    notes, onsets = [f[0] for f in files], [f[1] for f in files]
    lens = [a.shape[0] for a in notes]
    chunk = int(lib.bp_decode_grid_chunk_params(sum(lens), len(files)))
    distinct = [dict(onset_thresh=0.5, frame_thresh=0.3), dict(frame_thresh=0.05, min_note_len=0, infer_onsets=False),
                dict(onset_thresh=0.95, min_note_len=1, energy_tol=64), dict(onset_thresh=0.0, melodia_trick=False),
                dict(min_pitch_idx=20, max_pitch_idx=70)]
    settings = [distinct[k % len(distinct)] for k in range(chunk + 3)]
    n_chunks = -(-len(settings) // chunk)
    assert n_chunks >= 2, chunk
    res = model.decode_grid(notes, onsets, None, [{**s, "include_pitch_bends": False} for s in distinct])
    refs = []
    for i, r in enumerate(res[0]):
        et, ev = _est_values(r, lens[i])
        t = np.arange(0, lens[i] * 256 / 22050, 0.01)
        hz = [2.0 ** ((m - 69.0) / 12.0) * 440.0 for m, _ in ev]
        idx = mr.resample_index(et, t)
        refs.append((t, [hz[j] if j >= 0 else np.zeros(0) for j in idx]))
    single = _oracle_grid(res, lens, refs)
    got = model.score_frames_grid(notes, onsets, settings, refs)
    for k in range(len(settings)):
        np.testing.assert_array_equal(got[k], single[k % len(distinct)], err_msg=f"setting {k}")

    small, _ = _set(edges, "nan_file")
    sn, so = [f[0] for f in small], [f[1] for f in small]
    srefs = [(np.array([0.1, 0.2]), [np.array([261.6]), np.array([])])] * len(small)
    deltas = []
    for p in (1, 64):
        before = model.launch_count
        model.score_frames_grid(sn, so, [distinct[k % len(distinct)] for k in range(p)], srefs)
        deltas.append(model.launch_count - before)
    assert deltas == [6, 6], deltas  # prep, candidates, loops + roll scatter, roll prefix sum, match
    before = model.launch_count
    model.score_multipitch(srefs[:3], srefs[:3])
    assert model.launch_count - before == 1


def test_invalid_inputs_are_rejected_by_index_without_a_launch(model, edges):
    from basic_pitch_b200 import _lib

    files, _ = _set(edges, "nan_file")
    notes, onsets = [f[0] for f in files], [f[1] for f in files]
    n = len(files)

    def good():
        return [(np.array([0.0, 0.1, 0.2]), [np.array([261.6]), np.array([]), np.array([220.0, 440.0])]) for _ in range(n)]

    def bad_time(i, k, v):
        r = good()
        r[i][0][k] = v
        return r

    def bad_hz(i, k, j, v):
        r = good()
        r[i][1][k][j] = v
        return r

    cases = [(bad_time(1, 2, np.nan), "file 1 frame 2: non-finite time"), (bad_time(0, 0, -0.5), "file 0 frame 0: time < 0"),
             (bad_time(2, 2, 0.05), "file 2 frame 2: time decreases"),
             (bad_hz(0, 2, 1, 0.0), "file 0 frame 2 value 1: non-finite midi"),
             (bad_hz(2, 0, 0, -3.0), "file 2 frame 0 value 0: non-finite midi")]
    for refs, msg in cases:
        before = model.launch_count
        with pytest.raises(_lib.BpError) as e:
            model.score_frames_grid(notes, onsets, [dict(), dict(onset_thresh=0.3)], refs)
        assert e.value.code == _lib.BP_E_INVALID and msg in str(e.value) and "references" in str(e.value), str(e.value)
        with pytest.raises(_lib.BpError) as e:
            model.score_multipitch(good(), refs)
        assert msg.replace("file", "item") in str(e.value) and "references" in str(e.value), str(e.value)
        with pytest.raises(_lib.BpError) as e:
            model.score_multipitch(refs, good())
        assert "estimates item" in str(e.value) and model.launch_count == before
    # chroma outside [0, 12), through the C ABI
    t0 = (np.array([0.0]), [(np.array([60.0]), np.array([12.0]))])
    before = model.launch_count
    with pytest.raises(_lib.BpError, match="item 0 frame 0 value 0: chroma outside"):
        _mp(model, [(*t0, *t0)], 0.5)
    for w in (-0.1, np.inf, np.nan):
        with pytest.raises(_lib.BpError, match="window"):
            model.score_frames_grid(notes, onsets, [dict()], good(), window=w)
        with pytest.raises(_lib.BpError, match="window"):
            model.score_multipitch(good(), good(), window=w)
    # the estimate tables
    from basic_pitch_b200.evaluate import EST_CHROMA, EST_MIDI

    ps = model._grid_params([dict()])
    ms, keep = model._multipitch_set(good(), "references")
    foff = np.cumsum([0] + [a.shape[0] for a in notes]).astype(np.int64)
    n_all, o_all = np.concatenate(notes), np.concatenate(onsets)
    out = np.zeros((1, n, 7), np.int64)
    for tm, tc, msg in ((np.where(np.arange(128) == 40, np.nan, EST_MIDI), EST_CHROMA, "entry 40: non-finite midi"),
                        (np.where(np.arange(128) == 41, 0.0, EST_MIDI), EST_CHROMA, "entry 41: midi decreases"),
                        (EST_MIDI, np.where(np.arange(128) == 7, 12.0, EST_CHROMA), "entry 7: chroma outside")):
        tm, tc = np.ascontiguousarray(tm), np.ascontiguousarray(tc)
        with pytest.raises(_lib.BpError, match=msg):
            model._lib.bp_score_frames_grid_host(model.handle, n_all.ctypes.data, o_all.ctypes.data, foff.ctypes.data, n,
                                                 ps, 1, C.byref(ms), 0.5, tm.ctypes.data, tc.ctypes.data, out.ctypes.data)
    with pytest.raises(_lib.BpError) as e:
        model.score_frames_grid(notes, onsets, [dict(), dict(energy_tol=0)], good())
    assert "decode params[1]" in str(e.value)
    assert model.score_frames_grid(notes, onsets, [], good()).shape == (0, n, 7)
    assert model.score_multipitch([], []).shape == (0, 7)
    assert model.launch_count == before


# ------------------------------------------------------------------------------------------------ evaluate_frames_grid
def test_evaluate_frames_grid_on_arrays_and_a_wav_path(model, golden_dir, tmp_path):
    from scipy.io import wavfile

    from basic_pitch_b200 import inference, synth
    from basic_pitch_b200.audio_io import load_audio_device
    from basic_pitch_b200.evaluate import frame_scores
    from basic_pitch_b200.note_creation import grid_setting

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    wav = tmp_path / "vocadito_10.wav"
    wavfile.write(wav, int(zp["sample_rate"]), zp["pcm"])
    z = np.load(golden_dir / "vocadito10.npz")
    voc = (np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"]))
    clip = synth.random_notes_clip(6.0, 77)
    clip_notes = synth.random_notes_events(6.0, 77)
    refs = [_series_from_notes(voc, np.arange(0, 9.5, 0.01)), _series_from_notes(clip_notes, np.arange(0, 6.0, 0.01))]
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2, minimum_note_length=58.0),
                dict(minimum_frequency=150.0, maximum_frequency=700.0), dict(melodia_trick=False)]
    counts, scores = inference.evaluate_frames_grid([wav, clip], refs, settings, model)
    audio, _ = load_audio_device(wav, model)
    outs = model.run_inference_arrays([audio, clip])
    decode = [{**grid_setting(s, predict_names=True)[0], "include_pitch_bends": False} for s in settings]
    res = model.decode_grid([o["note"] for o in outs], [o["onset"] for o in outs], None, decode)
    exp = _oracle_grid(res, [o["note"].shape[0] for o in outs], refs)
    np.testing.assert_array_equal(counts, exp)
    ref_scores = frame_scores(exp)
    for k in ("precision", "recall", "accuracy", "total_error", "chroma_precision"):
        np.testing.assert_array_equal(scores[k], ref_scores[k])
        np.testing.assert_array_equal(scores["mean"][k], ref_scores["mean"][k])
    assert counts[0, 0, 2] > 100
    counts2, _ = inference.evaluate_frames_grid([audio, clip], refs, settings, model, window=1.0)
    np.testing.assert_array_equal(counts2, _oracle_grid(res, [o["note"].shape[0] for o in outs], refs, 1.0))
