"""GPU: posteriorgrams scored as multi-f0 estimates on the device (the posteriorgram kind of csrc/score_frames.cu's match
kernel, bp_score_salience_grid_* in csrc/api.cu) and their Python entry points (Model.score_salience_grid,
inference.evaluate_salience_grid).

Every count must equal oracle/multipitch_ref.py (mir_eval.multipitch restated with SciPy) applied to
evaluate.salience_to_multipitch of the same posteriorgram and setting, or, for tables other than the model's, to the
bins the rule of include/bp_b200.h selects cell by cell."""
import ctypes as C

import numpy as np
import pytest

from oracle import multipitch_ref as mr
from tests.test_gpu_frame_score import _oracle, _series_from_notes, _times, _vals
from tests.test_gpu_score import _annotated_clips, _hz

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def clips_outs(model, golden_dir):
    clips, notes_refs = _annotated_clips(golden_dir)
    return clips, notes_refs, model.run_inference_arrays(clips)


def _grid(kind):
    """Thresholds 0.05 .. 0.95, peak picking on and off, the whole range, a middle range, a range cut inside a bin gap
    and an empty range."""
    from basic_pitch_b200.evaluate import salience_bins

    hz = salience_bins(kind)[0]
    n = len(hz)
    ranges = [(None, None), (hz[n // 4], hz[3 * n // 4]), (hz[10] * 1.0001, hz[n - 10] * 0.9999), (hz[n // 2], hz[n // 3])]
    return [dict(threshold=t, peak_picking=p, minimum_frequency=a, maximum_frequency=b)
            for t in (0.05, 0.2, 0.35, 0.5, 0.65, 0.8, 0.95) for p in (True, False) for a, b in ranges]


def _oracle_grid(grams, settings, refs, kind, window=0.5):
    from basic_pitch_b200.evaluate import salience_to_multipitch

    out = np.zeros((len(settings), len(grams), 7), np.int64)
    rv = [_vals(r) for r in refs]
    for k, s in enumerate(settings):
        for i, g in enumerate(grams):
            et, ev = _vals(salience_to_multipitch(g, kind=kind, **s))
            out[k, i] = _oracle(rv[i][0], rv[i][1], et, ev, window)
    return out


# ------------------------------------------------------------------------------------------------ model output
@pytest.mark.parametrize("kind", ["contour", "note"])
def test_grid_counts_equal_the_oracle_on_model_output(model, clips_outs, kind):
    """The annotated clips (an empty one and one without annotations among them) under thresholds 0.05 .. 0.95, peak
    picking on and off and four frequency ranges, one empty: references at a 10 ms hop (interp1d map) and at the model
    frame times (identity map)."""
    import torch

    from basic_pitch_b200.evaluate import salience_bins

    clips, notes_refs, outs = clips_outs
    grams = [o[kind] for o in outs]
    lens = [g.shape[0] for g in grams]
    settings = _grid(kind)
    for hop in (0.01, None):
        refs = []
        for i, nr in enumerate(notes_refs):
            t = _times(lens[i]) if hop is None else np.arange(0, max(lens[i] * 256 / 22050, 0.5), hop)
            refs.append(_series_from_notes(nr, t))
        sel = settings if (hop is not None and kind == "contour") else settings[::3]
        exp = _oracle_grid(grams, sel, refs, kind)
        got = model.score_salience_grid(grams, sel, refs, kind=kind)
        np.testing.assert_array_equal(got, exp, err_msg=f"{kind} {hop}")
        assert exp[..., 2].sum() > 1000 and exp[..., 1].sum() > exp[..., 2].sum(), (kind, hop)
        empty = [k for k, s in enumerate(sel) if s["minimum_frequency"] is not None and s["maximum_frequency"] is not None
                 and s["minimum_frequency"] > s["maximum_frequency"]]
        assert empty and (exp[empty, :, 1] == 0).all()  # the empty range
    # the same through bp_score_salience_grid_device on a caller stream, against mir_eval's own entry point restated
    hz, midi, chroma = salience_bins(kind)
    dev = f"cuda:{model.device}"
    d = torch.from_numpy(np.ascontiguousarray(np.concatenate(grams), np.float32)).to(dev)
    foff = np.cumsum([0] + lens).astype(np.int64)
    ps = model._salience_params(settings[:8], kind)
    ms, keep = model._multipitch_set(refs, "references")
    got = np.full((8, len(grams), 7), -1, np.int64)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    with torch.cuda.stream(stream):
        model._lib.bp_score_salience_grid_device(model.handle, d.data_ptr(), len(hz), foff.ctypes.data, len(grams), ps, 8,
                                                 C.byref(ms), 0.5, midi.ctypes.data, chroma.ctypes.data,
                                                 got.ctypes.data, stream.cuda_stream)
    from basic_pitch_b200.evaluate import salience_to_multipitch

    for k in range(8):
        for i in (0, 3):
            et, ef = salience_to_multipitch(grams[i], kind=kind, **settings[k])
            assert got[k, i].tolist() == mr.counts(refs[i][0], refs[i][1], et, ef), (k, i)
    for w in (0.0, 1.0, 6.0):
        np.testing.assert_array_equal(model.score_salience_grid(grams, settings[:4], refs, kind=kind, window=w),
                                      _oracle_grid(grams, settings[:4], refs, kind, w), err_msg=str(w))


def test_a_contour_scores_perfectly_against_its_own_estimate(model, clips_outs):
    """The reference is the clip's own contour estimate under setting s: s scores tp = n_ref = n_est with no miss or
    false alarm, and for every peak-picking choice n_est does not increase with the threshold."""
    from basic_pitch_b200.evaluate import salience_bins, salience_to_multipitch

    _, _, outs = clips_outs
    grams = [o["contour"] for o in outs]
    hz = salience_bins("contour")[0]
    thresholds = [round(0.05 * k, 2) for k in range(1, 20)]
    settings = [dict(threshold=t, peak_picking=p) for p in (True, False) for t in thresholds]
    settings += [dict(threshold=t, peak_picking=True, minimum_frequency=hz[60], maximum_frequency=hz[200])
                 for t in thresholds]
    for own in (settings[5], settings[19 + 1], settings[38 + 9]):
        refs = [salience_to_multipitch(g, **own) for g in grams]
        counts = model.score_salience_grid(grams, settings, refs)
        c = counts[settings.index(own)]
        n = c[:, 0]
        assert n.sum() > 300
        np.testing.assert_array_equal(c[:, 1], n)
        np.testing.assert_array_equal(c[:, 2], n)
        np.testing.assert_array_equal(c[:, 3], n)
        np.testing.assert_array_equal(c[:, 4], n)
        assert (c[:, 5] == 0).all() and (c[:, 6] == 0).all()
        for g0 in range(0, len(settings), len(thresholds)):
            n_est = counts[g0 : g0 + len(thresholds), :, 1]
            assert (np.diff(n_est, axis=0) <= 0).all()
            assert n_est[0].sum() > n_est[-1].sum()
        assert (counts[len(thresholds) : 2 * len(thresholds), :, 1] >= counts[: len(thresholds), :, 1]).all()


# ------------------------------------------------------------------------------------------------ adversarial
def _ms(sets):
    """bp_multipitch_set_t of [(times, [(midi, chroma) per frame])] given as bits."""
    from basic_pitch_b200 import _lib

    f_off = np.cumsum([0] + [len(t) for t, _ in sets]).astype(np.int64)
    vals = [v for _, vs in sets for v in vs]
    v_off = np.cumsum([0] + [len(m) for m, _ in vals]).astype(np.int64)
    cat = lambda xs: np.ascontiguousarray(np.concatenate(xs) if xs else np.zeros(0), np.float64)  # noqa: E731
    arrs = (f_off, cat([np.asarray(t, np.float64) for t, _ in sets]), v_off, cat([m for m, _ in vals]),
            cat([c for _, c in vals]))
    s = _lib.MultipitchSet()
    s.frame_off, s.time_s, s.value_off, s.midi, s.chroma = (a.ctypes.data for a in arrs)
    return s, arrs


def _call(model, grams, params, refs, tab, window=0.5, device=False):
    """bp_score_salience_grid_host (or _device, from a torch copy of the posteriorgrams) on raw arguments."""
    import torch

    from basic_pitch_b200 import _lib

    width = len(tab[0])
    foff = np.cumsum([0] + [g.shape[0] for g in grams]).astype(np.int64)
    g_all = np.ascontiguousarray(np.concatenate(grams) if grams else np.zeros((0, width)), np.float32)
    ps = (_lib.SalienceParams * max(len(params), 1))(*[_lib.SalienceParams(*p, 0) for p in params])
    ms, keep = _ms(refs)
    midi, chroma = (np.ascontiguousarray(a, np.float64) for a in tab)
    out = np.full((len(params), len(grams), 7), -1, np.int64)
    if device:
        dev = f"cuda:{model.device}"
        d = torch.from_numpy(g_all).to(dev) if g_all.size else None
        torch.cuda.synchronize(dev)
        model._lib.bp_score_salience_grid_device(model.handle, d.data_ptr() if d is not None else None, width,
                                                 foff.ctypes.data, len(grams), ps, len(params), C.byref(ms), window,
                                                 midi.ctypes.data, chroma.ctypes.data, out.ctypes.data,
                                                 torch.cuda.current_stream(dev).cuda_stream)
    else:
        model._lib.bp_score_salience_grid_host(model.handle, g_all.ctypes.data, width, foff.ctypes.data, len(grams), ps,
                                               len(params), C.byref(ms), window, midi.ctypes.data, chroma.ctypes.data,
                                               out.ctypes.data)
    return out


def _est_bins(gram, thr, peak, lo, hi):
    """Estimate bins of every frame by the rule of include/bp_b200.h, cell by cell."""
    out = []
    for row in np.asarray(gram, np.float32):
        w = len(row)
        out.append(np.array([b for b in range(lo, hi) if float(row[b]) >= thr and (
            not peak or (1 <= b <= w - 2 and row[b] > row[b - 1] and row[b] > row[b + 1]))], np.int64))
    return out


def _oracle_raw(grams, params, refs, tab, window):
    midi, chroma = tab
    out = np.zeros((len(params), len(grams), 7), np.int64)
    for k, (thr, peak, lo, hi) in enumerate(params):
        for i, g in enumerate(grams):
            ev = [(midi[b], chroma[b]) for b in _est_bins(g, thr, peak, lo, hi)]
            out[k, i] = mr.counts_values(refs[i][0], refs[i][1], _times(g.shape[0]), ev, window=window)
    return out


def _tables(width):
    from basic_pitch_b200.evaluate import multipitch_values, salience_bins

    if width == 264:
        return salience_bins("contour")[1:]
    m = np.array([60.0, 60.0, 72.4, 72.6][:width]) if width < 4 else 40.0 + np.arange(width) / 3.0  # equal entries
    return m, np.mod(np.mod(m, 12), 12)


@pytest.mark.parametrize("width", [1, 2, 3, 264])
def test_adversarial_posteriorgrams_host_and_device(model, width):
    """Plateaus, ties at the threshold, NaN cells and all-zero frames; files of 0 and 1 frames; reference frames at the
    first estimate time (frame 0 is at 0 s, so none can lie before it), past the last, repeated and empty; a file with
    no reference frame.  _host and _device agree bit for bit and with the rule."""
    rng = np.random.default_rng(width)
    tab = _tables(width)
    pool = np.array([0.0, 0.25, 0.5, 0.5, 0.75, 1.0, np.nan], np.float32)
    grams = []
    for T in (0, 1, 9, 1, 0, 30):
        g = rng.choice(pool, size=(T, width))
        if T >= 9:
            g[2] = 0.0
            g[3] = 0.5
            g[4, ::2] = 0.75
            g[5] = np.nan
            g[6, : width // 2 + 1] = 1.0
        grams.append(g)
    lo_hi = sorted({(0, width), (min(1, width), max(width - 1, min(1, width))), (width // 2, width // 2), (0, 1)})
    params = [(thr, peak, lo, hi) for thr in (1e-9, 0.25, 0.5, 0.75, 1.0) for peak in (0, 1) for lo, hi in lo_hi]
    refs = []
    for i, g in enumerate(grams):
        T = g.shape[0]
        if i == 4:
            refs.append((np.zeros(0), []))
            continue
        et = _times(max(T, 1))
        t = np.sort(np.concatenate([[0.0, 0.0], rng.uniform(0, et[-1] + 0.2, 12), [et[-1], et[-1] + 0.01, 5.0]]))
        vals = []
        for k in range(len(t)):
            n = rng.integers(0, 5)
            m = np.where(rng.random(n) < 0.6, rng.choice(tab[0], n), rng.uniform(tab[0][0] - 1, tab[0][-1] + 13, n))
            vals.append((m, np.mod(np.mod(m, 12), 12)))
        refs.append((t, vals))
    refs[1] = (_times(1), [(np.array([tab[0][0]]), np.array([tab[1][0]]))])  # identity map on a 1-frame file
    for window in (0.5, 1.0):
        host = _call(model, grams, params, refs, tab, window)
        dev = _call(model, grams, params, refs, tab, window, device=True)
        assert host.tobytes() == dev.tobytes()
        np.testing.assert_array_equal(host, _oracle_raw(grams, params, refs, tab, window), err_msg=str(window))
    if width >= 3:
        assert host[..., 2].sum() > 0 and host[..., 1].sum() > host[..., 2].sum()
    assert (host[:, 4, 0] == 0).all() and (host[:, 0, 1] == 0).all()


# ------------------------------------------------------------------------------------------------ chunks, launches
def test_chunked_grid_equals_per_setting_calls_and_launch_counts(model):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    rng = np.random.default_rng(4)
    tab = _tables(264)
    T, K, per = 3000, 2_000_000, 8
    gram = rng.choice(np.array([0.0, 0.1, 0.3, 0.5, 0.7, 0.9], np.float32), size=(T, 264))
    t = np.linspace(0.0, _times(T)[-1] + 0.05, K)
    m = rng.choice(tab[0], K * per) + rng.choice([0.0, 0.0, 0.2, 12.0, -0.6], K * per)
    c = np.mod(np.mod(m, 12), 12)
    ms = _lib.MultipitchSet()
    arrs = (np.array([0, K], np.int64), t, np.arange(0, K * per + 1, per, dtype=np.int64), m, c)
    ms.frame_off, ms.time_s, ms.value_off, ms.midi, ms.chroma = (a.ctypes.data for a in arrs)
    chunk = int(lib.bp_score_salience_chunk_params(K, K * per))
    assert chunk == 7
    params = [(0.05 + 0.1 * k, k % 2, 5 * k, 264 - 3 * k) for k in range(9)]
    n_chunks = -(-len(params) // chunk)
    foff = np.array([0, T], np.int64)
    midi, chroma = tab
    g = np.ascontiguousarray(gram)

    def run(ps_list):
        ps = (_lib.SalienceParams * len(ps_list))(*[_lib.SalienceParams(*p, 0) for p in ps_list])
        out = np.full((len(ps_list), 1, 7), -1, np.int64)
        model._lib.bp_score_salience_grid_host(model.handle, g.ctypes.data, 264, foff.ctypes.data, 1, ps, len(ps_list),
                                               C.byref(ms), 0.5, midi.ctypes.data, chroma.ctypes.data, out.ctypes.data)
        return out

    before = model.launch_count
    got = run(params)
    assert model.launch_count - before == n_chunks == 2
    for k, p in enumerate(params):
        before = model.launch_count
        np.testing.assert_array_equal(got[k], run([p])[0], err_msg=str(k))
        assert model.launch_count - before == 1
    assert got[:, 0, 2].min() > 0 and got[:, 0, 0].tolist() == [K * per] * len(params)

    # a small grid is one launch whatever the number of settings; an empty one none
    small = [np.zeros((4, 264), np.float32), np.zeros((0, 264), np.float32)]
    srefs = [(np.array([0.0, 0.02]), [np.array([261.6]), np.array([])])] * 2
    for n in (1, 64):
        before = model.launch_count
        model.score_salience_grid(small, [dict(threshold=0.1 + 0.01 * k) for k in range(n)], srefs)
        assert model.launch_count - before == 1
    before = model.launch_count
    assert model.score_salience_grid(small, [], srefs).shape == (0, 2, 7)
    assert model.score_salience_grid([], [dict(threshold=0.5)], []).shape == (1, 0, 7)
    assert model.launch_count == before


def test_invalid_inputs_are_rejected_by_index_without_a_launch(model):
    from basic_pitch_b200 import _lib

    grams = [np.zeros((5, 264), np.float32)] * 3
    good = [(np.array([0.0, 0.1]), [np.array([261.6]), np.array([])])] * 3
    ok = dict(threshold=0.5)
    before = model.launch_count
    for k, bad, msg in ((2, dict(threshold=0.0), "salience params[2]: threshold must be finite and > 0"),
                        (1, dict(threshold=-0.5), "salience params[1]: threshold"),
                        (3, dict(threshold=np.nan), "salience params[3]: threshold"),
                        (0, dict(threshold=np.inf), "salience params[0]: threshold")):
        settings = [ok] * 4
        settings[k] = bad
        with pytest.raises(_lib.BpError, match=msg.replace("[", r"\[").replace("]", r"\]")) as e:
            model.score_salience_grid(grams, settings, good)
        assert e.value.code == _lib.BP_E_INVALID
    tab = _tables(264)
    refs = [(np.array([0.0]), [(np.array([60.0]), np.array([0.0]))])] * 3
    cases = [(dict(params=[(0.5, 2, 0, 264)]), r"salience params\[0\]: peak_pick must be 0 or 1"),
             (dict(params=[(0.5, 1, 0, 264), (0.5, 0, 10, 9)]), r"salience params\[1\]: need 0 <= bin_lo"),
             (dict(params=[(0.5, 0, -1, 9)]), r"salience params\[0\]: need"),
             (dict(params=[(0.5, 0, 0, 265)]), r"salience params\[0\]: need"),
             (dict(tab=(np.where(np.arange(264) == 17, tab[0][16] - 1, tab[0]), tab[1])), "bin table entry 17: midi decreases"),
             (dict(tab=(np.where(np.arange(264) == 5, np.nan, tab[0]), tab[1])), "bin table entry 5: non-finite midi"),
             (dict(tab=(tab[0], np.where(np.arange(264) == 9, 12.0, tab[1]))), "bin table entry 9: chroma outside"),
             (dict(refs=[refs[0], (np.array([0.0, -1.0]), refs[0][1] * 2), refs[0]]), "references file 1 frame 1: time < 0"),
             (dict(refs=[refs[0], refs[0], (np.array([0.0]), [(np.array([60.0]), np.array([12.5]))])]),
              "references file 2 frame 0 value 0: chroma outside"),
             (dict(window=-1.0), "window"), (dict(window=np.nan), "window")]
    for over, msg in cases:
        kw = dict(grams=grams, params=[(0.5, 1, 0, 264)], refs=refs, tab=tab, window=0.5)
        kw.update(over)
        with pytest.raises(_lib.BpError, match=msg):
            _call(model, kw["grams"], kw["params"], kw["refs"], kw["tab"], kw["window"])
    # width and frame offsets, through the C ABI
    ps = (_lib.SalienceParams * 1)(_lib.SalienceParams(0.5, 1, 0, 1, 0))
    ms, keep = _ms(refs)
    out = np.zeros((1, 3, 7), np.int64)
    g = np.zeros((15, 1024 + 1), np.float32)
    big = np.zeros(1025)
    for width, foff, msg in ((0, [0, 5, 10, 15], r"width must be in \[1, 1024\]"),
                             (1025, [0, 5, 10, 15], r"width must be in \[1, 1024\]"),
                             (1, [1, 5, 10, 15], r"frame_off\[0\] must be 0"),
                             (1, [0, 5, 4, 15], "file 1: bad frame_off")):
        foff = np.array(foff, np.int64)
        with pytest.raises(_lib.BpError, match=msg):
            model._lib.bp_score_salience_grid_host(model.handle, g.ctypes.data, width, foff.ctypes.data, 3, ps, 1,
                                                   C.byref(ms), 0.5, big.ctypes.data, big.ctypes.data, out.ctypes.data)
    with pytest.raises(TypeError):
        model.score_salience_grid(grams, [dict(threshold=0.5, frame_thresh=0.3)], good)
    with pytest.raises(ValueError):
        model.score_salience_grid([np.zeros((5, 88), np.float32)], [ok], good[:1])
    assert model.launch_count == before


# ------------------------------------------------------------------------------------------------ evaluate_salience_grid
@pytest.mark.parametrize("kind", ["contour", "note"])
def test_evaluate_salience_grid_on_arrays_and_a_wav_path(model, golden_dir, tmp_path, kind):
    from scipy.io import wavfile

    from basic_pitch_b200 import inference, synth
    from basic_pitch_b200.audio_io import load_audio_device
    from basic_pitch_b200.evaluate import frame_scores

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    wav = tmp_path / "vocadito_10.wav"
    wavfile.write(wav, int(zp["sample_rate"]), zp["pcm"])
    z = np.load(golden_dir / "vocadito10.npz")
    voc = (np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"]))
    clip = synth.random_notes_clip(6.0, 78)
    refs = [_series_from_notes(voc, np.arange(0, 9.5, 0.01)),
            _series_from_notes(synth.random_notes_events(6.0, 78), np.arange(0, 6.0, 0.01))]
    settings = [dict(threshold=0.3), dict(threshold=0.5, peak_picking=False),
                dict(threshold=0.2, minimum_frequency=150.0, maximum_frequency=700.0)]
    counts, scores = inference.evaluate_salience_grid([wav, clip], refs, settings, kind=kind, model_or_model_path=model)
    audio, _ = load_audio_device(wav, model)
    outs = model.run_inference_arrays([audio, clip])
    exp = model.score_salience_grid([o[kind] for o in outs], settings, refs, kind=kind)
    np.testing.assert_array_equal(counts, exp)
    np.testing.assert_array_equal(exp, _oracle_grid([o[kind] for o in outs], settings, refs, kind))
    ref_scores = frame_scores(exp)
    for k in ("precision", "recall", "accuracy", "total_error", "chroma_precision"):
        np.testing.assert_array_equal(scores[k], ref_scores[k])
        np.testing.assert_array_equal(scores["mean"][k], ref_scores["mean"][k])
    assert counts[0, 0, 2] > 100
    counts2, _ = inference.evaluate_salience_grid([audio, clip], refs, settings, kind, model, window=1.0)
    np.testing.assert_array_equal(counts2, model.score_salience_grid([o[kind] for o in outs], settings, refs, kind=kind,
                                                                     window=1.0))
