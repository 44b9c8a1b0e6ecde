"""GPU: onset-only and offset-only scores on the device (onset_offset_kernel of csrc/score.cu, bp_score_onset_offset_* of
csrc/api.cu) and their Python entry points (Model.score_onset_offset_grid, Model.score_onsets_offsets,
inference.evaluate_transcription_grid).

Every count must equal oracle/onset_offset_ref.py (mir_eval 0.7's match_note_onsets / match_note_offsets restated in
NumPy) applied to the notes of the same decode; evaluate_transcription_grid's 14 values must equal the restatement of
mir_eval.transcription.evaluate bit for bit."""
import ctypes as C

import numpy as np
import pytest

from oracle import onset_offset_ref as oo
from tests.test_gpu_decode_edges import _set
from tests.test_gpu_decode_grid import _model_grid
from tests.test_gpu_score import _annotated_clips, _chain, _est_of, _hz, _random_items
from tests.test_onset_offset_cpu import _boundary_sets, _random_set, _tolerance_sets

pytestmark = pytest.mark.gpu

EST_HZ = 440.0 * 2.0 ** ((np.arange(128, dtype=np.float64) - 69.0) / 12.0)  # np.log2 of it is evaluate.EST_LOG2_HZ


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def edges(golden_dir):
    return dict(np.load(golden_dir / "decode_edges.npz"))


def _oracle_grid(res, lens, ref_ivs, **tol):
    out = np.zeros((len(res), len(lens), 4), np.int64)
    for k, per in enumerate(res):
        for i, r in enumerate(per):
            out[k, i] = oo.counts(ref_ivs[i], _est_of(r, lens[i])[0], **tol)
    return out


def _decode(model, notes, onsets, settings):
    return model.decode_grid(notes, onsets, None, [{**s, "include_pitch_bends": False} for s in settings])


# ------------------------------------------------------------------------------------------------ model output, grid
def test_grid_counts_equal_the_oracle_on_model_output(model, golden_dir):
    """The annotated clips of test_gpu_score under 48 settings: _host and _device on a caller stream equal the oracle on
    decode_grid's notes; n_ref / n_est equal score_grid's, and the pitch-aware matched counts (subgraphs) never exceed
    these."""
    import torch

    clips, refs = _annotated_clips(golden_dir)
    outs = model.run_inference_arrays(clips)
    notes, onsets = [o["note"] for o in outs], [o["onset"] for o in outs]
    lens = [a.shape[0] for a in notes]
    settings = _model_grid()
    assert len(settings) >= 48
    ref_ivs = [iv for iv, _ in refs]
    got = model.score_onset_offset_grid(notes, onsets, settings, ref_ivs)
    np.testing.assert_array_equal(got, _oracle_grid(_decode(model, notes, onsets, settings), lens, ref_ivs))
    sc = model.score_grid(notes, onsets, settings, refs)
    np.testing.assert_array_equal(got[..., :2], sc[..., :2])
    assert (got[..., 2] >= sc[..., 2]).all() and (got[..., 3] >= sc[..., 3]).all()
    assert (got[..., 2:] <= np.minimum(got[..., 0], got[..., 1])[..., None]).all()
    assert (got[..., 2] > sc[..., 2]).any() and (got[..., 3] > sc[..., 3]).any() and got[..., 3].sum() > 100

    foff = np.cumsum([0] + lens).astype(np.int64)
    dev = f"cuda:{model.device}"
    d = [torch.from_numpy(np.ascontiguousarray(np.concatenate(x))).to(dev) for x in (notes, onsets)]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    sub = settings[:12]
    ps = model._grid_params(sub)
    ns, keep = model._interval_set(ref_ivs, "references")
    sp = model._score_params({})
    h = np.full((len(sub), len(clips), 4), -7, np.int64)
    with torch.cuda.stream(stream):
        model._lib.bp_score_onset_offset_grid_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), foff.ctypes.data,
                                                     len(clips), ps, len(sub), C.byref(ns), C.byref(sp), None,
                                                     h.ctypes.data, stream.cuda_stream)
    np.testing.assert_array_equal(h, got[: len(sub)])


# ------------------------------------------------------------------------------------------------ explicit notes
def _check_items(model, items, **tol):
    """items [(ref_iv, est_iv)]: score_onsets_offsets equals the oracle item for item."""
    got = model.score_onsets_offsets([e for _, e in items], [r for r, _ in items], **tol)
    for q, (r, e) in enumerate(items):
        assert got[q].tolist() == oo.counts(r, e, **tol), (q, tol)
    return got


def test_explicit_items_equal_the_oracle(model):
    """Duplicates, a chord with one shared onset, chains, the greedy counter-example, distances on the rounding
    boundary, empty sides and random sets on 0.1 ms, 0.05 ms, 1 ms and model-frame grids, under four tolerance sets."""
    rng = np.random.default_rng(31)
    one = np.array([[1.0, 2.0]])
    items = [(np.repeat(one, 64, 0), np.repeat(one, 64, 0)), (np.repeat(one, 3, 0), np.repeat(one, 5, 0)),
             (np.repeat(one, 5, 0), np.repeat(one, 3, 0)),  # duplicates
             (np.array([[3.0, 3.5], [3.0, 3.8], [3.0, 4.0], [3.0, 3.2]]), np.array([[3.0, 3.52], [3.0, 3.9]])),  # chord
             (np.array([[0.0, 1.15], [0.9, 1.0]]), np.array([[0.5, 1.0], [0.6, 1.3]])),  # greedy counter-example
             (np.array([[0.0, 1.15], [0.9, 1.0]]), np.array([[0.6, 1.3], [0.5, 1.0]])),
             (np.zeros((0, 2)), one), (one, np.zeros((0, 2))), (np.zeros((0, 2)), np.zeros((0, 2)))]
    for L in list(range(1, 9)) + [16, 31, 64]:
        for shuffle in (False, True):
            ref_iv, _, est_iv, _ = _chain(L, rng, shuffle)
            items.append((ref_iv, est_iv))
    items += _boundary_sets()
    for grid in (1e-4, 5e-5, 1e-3, None):
        items += [_random_set(rng, grid, span=0.3 if k % 2 else 2.0) for k in range(40)]
    for tol in _tolerance_sets()[1:]:
        _check_items(model, items, **tol)
    got = _check_items(model, items)
    assert got[4, 3] == 2 and got[5, 3] == 2
    assert got[6].tolist() == [0, 1, 0, 0] and got[7].tolist() == [1, 0, 0, 0]


@pytest.mark.parametrize("n_items", [63, 64, 65, 127, 128, 129])
def test_item_counts_around_the_cta_width(model, n_items):
    """Two threads per item and 128 per CTA: item counts around 64 and 128."""
    rng = np.random.default_rng(n_items)
    _check_items(model, [(a, c) for a, _, c, _ in _random_items(rng, n_items, 30)])


def _sparse_counts(ref_iv, est_iv, block=4000, **tol):
    """The oracle's counts for an item too large for dense hit matrices: per block of estimates (in order of the
    tested time), only the references whose tested time lies within the largest limit, through the oracle's hit
    matrices; SciPy's maximum matching size (equal to the oracle's, test_onset_offset_cpu)."""
    import scipy.sparse

    from tests.test_gpu_score import _sparse_max_matching

    tol = {**dict(onset_tolerance=0.05, offset_ratio=0.2, offset_min_tolerance=0.05), **tol}
    out = [len(ref_iv), len(est_iv)]
    for test in (0, 1):
        lim = tol["onset_tolerance"] if test == 0 else max(tol["offset_ratio"] * np.abs(np.diff(ref_iv, axis=-1)).max(),
                                                          tol["offset_min_tolerance"])
        order = np.argsort(ref_iv[:, test], kind="stable")
        r_t = ref_iv[order, test]
        eo = np.argsort(est_iv[:, test], kind="stable")
        rows, cols = [], []
        for e0 in range(0, len(eo), block):
            sl = eo[e0 : e0 + block]
            lo = np.searchsorted(r_t, est_iv[sl, test].min() - lim - 1e-3)
            hi = np.searchsorted(r_t, est_iv[sl, test].max() + lim + 1e-3, side="right")
            idx = order[lo:hi]
            h = (oo.onset_hits(ref_iv[idx], est_iv[sl], tol["onset_tolerance"]) if test == 0 else
                 oo.offset_hits(ref_iv[idx], est_iv[sl], tol["offset_ratio"], tol["offset_min_tolerance"]))
            r, c = np.nonzero(h)
            rows.append(idx[r]), cols.append(sl[c])
        r, c = np.concatenate(rows), np.concatenate(cols)
        m = scipy.sparse.csr_matrix((np.ones(len(r), bool), (r, c)), shape=(len(ref_iv), len(est_iv)))
        out.append(_sparse_max_matching(m))
    return out


def test_item_of_fifty_thousand_notes(model):
    rng = np.random.default_rng(50)
    n = 50_000
    on = np.sort(np.round(rng.uniform(0, 2500, n), 3))
    ref_iv = np.stack([on, on + np.round(rng.uniform(0.05, 2.0, n), 3)], 1)
    jit = np.round(rng.normal(0, 0.03, n), 3)
    est_iv = np.maximum(ref_iv + jit[:, None] + np.round(rng.normal(0, 0.1, (n, 1)), 3) * [0, 1], 0)
    est_iv[:, 1] = np.maximum(est_iv[:, 1], est_iv[:, 0] + 0.01)
    est_iv = est_iv[rng.permutation(n)]
    got = model.score_onsets_offsets([est_iv], [ref_iv])
    assert got[0].tolist() == _sparse_counts(ref_iv, est_iv)
    assert 0 < got[0, 2] < n and 0 < got[0, 3] < n


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
    assert -(-len(settings) // chunk) >= 2, chunk
    first = _decode(model, notes, onsets, distinct[:1])[0]
    rng = np.random.default_rng(3)
    refs = []
    for i, r in enumerate(first):
        iv = _est_of(r, lens[i])[0] + np.round(rng.uniform(-0.06, 0.06, (len(r["start"]), 2)), 3)
        iv[:, 0] = np.maximum(iv[:, 0], 0.0)
        iv[:, 1] = np.maximum(iv[:, 1], iv[:, 0] + 0.01)
        refs.append(iv)
    single = [model.score_onset_offset_grid(notes, onsets, [s], refs)[0] for s in distinct]
    before = model.launch_count
    got = model.score_onset_offset_grid(notes, onsets, settings, refs)
    n_launch = model.launch_count - before
    for k in range(len(settings)):
        np.testing.assert_array_equal(got[k], single[k % len(distinct)], err_msg=f"setting {k}")
    np.testing.assert_array_equal(got[:1], _oracle_grid([first], lens, refs))
    before = model.launch_count
    model.score_grid(notes, onsets, settings, [(iv, _hz(np.full(len(iv), 60))) for iv in refs])
    assert n_launch == model.launch_count - before  # both: the grid decode's launches + 1 per chunk

    small, _ = _set(edges, "nan_file")
    sn, so = [f[0] for f in small], [f[1] for f in small]
    srefs = [np.array([[0.1, 0.5]])] * len(small)
    for p in (1, 64):
        before = model.launch_count
        model.score_onset_offset_grid(sn, so, [distinct[k % len(distinct)] for k in range(p)], srefs)
        assert model.launch_count - before == 4, p  # prep, candidates, loops + the onset / offset kernel
    before = model.launch_count
    model.score_onsets_offsets([srefs[0]] * 3, srefs[:3])
    assert model.launch_count - before == 1
    assert model.score_onsets_offsets([], []).shape == (0, 4)
    assert model.launch_count - before == 1


def test_invalid_inputs_are_rejected_by_index_without_a_launch(model, edges):
    from basic_pitch_b200 import _lib

    files, _ = _set(edges, "nan_file")
    notes, onsets = [f[0] for f in files], [f[1] for f in files]
    n = len(files)
    good = [np.array([[0.1, 0.5], [0.2, 0.9], [1.0, 1.5]]) for _ in range(n)]

    def bad(i, j, col, value):
        refs = [iv.copy() for iv in good]
        refs[i][j, col] = value
        return refs

    cases = [(bad(1, 2, 0, np.nan), "file 1 note 2: non-finite time"), (bad(2, 0, 0, -0.5), "file 2 note 0: onset < 0"),
             (bad(1, 1, 1, 0.2), "file 1 note 1: offset <= onset"), (bad(0, 0, 1, np.inf), "file 0 note 0: non-finite")]
    for refs, msg in cases:
        before = model.launch_count
        with pytest.raises(_lib.BpError) as e:
            model.score_onset_offset_grid(notes, onsets, [dict(), dict(onset_thresh=0.3)], refs)
        assert e.value.code == _lib.BP_E_INVALID and msg in str(e.value), str(e.value)
        assert "bp_score_onset_offset_grid_host: references" in str(e.value)
        with pytest.raises(_lib.BpError) as e:
            model.score_onsets_offsets(good, refs)
        assert e.value.code == _lib.BP_E_INVALID and "references " + msg.replace("file", "item") in str(e.value)
        with pytest.raises(_lib.BpError) as e:
            model.score_onsets_offsets(refs, good)
        assert "estimates " + msg.replace("file", "item") in str(e.value)
        assert model.launch_count == before
    before = model.launch_count
    for tol in (dict(onset_tolerance=-0.01), dict(pitch_tolerance=np.inf), dict(offset_ratio=np.nan),
                dict(offset_min_tolerance=-1.0)):
        with pytest.raises(_lib.BpError) as e:
            model.score_onset_offset_grid(notes, onsets, [dict()], good, **tol)
        assert e.value.code == _lib.BP_E_INVALID and next(iter(tol)) in str(e.value)
        with pytest.raises(_lib.BpError):
            model.score_onsets_offsets(good, good, **tol)
    with pytest.raises(_lib.BpError) as e:
        model.score_onset_offset_grid(notes, onsets, [dict(), dict(energy_tol=0)], good)
    assert "decode params[1]" in str(e.value)
    with pytest.raises(ValueError, match=r"references\[1\]"):
        model.score_onsets_offsets(good[:2], [good[0], np.zeros(3)])
    assert model.launch_count == before
    assert model.score_onset_offset_grid(notes, onsets, [], good).shape == (0, n, 4)
    assert model.launch_count == before


# ------------------------------------------------------------------------------------------------ evaluate_transcription_grid
def test_evaluate_transcription_grid_on_arrays_and_a_wav_path(model, golden_dir, tmp_path):
    from scipy.io import wavfile

    from basic_pitch_b200 import inference, synth
    from basic_pitch_b200.audio_io import load_audio_device
    from basic_pitch_b200.evaluate import TRANSCRIPTION_KEYS
    from basic_pitch_b200.note_creation import grid_setting

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    wav = tmp_path / "vocadito_10.wav"
    wavfile.write(wav, int(zp["sample_rate"]), zp["pcm"])
    z = np.load(golden_dir / "vocadito10.npz")
    clip = synth.random_notes_clip(6.0, 77)
    refs = [(np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"])),
            synth.random_notes_events(6.0, 77), (np.zeros((0, 2)), np.zeros(0))]
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2, minimum_note_length=58.0),
                dict(minimum_frequency=150.0, maximum_frequency=700.0), dict(melodia_trick=False)]
    audio = [wav, clip, synth.random_notes_clip(3.0, 78)]
    counts, scores = inference.evaluate_transcription_grid(audio, refs, settings, model)
    assert counts.shape == (4, 3, 6) and list(scores) == list(TRANSCRIPTION_KEYS.values()) + ["mean"]
    np.testing.assert_array_equal(counts[..., :4], inference.evaluate_grid(audio, refs, settings, model)[0])
    a, _ = load_audio_device(wav, model)
    outs = model.run_inference_arrays([a, *audio[1:]])
    nt, on = [o["note"] for o in outs], [o["onset"] for o in outs]
    decode = [grid_setting(s, predict_names=True)[0] for s in settings]
    np.testing.assert_array_equal(counts[..., 4:], model.score_onset_offset_grid(nt, on, decode,
                                                                                 [iv for iv, _ in refs])[..., 2:])
    res = _decode(model, nt, on, decode)
    for k in range(len(settings)):
        for i, o in enumerate(outs):
            est_iv = _est_of(res[k][i], o["note"].shape[0])[0]
            exp = oo.evaluate(refs[i][0], refs[i][1], est_iv, EST_HZ[res[k][i]["pitch"]])
            for key, name in TRANSCRIPTION_KEYS.items():
                assert scores[name][k, i] == exp[key], (key, k, i)
    for name in TRANSCRIPTION_KEYS.values():
        np.testing.assert_array_equal(scores["mean"][name], scores[name].mean(axis=-1))
    assert counts[0, 0, 4] > 10 and (counts[..., 4] > counts[..., 2]).any()
    assert (scores["onset_f_measure"] > 0).any() and (scores["offset_f_measure"] > 0).any()
    counts2, _ = inference.evaluate_transcription_grid(audio[1:2], refs[1:2], settings[:2], model, onset_tolerance=0.1,
                                                       offset_ratio=0.5)
    np.testing.assert_array_equal(counts2[..., 4:], model.score_onset_offset_grid(
        nt[1:2], on[1:2], decode[:2], [refs[1][0]], onset_tolerance=0.1, offset_ratio=0.5)[..., 2:])
