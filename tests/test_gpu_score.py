"""GPU: note-level scoring on the device (csrc/score.cu, the bp_score_* half of csrc/api.cu) and its Python entry points
(Model.score_grid, Model.score_notes, inference.evaluate_grid).

Every count must equal oracle/transcription_ref.py (mir_eval.transcription's hit matrices restated in NumPy, SciPy's
maximum matching) applied to the notes of the same decode."""
import ctypes as C

import numpy as np
import pytest

from oracle import transcription_ref as tr
from tests import postsets
from tests.test_gpu_decode_edges import _fixture_file, _kw, _set
from tests.test_gpu_decode_grid import _model_grid
from tests.test_score_cpu import fifty_cents

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
    from basic_pitch_b200.note_creation import model_frames_to_time

    return model_frames_to_time(n)


def _est_of(res, n_frames):
    """Decode arrays of one file -> (intervals, log2 Hz) as note_events_batch / mir_eval would see them."""
    from basic_pitch_b200.evaluate import EST_LOG2_HZ

    t = _times(max(n_frames, 1) + 1)
    iv = np.stack([t[res["start"]], t[res["end"]]], 1) if len(res["start"]) else np.zeros((0, 2))
    return iv, EST_LOG2_HZ[np.asarray(res["pitch"], np.int64)]


def _oracle(ref_iv, ref_l2, est_iv, est_l2, **tol):
    tol = {**tr.TOLERANCES, **tol}
    n_ref, n_est = len(ref_l2), len(est_l2)
    if n_ref == 0 or n_est == 0:
        return [n_ref, n_est, 0, 0]
    a, b = tr.hit_matrices(ref_iv, ref_l2, est_iv, est_l2, **tol)
    return [n_ref, n_est, tr.max_matching(a), tr.max_matching(b)]


def _oracle_grid(grid_res, lens, refs, **tol):
    """grid_res[setting][file] decode arrays; refs[file] = (intervals, Hz)."""
    out = np.zeros((len(grid_res), len(lens), 4), np.int64)
    for k, per in enumerate(grid_res):
        for i, r in enumerate(per):
            est_iv, est_l2 = _est_of(r, lens[i])
            out[k, i] = _oracle(refs[i][0], np.log2(refs[i][1]), est_iv, est_l2, **tol)
    return out


def _hz(midi):
    from basic_pitch_b200.note_creation import midi_to_hz

    return midi_to_hz(np.asarray(midi, np.float64))


# ------------------------------------------------------------------------------------------------ model output, grid
def _annotated_clips(golden_dir):
    from basic_pitch_b200 import synth

    z = np.load(golden_dir / "vocadito10.npz")
    clips = [z["audio22k"].astype(np.float32)]
    refs = [(np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"]))]
    for k, (sec, nps) in enumerate(((4.0, 5.0), (7.5, 3.0), (12.0, 8.0))):
        clips.append(synth.random_notes_clip(sec, 900 + k, nps))
        refs.append(synth.random_notes_events(sec, 900 + k, nps))
    clips.append(synth.dense_chords_clip(3.0, seed=910))
    refs.append(synth.dense_chords_events(3.0))
    clips.append(synth.tones_clip(2.0, seed=911))
    refs.append((np.array([[0.0, 2.0]] * 3), _hz([57, 64, 72])))
    clips.append(np.zeros(0, np.float32))
    refs.append((np.array([[0.5, 1.0]]), _hz([60])))
    clips.append(synth.random_notes_clip(5.0, 913))
    refs.append((np.zeros((0, 2)), np.zeros(0)))  # no annotation at all
    return clips, refs


def _cat_refs(model, refs):
    return model._note_set(refs, "references")


def test_grid_counts_equal_the_oracle_on_model_output(model, golden_dir):
    """About eight annotated clips, >= 48 settings: bp_score_grid_device on a caller stream and bp_score_grid_host equal
    the oracle applied to Model.decode_grid's notes of every (setting, file)."""
    import torch

    from basic_pitch_b200.evaluate import EST_LOG2_HZ

    clips, refs = _annotated_clips(golden_dir)
    outs = model.run_inference_arrays(clips)
    notes, onsets = [o["note"] for o in outs], [o["onset"] for o in outs]
    lens = [a.shape[0] for a in notes]
    settings = _model_grid()
    assert len(settings) >= 48
    exp = _oracle_grid(model.decode_grid(notes, onsets, None, [{**s, "include_pitch_bends": False} for s in settings]),
                       lens, refs)
    assert exp[..., 2].sum() > 300 and (exp[..., 3] < exp[..., 2]).any() and (exp[..., 2] < exp[..., 1]).any()

    host = model.score_grid(notes, onsets, settings, refs)
    np.testing.assert_array_equal(host, exp)

    foff = np.cumsum([0] + lens).astype(np.int64)
    dev = f"cuda:{model.device}"
    d = [torch.from_numpy(np.ascontiguousarray(np.concatenate(x))).to(dev) for x in (notes, onsets)]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    ps = model._grid_params(settings)
    ns, keep = _cat_refs(model, refs)
    sp = model._score_params({})
    got = np.full((len(settings), len(clips), 4), -1, np.int64)
    with torch.cuda.stream(stream):
        model._lib.bp_score_grid_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), foff.ctypes.data, len(clips), ps,
                                        len(settings), C.byref(ns), C.byref(sp), EST_LOG2_HZ.ctypes.data,
                                        got.ctypes.data, stream.cuda_stream)
    np.testing.assert_array_equal(got, exp)
    # a looser and a tighter tolerance set, host entry point
    for tol in (dict(onset_tolerance=0.1, pitch_tolerance=150.0, offset_ratio=0.5), dict(onset_tolerance=0.0)):
        np.testing.assert_array_equal(model.score_grid(notes, onsets, settings[:6], refs, **tol),
                                      _oracle_grid(model.decode_grid(notes, onsets, None, [{**s, "include_pitch_bends": False}
                                                                                           for s in settings[:6]]),
                                                   lens, refs, **tol), err_msg=str(tol))


def test_golden_vocadito_scores_perfectly_against_its_own_events(model, golden_dir):
    z = np.load(golden_dir / "vocadito10.npz")
    n = len(z["gold_events/pitch"])
    refs = [(np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"]))]
    counts = model.score_grid([z["gold_note"]], [z["gold_onset"]], [dict()], refs)
    assert counts.tolist() == [[[n, n, n, n]]]


# ------------------------------------------------------------------------------------------------ adversarial decodes
def _boundary_refs(est_iv, est_l2, rng):
    """References made by moving each decoded note onto one side of one predicate boundary (kinds cycle)."""
    iv, l2 = est_iv.copy(), est_l2.copy()
    kind = np.arange(len(l2)) % 8
    for j, k in enumerate(kind):
        on, off = iv[j]
        if k == 0:
            iv[j] = (on + 0.05, off + 0.05)  # rounds to exactly the onset tolerance: hit
        elif k == 1:
            iv[j] = (on + 0.05006, off + 0.05006)  # rounds above: miss
        elif k == 2:
            iv[j, 1] = off + max(0.2 * (off - on), 0.05)  # offset at its tolerance (up to rounding)
        elif k == 3:
            iv[j, 1] = off + max(0.2 * (off - on), 0.05) + 0.0003  # offset beyond it
        elif k == 4:
            l2[j] = l2[j] + 50.0 / 1200.0 * (1 - 1e-12)  # just within 50 cents
        elif k == 5:
            l2[j] = l2[j] + 50.0 / 1200.0 * (1 + 1e-9)  # just beyond
        elif k == 6:
            l2[j] = l2[j] - 1.0 / 12.0  # a semitone down: a neighbour bucket, no hit
    if len(l2):
        keep = rng.random(len(l2)) < 0.9
        iv, l2 = iv[keep], l2[keep]
    return iv, l2


@pytest.mark.parametrize("name", postsets.NAMES)
def test_adversarial_sets_against_boundary_references(model, edges, name):
    """The pinned sets of tests/postsets.py under their grids (crowded reruns a chunk for its slots): references sit on
    either side of every predicate boundary around the notes the oracle decodes; every count equals the oracle."""
    files, grid = _set(edges, name)
    notes, onsets = [f[0] for f in files], [f[1] for f in files]
    lens = [a.shape[0] for a in notes]
    rng = np.random.default_rng(41)
    refs_l2, refs = [], []
    for i in range(len(files)):
        est_iv, est_l2 = _est_of(_fixture_file(edges, f"{name}/p0", i), lens[i])
        iv, l2 = _boundary_refs(est_iv, est_l2, rng)
        refs_l2.append(l2)
        refs.append((iv, 2.0**l2))
    settings = [_kw(p) for p in grid]
    exp = np.zeros((len(grid), len(files), 4), np.int64)
    live = np.zeros(4, bool)
    for j in range(len(grid)):
        for i in range(len(files)):
            est_iv, est_l2 = _est_of(_fixture_file(edges, f"{name}/p{j}", i), lens[i])
            ref_l2 = np.log2(refs[i][1])
            exp[j, i] = _oracle(refs[i][0], ref_l2, est_iv, est_l2)
            if len(ref_l2) and len(est_l2) and j == 0:
                a, b = tr.hit_matrices(refs[i][0], ref_l2, est_iv, est_l2, **tr.TOLERANCES)
                live |= [a.any(), (~a).any(), (a & ~b).any(), b.any()]
    got = model.score_grid(notes, onsets, settings, refs)
    np.testing.assert_array_equal(got, exp)
    if exp[0, :, 1].sum() > 8:  # each boundary is live on both sides: hits, misses, and hits lost to the offset test
        assert live.all(), (name, live)


# ------------------------------------------------------------------------------------------------ explicit notes
def _score_notes_log2(model, items, **tol):
    """bp_score_notes_host on items [(ref_iv, ref_l2, est_iv, est_l2)] with log2 values given as bits."""
    from basic_pitch_b200 import _lib

    def ns(sets):
        off = np.cumsum([0] + [len(l2) for _, l2 in sets]).astype(np.int64)
        iv = np.concatenate([np.asarray(x, np.float64).reshape(-1, 2) for x, _ in sets]) if sets else np.zeros((0, 2))
        l2 = np.concatenate([np.asarray(y, np.float64) for _, y in sets]) if sets else np.zeros(0)
        arrs = (off, np.ascontiguousarray(iv[:, 0]), np.ascontiguousarray(iv[:, 1]), np.ascontiguousarray(l2))
        s = _lib.NoteSet()
        s.note_off, s.onset_s, s.offset_s, s.log2_hz = (a.ctypes.data for a in arrs)
        return s, arrs

    r, kr = ns([(a, b) for a, b, _, _ in items])
    e, ke = ns([(c, d) for _, _, c, d in items])
    sp = model._score_params(tol)
    out = np.full((len(items), 4), -1, np.int64)
    model._lib.bp_score_notes_host(model.handle, C.byref(e), C.byref(r), len(items), C.byref(sp), out.ctypes.data)
    return out


def _chain(L, rng, shuffle):
    """An item whose greedy pass leaves one estimate free that only an augmenting path of 2 L + 1 edges matches: e_k hits
    r_k and r_k+1 (onsets 0.03 apart, tolerance 0.02), and r_k+1 comes first in the kernel's scan."""
    t = 10.0 - 0.03 * np.arange(L + 1)
    ref_iv = np.stack([t, t + 1.0], 1)
    est_iv = np.stack([t - 0.015, t - 0.015 + 1.0], 1)
    l2 = np.full(L + 1, 8.0)
    order = rng.permutation(L + 1) if shuffle else np.arange(L + 1)
    return ref_iv, l2, est_iv[order], l2


def test_score_notes_on_adversarial_items(model):
    rng = np.random.default_rng(9)
    items = []
    for L in list(range(1, 9)) + [16, 31, 64]:  # augmenting paths of 3 .. 129 edges
        items.append(_chain(L, rng, False))
        items.append(_chain(L, rng, True))
    one = np.array([[1.0, 2.0]])
    items.append((np.repeat(one, 64, 0), np.full(64, 7.0), np.repeat(one, 64, 0), np.full(64, 7.0)))  # 64 x 64
    # ties at exactly 50 cents between notes of neighbouring semitone buckets (and the next double beyond)
    a, b, nb = fifty_cents(-0.03)
    assert np.rint(12 * (a - np.log2(440.0)) + 69) != np.rint(12 * (b - np.log2(440.0)) + 69)
    items.append((one, [a], one, [b]))
    items.append((one, [b], one, [a]))
    items.append((one, [a], one, [nb]))
    items.append((np.repeat(one, 3, 0), np.full(3, 6.0), np.repeat(one, 5, 0), np.full(5, 6.0)))  # duplicates
    items.append((np.zeros((0, 2)), np.zeros(0), one, [6.0]))  # empty sides
    items.append((one, [6.0], np.zeros((0, 2)), np.zeros(0)))
    items.append((np.zeros((0, 2)), np.zeros(0), np.zeros((0, 2)), np.zeros(0)))
    got = _score_notes_log2(model, items, onset_tolerance=0.02)
    for q, it in enumerate(items):
        assert got[q].tolist() == _oracle(*it, onset_tolerance=0.02), q
    for q, L in enumerate(list(range(1, 9)) + [16, 31, 64]):
        assert got[2 * q].tolist() == [L + 1] * 4
    assert got[2 * 11].tolist() == [64] * 4
    assert got[2 * 11 + 1, 2] == 1 and got[2 * 11 + 2, 2] == 1 and got[2 * 11 + 3, 2] == 0


def _random_items(rng, n_items, n_max, grid=0.01):
    items = []
    for _ in range(n_items):
        nr, ne = rng.integers(0, n_max, 2)
        def notes(n):
            on = np.round(rng.uniform(0, 3, n) / grid) * grid
            iv = np.stack([on, on + np.round(rng.uniform(0.02, 1.0, n) / grid) * grid], 1)
            l2 = np.log2(440.0) + (rng.integers(-4, 5, n) + rng.choice([0.0, 0.25, 0.5, 1.25, -0.5], n)) / 12.0
            return iv, l2
        items.append((*notes(nr), *notes(ne)))
    return items


@pytest.mark.parametrize("cents", [0.0, 50.0, 150.0])
def test_score_notes_tolerance_grid(model, cents):
    rng = np.random.default_rng(int(cents) + 1)
    items = _random_items(rng, 40, 60)
    for onset in (0.0, 0.05, 0.5):
        for ratio in (0.0, 0.2, 5.0):
            tol = dict(onset_tolerance=onset, pitch_tolerance=cents, offset_ratio=ratio)
            got = _score_notes_log2(model, items, **tol)
            for q, it in enumerate(items):
                assert got[q].tolist() == _oracle(*it, **tol), (q, tol)


def _sparse_oracle(ref_iv, ref_l2, est_iv, est_l2, block=4000):
    """The oracle for an item too large for dense hit matrices: per block of estimates, only the references whose onset
    can round into the window, through the same hit_matrices."""
    import scipy.sparse

    order = np.argsort(ref_iv[:, 0], kind="stable")
    r_on = ref_iv[order, 0]
    rows, cols, rows1, cols1 = [], [], [], []
    for e0 in range(0, len(est_l2), block):
        sl = slice(e0, e0 + block)
        lo = np.searchsorted(r_on, est_iv[sl, 0].min() - 0.06)
        hi = np.searchsorted(r_on, est_iv[sl, 0].max() + 0.06, side="right")
        idx = order[lo:hi]
        a, b = tr.hit_matrices(ref_iv[idx], ref_l2[idx], est_iv[sl], est_l2[sl], **tr.TOLERANCES)
        ra, ca = np.nonzero(a)
        rb, cb = np.nonzero(b)
        rows.append(idx[ra]), cols.append(ca + e0), rows1.append(idx[rb]), cols1.append(cb + e0)
    out = [len(ref_l2), len(est_l2)]
    for r, c in ((rows, cols), (rows1, cols1)):
        r, c = np.concatenate(r), np.concatenate(c)
        m = scipy.sparse.csr_matrix((np.ones(len(r), bool), (r, c)), shape=(len(ref_l2), len(est_l2)))
        out.append(_sparse_max_matching(m))
    return out


def _sparse_max_matching(m):
    from scipy.sparse.csgraph import maximum_bipartite_matching

    if m.nnz == 0:
        return 0
    return int((maximum_bipartite_matching(m, perm_type="column") >= 0).sum())


def test_score_notes_item_of_fifty_thousand_notes(model):
    rng = np.random.default_rng(50)
    n = 50_000
    on = np.sort(np.round(rng.uniform(0, 2500, n), 3))
    ref_iv = np.stack([on, on + np.round(rng.uniform(0.05, 2.0, n), 3)], 1)
    ref_l2 = np.log2(440.0) + rng.integers(-30, 30, n) / 12.0
    jit = np.round(rng.normal(0, 0.03, n), 3)
    est_iv = np.maximum(ref_iv + jit[:, None] + np.round(rng.normal(0, 0.1, (n, 1)), 3) * [0, 1], 0)
    est_iv[:, 1] = np.maximum(est_iv[:, 1], est_iv[:, 0] + 0.01)
    est_l2 = ref_l2 + rng.choice([0.0, 0.0, 1 / 24, 1 / 12], n)
    perm = rng.permutation(n)
    got = _score_notes_log2(model, [(ref_iv, ref_l2, est_iv[perm], est_l2[perm])])
    assert got[0].tolist() == _sparse_oracle(ref_iv, ref_l2, est_iv[perm], est_l2[perm])
    assert 0 < got[0, 3] < got[0, 2] < n


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
    n = len(files)
    chunk = int(lib.bp_decode_grid_chunk_params(sum(lens), n))
    distinct = [dict(onset_thresh=0.5, frame_thresh=0.3), dict(frame_thresh=0.05, min_note_len=0, infer_onsets=False),
                dict(onset_thresh=0.95, min_note_len=1, energy_tol=64), dict(onset_thresh=0.0, melodia_trick=False),
                dict(min_pitch_idx=20, max_pitch_idx=70)]
    settings = [distinct[k % len(distinct)] for k in range(chunk + 3)]
    assert -(-len(settings) // chunk) >= 2, chunk
    first = model.decode_grid(notes, onsets, None, [{**distinct[0], "include_pitch_bends": False}])[0]
    rng = np.random.default_rng(3)
    refs = []
    for i, r in enumerate(first):
        iv, l2 = _est_of(r, lens[i])
        iv = iv + np.round(rng.uniform(-0.06, 0.06, (len(iv), 1)), 3)
        iv[:, 0] = np.maximum(iv[:, 0], 0.0)
        refs.append((iv, 2.0**l2))
    single = _oracle_grid(model.decode_grid(notes, onsets, None, [{**s, "include_pitch_bends": False} for s in distinct]),
                          lens, refs)
    got = model.score_grid(notes, onsets, settings, refs)
    for k in range(len(settings)):
        np.testing.assert_array_equal(got[k], single[k % len(distinct)], err_msg=f"setting {k}")

    small, _ = _set(edges, "nan_file")
    sn, so = [f[0] for f in small], [f[1] for f in small]
    srefs = [(np.array([[0.1, 0.5]]), _hz([60]))] * len(small)
    deltas = []
    for p in (1, 64):
        before = model.launch_count
        model.score_grid(sn, so, [distinct[k % len(distinct)] for k in range(p)], srefs)
        deltas.append(model.launch_count - before)
    assert deltas == [4, 4], deltas  # prep, candidates, loops + the match kernel
    before = model.launch_count
    model.score_notes([srefs[0]] * 3, srefs[:3])
    assert model.launch_count - before == 1


def test_invalid_inputs_are_rejected_by_index_without_a_launch(model, edges):
    from basic_pitch_b200 import _lib

    files, _ = _set(edges, "nan_file")
    notes, onsets = [f[0] for f in files], [f[1] for f in files]
    n = len(files)
    good = [(np.array([[0.1, 0.5], [0.2, 0.9], [1.0, 1.5]]), _hz([60, 62, 64])) for _ in range(n)]

    def bad(i, j, col, value, hz=None):
        refs = [(iv.copy(), p.copy()) for iv, p in good]
        if col is not None:
            refs[i][0][j, col] = value
        else:
            refs[i][1][j] = hz
        return refs

    cases = [(bad(1, 2, 0, np.nan), "file 1 note 2: non-finite time"), (bad(0, 1, 1, np.inf), "file 0 note 1: non-finite time"),
             (bad(2, 0, 0, -0.5), "file 2 note 0: onset < 0"), (bad(1, 1, 1, 0.2), "file 1 note 1: offset <= onset"),
             (bad(0, 2, None, None, 0.0), "file 0 note 2: non-finite log2_hz"),
             (bad(2, 1, None, None, -3.0), "file 2 note 1: non-finite log2_hz")]
    for refs, msg in cases:
        before = model.launch_count
        with pytest.raises(_lib.BpError) as e:
            model.score_grid(notes, onsets, [dict(), dict(onset_thresh=0.3)], refs)
        assert e.value.code == _lib.BP_E_INVALID and msg in str(e.value), (msg, str(e.value))
        assert model.launch_count == before
        with pytest.raises(_lib.BpError) as e:
            model.score_notes(good, refs)
        assert e.value.code == _lib.BP_E_INVALID and msg.replace("file", "item") in str(e.value), str(e.value)
        assert "references" in str(e.value)
        with pytest.raises(_lib.BpError) as e:
            model.score_notes(refs, good)
        assert "estimates item" in str(e.value) and model.launch_count == before
    for tol in (dict(onset_tolerance=-0.01), dict(pitch_tolerance=np.inf), dict(offset_ratio=np.nan),
                dict(offset_min_tolerance=-1.0)):
        before = model.launch_count
        with pytest.raises(_lib.BpError) as e:
            model.score_grid(notes, onsets, [dict()], good, **tol)
        assert e.value.code == _lib.BP_E_INVALID and next(iter(tol)) in str(e.value)
        with pytest.raises(_lib.BpError):
            model.score_notes(good, good, **tol)
        assert model.launch_count == before
    before = model.launch_count
    with pytest.raises(_lib.BpError) as e:
        model.score_grid(notes, onsets, [dict(), dict(energy_tol=0)], good)
    assert "decode params[1]" in str(e.value) and model.launch_count == before
    assert model.score_grid(notes, onsets, [], good).shape == (0, n, 4)
    assert model.score_notes([], []).shape == (0, 4)
    assert model.launch_count == before


# ------------------------------------------------------------------------------------------------ evaluate_grid
def test_evaluate_grid_on_arrays_and_a_wav_path(model, golden_dir, tmp_path):
    from scipy.io import wavfile

    from basic_pitch_b200 import inference, synth
    from basic_pitch_b200.audio_io import load_audio_device
    from basic_pitch_b200.evaluate import note_scores
    from basic_pitch_b200.note_creation import grid_setting

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    wav = tmp_path / "vocadito_10.wav"
    wavfile.write(wav, int(zp["sample_rate"]), zp["pcm"])
    z = np.load(golden_dir / "vocadito10.npz")
    voc_ref = (np.stack([z["gold_events/start"], z["gold_events/end"]], 1), _hz(z["gold_events/pitch"]))
    clip = synth.random_notes_clip(6.0, 77)
    clip_ref = synth.random_notes_events(6.0, 77)
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2, minimum_note_length=58.0),
                dict(minimum_frequency=150.0, maximum_frequency=700.0), dict(melodia_trick=False)]
    counts, scores = inference.evaluate_grid([wav, clip], [voc_ref, clip_ref], settings, model)
    audio, _ = load_audio_device(wav, model)
    outs = model.run_inference_arrays([audio, clip])
    decode = [{**grid_setting(s, predict_names=True)[0], "include_pitch_bends": False} for s in settings]
    res = model.decode_grid([o["note"] for o in outs], [o["onset"] for o in outs], None, decode)
    exp = _oracle_grid(res, [o["note"].shape[0] for o in outs], [voc_ref, clip_ref])
    np.testing.assert_array_equal(counts, exp)
    ref_scores = note_scores(exp)
    for k in ("precision", "recall", "f_measure", "f_measure_no_offset"):
        np.testing.assert_array_equal(scores[k], ref_scores[k])
        np.testing.assert_array_equal(scores["mean"][k], ref_scores["mean"][k])
    assert counts[0, 0, 3] > 10
    counts2, _ = inference.evaluate_grid([audio, clip], [voc_ref, clip_ref], settings, model, offset_ratio=0.5)
    np.testing.assert_array_equal(counts2, _oracle_grid(res, [o["note"].shape[0] for o in outs], [voc_ref, clip_ref],
                                                        offset_ratio=0.5))
