"""GPU: mir_eval's note matching pair for pair on the device (the match kernels of csrc/score.cu, the bp_match_* half of
csrc/api.cu) and its Python entry points (Model.match_grid, Model.match_notes, inference.evaluate_velocity_grid).

Every matching must equal oracle/note_matching_ref.py (mir_eval 0.7's match_notes and _bipartite_match restated in
plain Python) applied to the notes of the same decode, for both passes; the scores built from them must equal the
restatement's."""
import ctypes as C

import numpy as np
import pytest

from oracle import note_matching_ref as nm
from tests import postsets
from tests.test_gpu_decode_edges import _fixture_file, _kw, _set
from tests.test_gpu_decode_grid import _model_grid
from tests.test_gpu_score import _annotated_clips, _boundary_refs, _chain, _est_of, _hz, _random_items

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def edges(golden_dir):
    return dict(np.load(golden_dir / "decode_edges.npz"))


def _oracle(ref_iv, ref_l2, est_iv, est_l2, **tol):
    """(2, n_ref) int32: row 0 without, row 1 with the offset test."""
    return np.stack([nm.match_array(nm.match_notes(np.asarray(ref_iv, np.float64).reshape(-1, 2), ref_l2,
                                                   np.asarray(est_iv, np.float64).reshape(-1, 2), est_l2, w, **tol),
                                    len(ref_l2)) for w in (False, True)])


def _assert_notes_equal(got, exp, msg):
    for k in ("start", "end", "pitch", "amp"):
        np.testing.assert_array_equal(got[k], exp[k], err_msg=f"{msg}: {k}")
    assert not got["bends"].size and not got["bend_off"].any(), msg


def _check_grid(model, notes, onsets, settings, refs, res, match, **tol):
    """res / match of Model.match_grid against decode_grid's notes, the oracle and score_grid's counts."""
    lens = [a.shape[0] for a in notes]
    exp_res = model.decode_grid(notes, onsets, None, [{**s, "include_pitch_bends": False} for s in settings])
    counts = model.score_grid(notes, onsets, settings, refs, **tol)
    for k in range(len(settings)):
        for i in range(len(notes)):
            _assert_notes_equal(res[k][i], exp_res[k][i], f"setting {k} file {i}")
            est_iv, est_l2 = _est_of(res[k][i], lens[i])
            exp = _oracle(refs[i][0], np.log2(refs[i][1]), est_iv, est_l2, **tol)
            np.testing.assert_array_equal(match[k][i], exp, err_msg=f"setting {k} file {i}")
            assert [(match[k][i][p] >= 0).sum() for p in (0, 1)] == counts[k, i, 2:].tolist()
    return counts


# ------------------------------------------------------------------------------------------------ model output, grid
def test_grid_matchings_equal_the_oracle_on_model_output(model, golden_dir):
    """The annotated clips of test_gpu_score (vocadito, random_notes_clip files, chords, tones, an empty clip, a clip
    without annotation) under >= 48 settings: every (setting, file, pass) equals the oracle on decode_grid's notes, the
    counts equal score_grid's, the notes equal decode_grid's; _device on a caller stream equals _host; the velocity
    scores equal the restatement's with seeded velocities."""
    import torch

    from basic_pitch_b200.evaluate import EST_LOG2_HZ, matching_scores, note_velocities

    clips, refs = _annotated_clips(golden_dir)
    outs = model.run_inference_arrays(clips)
    notes, onsets = [o["note"] for o in outs], [o["onset"] for o in outs]
    lens = [a.shape[0] for a in notes]
    settings = _model_grid()
    assert len(settings) >= 32
    res, match = model.match_grid(notes, onsets, settings, refs)
    counts = _check_grid(model, notes, onsets, settings, refs, res, match)
    assert counts[..., 2].sum() > 300 and (counts[..., 3] < counts[..., 2]).any()

    # velocities: seeded per reference note; estimates get the MIDI writer's
    rng = np.random.default_rng(17)
    n_diff = 0
    for i in range(len(clips)):
        rv = rng.integers(20, 128, len(refs[i][1]))
        for k in range(0, len(settings), 3):
            est_iv, _ = _est_of(res[k][i], lens[i])
            ev = note_velocities(res[k][i]["amp"])
            got = matching_scores(refs[i][0], rv, est_iv, ev, match[k][i])
            for suffix, p in (("_no_offset", 0), ("", 1)):
                pairs = [(r, int(match[k][i][p][r])) for r in np.flatnonzero(match[k][i][p] >= 0)]
                exp = nm.velocity_scores(refs[i][0], rv, est_iv, ev, pairs)
                assert tuple(got[f + suffix] for f in ("velocity_precision", "velocity_recall", "velocity_f_measure",
                                                       "velocity_average_overlap_ratio")) == exp
                if len(rv) and len(ev):
                    assert got["average_overlap_ratio" + suffix] == nm.average_overlap_ratio(refs[i][0], est_iv, pairs)
                n_diff += got["velocity_precision" + suffix] < (match[k][i][p] >= 0).sum() / max(len(ev), 1)
    assert n_diff > 0  # the velocity test drops pairs somewhere

    foff = np.cumsum([0] + lens).astype(np.int64)
    dev = f"cuda:{model.device}"
    d = [torch.from_numpy(np.ascontiguousarray(np.concatenate(x))).to(dev) for x in (notes, onsets)]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    sub = settings[:12]
    ps = model._grid_params(sub)
    ns, keep = model._note_set(refs, "references")
    sp = model._score_params({})
    n_refs = int(keep[0][-1])
    h = np.full((len(sub), 2, n_refs), -7, np.int32)
    nt, arrs = model._alloc_notes(len(sub) * len(clips), 400000, 16)
    with torch.cuda.stream(stream):
        model._lib.bp_match_grid_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), foff.ctypes.data, len(clips), ps,
                                        len(sub), C.byref(ns), C.byref(sp), EST_LOG2_HZ.ctypes.data, C.byref(nt),
                                        h.ctypes.data, stream.cuda_stream)
    flat = model._split_notes(arrs, len(sub) * len(clips))
    for k in range(len(sub)):
        for i in range(len(clips)):
            _assert_notes_equal(flat[k * len(clips) + i], res[k][i], f"device: setting {k} file {i}")
            np.testing.assert_array_equal(h[k, :, keep[0][i] : keep[0][i + 1]], match[k][i])


# ------------------------------------------------------------------------------------------------ adversarial notes
@pytest.mark.parametrize("name", postsets.NAMES)
def test_adversarial_sets_through_the_grid(model, edges, name):
    """The pinned posteriorgram sets of tests/postsets.py under their grids, with references on either side of every
    predicate boundary around the decoded notes, in shuffled order."""
    files, grid = _set(edges, name)
    notes, onsets = [f[0] for f in files], [f[1] for f in files]
    lens = [a.shape[0] for a in notes]
    rng = np.random.default_rng(43)
    refs = []
    for i in range(len(files)):
        est_iv, est_l2 = _est_of(_fixture_file(edges, f"{name}/p0", i), lens[i])
        iv, l2 = _boundary_refs(est_iv, est_l2, rng)
        if len(l2) > 1 and rng.random() < 0.5:  # duplicate some references
            dup = rng.integers(0, len(l2), len(l2) // 3 + 1)
            iv, l2 = np.concatenate([iv, iv[dup]]), np.concatenate([l2, l2[dup]])
        perm = rng.permutation(len(l2))
        refs.append((iv[perm], 2.0 ** l2[perm]))
    settings = [_kw(p) for p in grid]
    res, match = model.match_grid(notes, onsets, settings, refs)
    _check_grid(model, notes, onsets, settings, refs, res, match)


def _log2_items(items):
    """[(ref_iv, ref_l2, est_iv, est_l2)] -> (estimates, references) as Model.match_notes takes them (Hz)."""
    return ([(np.asarray(c, np.float64).reshape(-1, 2), 2.0 ** np.asarray(d, np.float64)) for _, _, c, d in items],
            [(np.asarray(a, np.float64).reshape(-1, 2), 2.0 ** np.asarray(b, np.float64)) for a, b, _, _ in items])


def _check_items(model, items, **tol):
    est, refs = _log2_items(items)
    got = model.match_notes(est, refs, **tol)
    for q in range(len(items)):
        exp = _oracle(refs[q][0], np.log2(refs[q][1]), est[q][0], np.log2(est[q][1]), **tol)
        np.testing.assert_array_equal(got[q], exp, err_msg=f"item {q}")
    return got


def _spaced(n, step, rng, shuffle):
    """n references and n estimates at onsets `step` apart (49.99 ms: each hits its neighbours, after np.around, within
    the default 50 ms), the estimates shifted by a quarter step: long alternating paths and several phases."""
    on = 1.0 + step * np.arange(n)
    ref_iv = np.stack([on, on + 0.5], 1)
    est_iv = ref_iv + step / 4
    l2 = np.full(n, 8.0)
    pr = rng.permutation(n) if shuffle else np.arange(n)
    pe = rng.permutation(n) if shuffle else np.arange(n)[::-1].copy()
    return ref_iv[pr], l2, est_iv[pe], l2


def test_match_notes_on_adversarial_items(model):
    """Chains forcing augmenting paths of up to 129 edges, notes 49.99 ms apart, duplicated references and estimates,
    ties at exactly 50 cents, empty sides; every item equals the oracle under three tolerance sets."""
    rng = np.random.default_rng(12)
    items = []
    for L in list(range(1, 9)) + [16, 31, 64]:
        items.append(_chain(L, rng, False))
        items.append(_chain(L, rng, True))
    for n in (2, 3, 7, 40, 150):
        items += [_spaced(n, 0.04999, rng, False), _spaced(n, 0.04999, rng, True)]
    one = np.array([[1.0, 2.0]])
    items.append((np.repeat(one, 64, 0), np.full(64, 7.0), np.repeat(one, 64, 0), np.full(64, 7.0)))
    items.append((np.repeat(one, 3, 0), np.full(3, 6.0), np.repeat(one, 5, 0), np.full(5, 6.0)))
    items.append((np.repeat(one, 5, 0), np.full(5, 6.0), np.repeat(one, 3, 0), np.full(3, 6.0)))
    items += [(np.zeros((0, 2)), np.zeros(0), one, [6.0]), (one, [6.0], np.zeros((0, 2)), np.zeros(0)),
              (np.zeros((0, 2)), np.zeros(0), np.zeros((0, 2)), np.zeros(0))]
    for it in _random_items(rng, 30, 40, grid=0.02):  # coarse grid: many duplicates and ties
        items.append(it)
    for tol in (dict(), dict(onset_tolerance=0.02), dict(onset_tolerance=0.1, pitch_tolerance=150.0, offset_ratio=0.0)):
        got = _check_items(model, items, **tol)
    assert all((g[0] >= 0).all() for g in got[: 2 * 11])  # the chains match completely


@pytest.mark.parametrize("n_items", [63, 64, 65, 127, 128, 129])
def test_pair_counts_around_the_cta_width(model, n_items):
    """Two threads per pair and 128 per CTA: item counts around 64 and 128 pairs."""
    rng = np.random.default_rng(n_items)
    _check_items(model, _random_items(rng, n_items, 30))


def test_a_pair_too_large_for_the_workspace_runs_alone(model):
    """34 million references (64 bytes each: 2.18 GB of workspace) against one estimate, between two small items: the
    match launch splits in three.  The estimate hits the first reference only."""
    rng = np.random.default_rng(4)
    small = _random_items(rng, 2, 30)
    n = 34_000_000
    on = 0.1 * np.arange(n)
    big = (np.stack([on, on + 0.5], 1), np.full(n, 8.0), np.array([[0.0, 0.5]]), np.array([8.0]))
    del on
    items = [small[0], big, small[1]]
    est, refs = _log2_items(items)
    del big, items
    before = model.launch_count
    got = model.match_notes(est, refs)
    assert model.launch_count - before == 1 + 3
    assert got[1].shape == (2, n) and (got[1][:, 0] == 0).all() and (got[1][:, 1:] == -1).all()
    for q in (0, 2):
        np.testing.assert_array_equal(got[q], _oracle(refs[q][0], np.log2(refs[q][1]), est[q][0], np.log2(est[q][1])))
    before = model.launch_count
    model.match_notes([est[0], est[2]], [refs[0], refs[2]])
    assert model.launch_count - before == 2


# ------------------------------------------------------------------------------------------------ chunks, launches, errors
def test_chunked_grid_equals_per_setting_calls(model, edges):
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
    first = model.decode_grid(notes, onsets, None, [{**distinct[0], "include_pitch_bends": False}])[0]
    rng = np.random.default_rng(3)
    refs = []
    for i, r in enumerate(first):
        iv, l2 = _est_of(r, lens[i])
        iv = iv + np.round(rng.uniform(-0.06, 0.06, (len(iv), 1)), 3)
        iv[:, 0] = np.maximum(iv[:, 0], 0.0)
        perm = rng.permutation(len(l2))
        refs.append((iv[perm], 2.0 ** l2[perm]))
    single = [model.match_grid(notes, onsets, [s], refs) for s in distinct]
    res, match = model.match_grid(notes, onsets, settings, refs)
    for k in range(len(settings)):
        sres, smatch = single[k % len(distinct)]
        for i in range(len(files)):
            _assert_notes_equal(res[k][i], sres[0][i], f"setting {k} file {i}")
            np.testing.assert_array_equal(match[k][i], smatch[0][i], err_msg=f"setting {k} file {i}")
    est_iv, est_l2 = _est_of(single[0][0][0][0], lens[0])
    np.testing.assert_array_equal(single[0][1][0][0], _oracle(refs[0][0], np.log2(refs[0][1]), est_iv, est_l2))

    small, _ = _set(edges, "nan_file")
    sn, so = [f[0] for f in small], [f[1] for f in small]
    srefs = [(np.array([[0.1, 0.5], [0.3, 0.9]]), _hz([60, 64]))] * len(small)
    for p in (1, 64):
        grid = [distinct[k % len(distinct)] for k in range(p)]
        n_notes = sum(len(r["start"]) for per in model.decode_grid(sn, so, None, [{**s, "include_pitch_bends": False}
                                                                                  for s in grid]) for r in per)
        before = model.launch_count
        model.match_grid(sn, so, grid, srefs)
        # prep, candidates, loops; compaction, amplitudes; count, match
        assert model.launch_count - before == (7 if n_notes else 3), (p, n_notes)
        assert n_notes > 0
    before = model.launch_count
    model.match_grid(sn, so, [dict()], [(np.zeros((0, 2)), np.zeros(0))] * len(small))
    assert model.launch_count - before == 5  # no references: the notes only
    before = model.launch_count
    model.match_notes([srefs[0]] * 3, srefs[:3])
    assert model.launch_count - before == 2


def test_invalid_inputs_are_rejected_by_index_without_a_launch(model, edges):
    from basic_pitch_b200 import _lib, inference

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

    cases = [(bad(1, 2, 0, np.nan), "file 1 note 2: non-finite time"), (bad(2, 0, 0, -0.5), "file 2 note 0: onset < 0"),
             (bad(1, 1, 1, 0.2), "file 1 note 1: offset <= onset"), (bad(0, 2, None, None, 0.0), "file 0 note 2: non-finite log2_hz")]
    for refs, msg in cases:
        before = model.launch_count
        with pytest.raises(_lib.BpError) as e:
            model.match_grid(notes, onsets, [dict(), dict(onset_thresh=0.3)], refs)
        assert e.value.code == _lib.BP_E_INVALID and msg in str(e.value) and "bp_match_grid_host" in str(e.value)
        with pytest.raises(_lib.BpError) as e:
            model.match_notes(good, refs)
        assert e.value.code == _lib.BP_E_INVALID and msg.replace("file", "item") in str(e.value)
        with pytest.raises(_lib.BpError) as e:
            model.match_notes(refs, good)
        assert "estimates item" in str(e.value)
        assert model.launch_count == before
    for tol in (dict(onset_tolerance=-0.01), dict(pitch_tolerance=np.inf), dict(offset_ratio=np.nan)):
        before = model.launch_count
        with pytest.raises(_lib.BpError) as e:
            model.match_grid(notes, onsets, [dict()], good, **tol)
        assert e.value.code == _lib.BP_E_INVALID and next(iter(tol)) in str(e.value)
        with pytest.raises(_lib.BpError):
            model.match_notes(good, good, **tol)
        assert model.launch_count == before
    before = model.launch_count
    with pytest.raises(_lib.BpError) as e:
        model.match_grid(notes, onsets, [dict(), dict(energy_tol=0)], good)
    assert "decode params[1]" in str(e.value)
    # velocities: checked before the model runs
    clip = np.zeros(22050, np.float32)
    vref = [(good[0][0], good[0][1], np.array([10.0, 20.0, 30.0])), (good[0][0], good[0][1], np.array([10.0, -1.0, 3.0]))]
    with pytest.raises(ValueError, match=r"references\[1\] note 1"):
        inference.evaluate_velocity_grid([clip, clip], vref, [dict()], model)
    vref[1] = (good[0][0], good[0][1], np.array([10.0, 2.0, np.inf]))
    with pytest.raises(ValueError, match=r"references\[1\] note 2"):
        inference.evaluate_velocity_grid([clip, clip], vref, [dict()], model)
    res, match = model.match_grid(notes, onsets, [], good)
    assert res == [] and match == []
    assert model.match_notes([], []) == []
    assert model.launch_count == before


# ------------------------------------------------------------------------------------------------ evaluate_velocity_grid
def test_evaluate_velocity_grid_on_arrays_and_a_wav_path(model, golden_dir, tmp_path):
    from scipy.io import wavfile

    from basic_pitch_b200 import inference, synth
    from basic_pitch_b200.audio_io import load_audio_device
    from basic_pitch_b200.evaluate import MATCH_FIELDS, matching_scores, note_scores, note_velocities
    from basic_pitch_b200.note_creation import grid_setting

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    wav = tmp_path / "vocadito_10.wav"
    wavfile.write(wav, int(zp["sample_rate"]), zp["pcm"])
    z = np.load(golden_dir / "vocadito10.npz")
    rng = np.random.default_rng(23)
    voc_iv = np.stack([z["gold_events/start"], z["gold_events/end"]], 1)
    clip = synth.random_notes_clip(6.0, 77)
    clip_iv, clip_hz = synth.random_notes_events(6.0, 77)
    refs = [(voc_iv, _hz(z["gold_events/pitch"]), rng.integers(30, 120, len(voc_iv))),
            (clip_iv, clip_hz, rng.integers(30, 120, len(clip_hz)))]
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2, minimum_note_length=58.0),
                dict(minimum_frequency=150.0, maximum_frequency=700.0), dict(melodia_trick=False)]
    counts, scores = inference.evaluate_velocity_grid([wav, clip], refs, settings, model)
    counts_g, _ = inference.evaluate_grid([wav, clip], [r[:2] for r in refs], settings, model)
    np.testing.assert_array_equal(counts, counts_g)
    assert counts[0, 0, 3] > 10
    audio, _ = load_audio_device(wav, model)
    outs = model.run_inference_arrays([audio, clip])
    decode = [{**grid_setting(s, predict_names=True)[0], "include_pitch_bends": False} for s in settings]
    res = model.decode_grid([o["note"] for o in outs], [o["onset"] for o in outs], None, decode)
    ref_scores = note_scores(counts)
    for key, v in ref_scores.items():
        if key != "mean":
            np.testing.assert_array_equal(scores[key], v)
    for k in range(len(settings)):
        for i, o in enumerate(outs):
            est_iv, est_l2 = _est_of(res[k][i], o["note"].shape[0])
            m = _oracle(refs[i][0], np.log2(refs[i][1]), est_iv, est_l2)
            exp = matching_scores(refs[i][0], refs[i][2], est_iv, note_velocities(res[k][i]["amp"]), m)
            for key in MATCH_FIELDS:
                for suffix in ("", "_no_offset"):
                    assert scores[key + suffix][k, i] == exp[key + suffix], (key + suffix, k, i)
    for key in MATCH_FIELDS:
        np.testing.assert_array_equal(scores["mean"][key], scores[key].mean(axis=-1))
    assert (scores["velocity_f_measure"] > 0).any()
    counts2, scores2 = inference.evaluate_velocity_grid([audio, clip], refs, settings[:2], model, velocity_tolerance=0.3,
                                                        offset_ratio=0.5)
    np.testing.assert_array_equal(counts2, inference.evaluate_grid([audio, clip], [r[:2] for r in refs], settings[:2], model,
                                                                   offset_ratio=0.5)[0])
    assert (scores2["velocity_recall"] >= scores2["recall"] * 0).all() and scores2["velocity_f_measure"].shape == (2, 2)
