"""GPU: the grid decode (bp_decode_grid_*: csrc/decode.cu kernels with kGrid, the grid half of csrc/api.cu) and its Python
entry points (Model.decode_grid, note_creation.model_output_to_notes_grid, inference.predict_grid).

Every cell (setting, file) of a grid must equal the single-setting decode bit for bit: start, end, pitch and order of
the notes, the float32 bytes of the amplitudes, the pitch bends and their offsets, and the per-(setting, file) note
offsets."""
import ctypes as C

import numpy as np
import pytest

from tests import postsets
from tests.golden_util import edges_case
from tests.test_gpu_decode_edges import _fixture_file, _kw, _set, assert_file_equal

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def edges(golden_dir):
    return dict(np.load(golden_dir / "decode_edges.npz"))


def _files(files):
    return [f[0] for f in files], [f[1] for f in files], [f[2] for f in files]


def _check_offsets(arrs, cells, n_files, ctx):
    """note_off of a concatenated grid result against the note counts of every (setting, file)."""
    counts = np.diff(arrs["note_off"][: len(cells) * n_files + 1])
    exp = [len(c["start"]) for c in cells]
    np.testing.assert_array_equal(counts, exp, err_msg=f"{ctx}: per-(setting, file) note offsets")


@pytest.mark.parametrize("name", postsets.NAMES)
def test_golden_grid_in_one_call(model, edges, name):
    """The set's whole parameter grid over all of its files in one bp_decode_grid_host call: every (setting, file) is the
    reference's (decode_edges.npz).  The grids mix pitch ranges (lo > hi included), infer_onsets and melodia_trick,
    onset_thresh <= 0, energy_tol = INT_MAX and the NaN file: several prep and candidate groups per call."""
    files, grid = _set(edges, name)
    notes, onsets, contours = _files(files)
    n = len(files)
    arrs = model.decode_grid(notes, onsets, contours, [_kw(p) for p in grid], split_notes=False)
    res = model._split_notes(arrs, len(grid) * n)
    exp = [_fixture_file(edges, f"{name}/p{j}", i) for j in range(len(grid)) for i in range(n)]
    _check_offsets(arrs, exp, n, name)
    for q, (r, e) in enumerate(zip(res, exp)):
        assert_file_equal(r, e, f"{name}/p{q // n} file {q % n} in the grid")
    np.testing.assert_array_equal(arrs["note_off"][: len(exp) + 1],
                                  np.concatenate([[0], np.cumsum([len(e["start"]) for e in exp])]))


@pytest.mark.parametrize("name", postsets.NAMES)
def test_grid_results_do_not_depend_on_neighbours(model, edges, name):
    """The same grid three times over, shuffled: each cell is its setting's result, whatever settings share its groups
    or sit beside it."""
    files, grid = _set(edges, name)
    notes, onsets, contours = _files(files)
    order = np.random.default_rng(17).permutation(np.tile(np.arange(len(grid)), 3))
    res = model.decode_grid(notes, onsets, contours, [_kw(grid[j]) for j in order])
    assert len(res) == len(order)
    for k, (j, per_file) in enumerate(zip(order, res)):
        for i, r in enumerate(per_file):
            assert_file_equal(r, _fixture_file(edges, f"{name}/p{j}", i), f"{name}: cell {k} (p{j}) file {i}")


def _model_grid():
    """>= 48 settings: onset x frame x min length x two pitch ranges x (infer, melodia) toggles, bends on and off."""
    out = []
    for onset in (0.3, 0.6):
        for frame in (0.2, 0.35):
            for mnl in (5, 11):
                for lo, hi in ((0, 88), (15, 60)):
                    for infer, melodia in ((True, True), (False, True), (True, False)):
                        out.append(dict(onset_thresh=onset, frame_thresh=frame, min_note_len=mnl, infer_onsets=infer,
                                        melodia_trick=melodia, min_pitch_idx=lo, max_pitch_idx=hi,
                                        include_pitch_bends=len(out) % 5 != 3))
    return out


def _single_device(model, d, foff, n, setting, stream):
    """bp_decode_device with one setting (the reference for a cell), on `stream`."""
    import torch

    s = {**model._DECODE_DEFAULTS, **setting}
    p = model._params(**s)
    nt, arrs = model._alloc_notes(n, 200000, 4000000)
    with torch.cuda.stream(stream):
        model._lib.bp_decode_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), foff.ctypes.data, n,
                                    C.byref(p), C.byref(nt), stream.cuda_stream)
    return model._split_notes(arrs, n)


def _posteriorgrams(model, golden_dir):
    from basic_pitch_b200 import synth

    clips = [np.load(golden_dir / "vocadito10.npz")["audio22k"].astype(np.float32)]
    clips += [synth.random_notes_clip(4.0 + 1.3 * i, seed=800 + i) for i in range(3)]
    clips += [synth.dense_chords_clip(3.0, seed=810), np.zeros(0, np.float32), synth.tones_clip(2.0, seed=811)]
    return model.run_inference_arrays(clips)


def test_grid_equals_single_decode_on_model_output(model, golden_dir):
    """Posteriorgrams of the model (vocadito and synthetic clips, one zero-length file) under 48 settings: the grid on a
    caller stream (bp_decode_grid_device) and from host memory (bp_decode_grid_host) equal bp_decode_device per setting."""
    import torch

    from basic_pitch_b200 import _lib

    outs = _posteriorgrams(model, golden_dir)
    n = len(outs)
    settings = _model_grid()
    assert len(settings) >= 48
    foff = np.cumsum([0] + [o["note"].shape[0] for o in outs]).astype(np.int64)
    dev = f"cuda:{model.device}"
    d = [torch.from_numpy(np.ascontiguousarray(np.concatenate([o[k] for o in outs]))).to(dev)
         for k in ("note", "onset", "contour")]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    exp = [_single_device(model, d, foff, n, s, stream) for s in settings]
    assert sum(len(r["start"]) for per in exp for r in per) > 500

    host = model.decode_grid([o["note"] for o in outs], [o["onset"] for o in outs], [o["contour"] for o in outs], settings)
    ps = (_lib.DecodeParams * len(settings))(*[model._params(**{**model._DECODE_DEFAULTS, **s}) for s in settings])
    nt, arrs = model._alloc_notes(n * len(settings), 400000, 8000000)
    with torch.cuda.stream(stream):
        model._lib.bp_decode_grid_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), foff.ctypes.data,
                                         n, ps, len(settings), C.byref(nt), stream.cuda_stream)
    flat = model._split_notes(arrs, n * len(settings))
    for k, s in enumerate(settings):
        for i in range(n):
            assert_file_equal(host[k][i], exp[k][i], f"bp_decode_grid_host setting {k} {s} file {i}")
            assert_file_equal(flat[k * n + i], exp[k][i], f"bp_decode_grid_device setting {k} {s} file {i}")
        if not s["include_pitch_bends"]:
            assert all(len(r["bends"]) == 0 and not r["bend_off"].any() for r in host[k])


def _need(lib):
    a, b = C.c_int64(0), C.c_int64(0)
    lib.bp_last_required(C.byref(a), C.byref(b))
    return a.value, b.value


def test_chunked_grid_and_launch_counts(model, edges):
    """A batch long enough that the grid runs in several chunks equals per-setting decodes, and its capacity errors
    report the need of the whole grid; within one chunk the launches of a call do not depend on the number of settings."""
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    base = []
    for name in ("ties", "long_notes", "nan_file", "runs", "crowded"):
        base += _set(edges, name)[0]
    files = []
    while sum(f[0].shape[0] for f in files) < 120_000:
        files += base
    notes, onsets, contours = _files(files)
    n = len(files)
    total = sum(a.shape[0] for a in notes)
    chunk = int(lib.bp_decode_grid_chunk_params(total, n))
    distinct = [dict(onset_thresh=0.5, frame_thresh=0.3, energy_tol=11),
                dict(onset_thresh=0.5, frame_thresh=0.05, min_note_len=0, energy_tol=1, infer_onsets=False),
                dict(onset_thresh=0.95, frame_thresh=0.3, min_note_len=1, energy_tol=64, include_pitch_bends=False),
                dict(onset_thresh=0.0, frame_thresh=0.3, min_note_len=11, energy_tol=33, melodia_trick=False),
                dict(onset_thresh=0.5, frame_thresh=0.3, min_pitch_idx=20, max_pitch_idx=70)]
    settings = [distinct[k % len(distinct)] for k in range(chunk + 3)]
    assert -(-len(settings) // chunk) >= 2, (total, chunk)
    single = [model.decode_arrays(notes, onsets, contours, **s) for s in distinct]
    before = model.launch_count
    res = model.decode_grid(notes, onsets, contours, settings, split_notes=False)
    print(f"{n} files, {total} frames: {chunk} settings per chunk, {len(settings)} settings, "
          f"{model.launch_count - before} launches, {int(res['note_off'][-1])} notes")
    cells = model._split_notes(res, n * len(settings))
    for k in range(len(settings)):
        for i in (0, 1, 2, 3, n // 2, n - 1):
            assert_file_equal(cells[k * n + i], single[k % len(distinct)][i], f"chunked grid setting {k} file {i}")
        got = [len(cells[k * n + i]["start"]) for i in range(n)]
        assert got == [len(r["start"]) for r in single[k % len(distinct)]], k

    # capacities one short of the whole grid's need, across chunks: BP_E_CAPACITY with the exact need
    need_n = int(res["note_off"][n * len(settings)])
    need_b = int(res["bend_off"][need_n])
    foff, n_all, o_all, c_all = model._cat_posteriorgrams(notes, onsets, contours, True)
    ps = (_lib.DecodeParams * len(settings))(*[model._params(**{**model._DECODE_DEFAULTS, **s}) for s in settings])
    for cap_n, cap_b, which in ((need_n - 1, need_b, 0), (need_n, need_b - 1, 1)):
        nt, _ = model._alloc_notes(n * len(settings), cap_n, cap_b)
        with pytest.raises(_lib.BpError) as e:
            lib.bp_decode_grid_host(model.handle, n_all.ctypes.data, o_all.ctypes.data, c_all.ctypes.data,
                                    foff.ctypes.data, n, ps, len(settings), C.byref(nt))
        assert e.value.code == _lib.BP_E_CAPACITY
        assert _need(lib)[which] == (need_n, need_b)[which], (which, _need(lib), need_n, need_b)

    # launches within one chunk: the same for 1 and 64 settings (prep, candidates, loops, compaction, finish)
    small, _ = _set(edges, "nan_file")
    sn, so, sc = _files(small)
    deltas = []
    for p in (1, 64):
        before = model.launch_count
        r = model.decode_grid(sn, so, sc, [distinct[k % len(distinct)] for k in range(p)])
        deltas.append(model.launch_count - before)
        assert sum(len(c["start"]) for c in r[0]) > 0
    before = model.launch_count
    model.decode_arrays(sn, so, sc)
    assert deltas == [model.launch_count - before] * 2 == [5, 5], deltas


def test_errors_and_empty_calls(model, edges):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    files, _ = _set(edges, "nan_file")
    notes, onsets, contours = _files(files)
    good = [dict(onset_thresh=0.5), dict(frame_thresh=0.1), dict(min_note_len=3)] * 4
    bad = [(7, dict(onset_thresh=float("nan"))), (3, dict(frame_thresh=float("nan"))),
           (5, dict(frame_thresh=-0.1, melodia_trick=True)), (0, dict(energy_tol=0)), (11, dict(min_note_len=-1))]
    for k, b in bad:
        settings = list(good)
        settings[k] = b
        before = model.launch_count
        with pytest.raises(_lib.BpError) as e:
            model.decode_grid(notes, onsets, contours, settings)
        assert e.value.code == _lib.BP_E_INVALID
        assert f"decode params[{k}]:" in str(e.value), str(e.value)
        assert model.launch_count == before, b
    # frame_thresh < 0 without melodia is a valid setting (the reference terminates)
    model.decode_grid(notes, onsets, contours, [dict(frame_thresh=-0.1, melodia_trick=False)])

    # n_params = 0, n_files = 0: nothing to do, no launch
    foff, n_all, o_all, c_all = model._cat_posteriorgrams(notes, onsets, contours, True)
    ps = (_lib.DecodeParams * 2)(*[model._params(**model._DECODE_DEFAULTS)] * 2)
    for n_files, n_params in ((len(files), 0), (0, 2)):
        nt, arrs = model._alloc_notes(1, 8, 8)
        arrs["note_off"][0] = 99
        before = model.launch_count
        lib.bp_decode_grid_host(model.handle, n_all.ctypes.data, o_all.ctypes.data, c_all.ctypes.data, foff.ctypes.data,
                                n_files, ps, n_params, C.byref(nt))
        assert arrs["note_off"][0] == 0 and model.launch_count == before
    assert model.decode_grid(notes, onsets, contours, []) == []
    assert model.decode_grid([], [], [], [dict(), dict(onset_thresh=0.2)]) == [[], []]

    # zero-frame files only: as bp_decode_device (no notes, the loop kernel alone)
    z = [np.zeros((0, 88), np.float32)] * 3
    zc = [np.zeros((0, 264), np.float32)] * 3
    before = model.launch_count
    single = model.decode_arrays(z, z, zc)
    d_single = model.launch_count - before
    before = model.launch_count
    grid = model.decode_grid(z, z, zc, [dict(), dict(melodia_trick=False)])
    assert model.launch_count - before == d_single == 1
    for per in grid:
        for r, s in zip(per, single):
            assert_file_equal(r, s, "zero-frame file")


def test_model_output_to_notes_grid_equals_per_setting_calls(model, golden_dir):
    from basic_pitch_b200 import note_creation as nc

    z = np.load(golden_dir / "vocadito10.npz")
    out = {k: np.array(z[f"gold_{k}"], np.float32) for k in ("note", "onset", "contour")}
    keep = {k: v.copy() for k, v in out.items()}
    settings = [dict(onset_thresh=0.5, frame_thresh=0.3),
                dict(onset_thresh=0.3, frame_thresh=0.2, min_note_len=5, min_freq=200.0, max_freq=800.0),
                dict(onset_thresh=0.6, frame_thresh=0.3, infer_onsets=False, melodia_trick=False, multiple_pitch_bends=True),
                dict(onset_thresh=0.5, frame_thresh=0.25, include_pitch_bends=False, max_freq=500.0, midi_tempo=90),
                dict(onset_thresh=0.4, frame_thresh=0.3, min_freq=20000.0)]
    grid = nc.model_output_to_notes_grid(out, settings, model=model)
    for k, v in out.items():
        np.testing.assert_array_equal(v, keep[k], err_msg=f"{k}: the grid call modified its input")
    assert len(grid) == len(settings)
    for s, (midi, events) in zip(settings, grid):
        ref_midi, ref_events = nc.model_output_to_notes({k: v.copy() for k, v in keep.items()}, model=model, **s)
        assert events == ref_events, s
        for a, b in zip(midi.instruments, ref_midi.instruments):
            assert [(n.start, n.end, n.pitch, n.velocity) for n in a.notes] == [(n.start, n.end, n.pitch, n.velocity)
                                                                               for n in b.notes], s
            assert [(p.pitch, p.time) for p in a.pitch_bends] == [(p.pitch, p.time) for p in b.pitch_bends], s
        assert len(midi.instruments) == len(ref_midi.instruments), s
    assert len(grid[0][1]) > 10 and len(grid[4][1]) == 0


def test_predict_grid_runs_the_model_once(model, golden_dir, tmp_path):
    """predict_grid on the reference's vocadito_10.wav (its stored 44.1 kHz PCM) equals predict per setting, with one
    forward pass for the whole grid."""
    from scipy.io import wavfile

    from basic_pitch_b200 import inference

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    wav = tmp_path / "vocadito_10.wav"
    wavfile.write(wav, int(zp["sample_rate"]), zp["pcm"])
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2, minimum_note_length=58.0),
                dict(minimum_frequency=150.0, maximum_frequency=700.0, multiple_pitch_bends=True),
                dict(melodia_trick=False, midi_tempo=100), dict(onset_threshold=0.7, minimum_note_length=300.0)]
    inference.predict_grid(wav, settings[:1], model)  # warm-up
    before = model.launch_count
    inference.predict_grid(wav, settings[:1], model)
    one = model.launch_count - before
    before = model.launch_count
    out, grid = inference.predict_grid(wav, settings, model)
    many = model.launch_count - before
    assert many == one, (one, many)  # the ingest, forward pass and decode launches do not grow with the settings
    assert len(grid) == len(settings)
    for s, (midi, events) in zip(settings, grid):
        ref_out, ref_midi, ref_events = inference.predict(wav, model, **s)
        assert isinstance(events, inference.infer.NoteEventList)
        assert events == ref_events, s
        assert [(n.start, n.end, n.pitch, n.velocity) for i in midi.instruments for n in i.notes] == \
            [(n.start, n.end, n.pitch, n.velocity) for i in ref_midi.instruments for n in i.notes], s
        assert [(p.pitch, p.time) for i in midi.instruments for p in i.pitch_bends] == \
            [(p.pitch, p.time) for i in ref_midi.instruments for p in i.pitch_bends], s
        if "minimum_frequency" not in s:  # predict zeroes the out-of-range columns of its output; the grid does not
            for k in ("note", "onset", "contour"):
                np.testing.assert_array_equal(out[k], ref_out[k], err_msg=k)
    assert len(grid[0][1]) > 10
