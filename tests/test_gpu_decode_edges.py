"""GPU: the note decode (csrc/decode.cu, the decode half of csrc/api.cu) on the adversarial posteriorgram sets of
tests/postsets.py, bit for bit against the unmodified reference decode (tests/golden/decode_edges.npz) or, where the
input is not in the fixture, against oracle/decode_ref.py on the same input.

Bit for bit means: start, end and pitch of every note and the order of the list; the float32 bytes of the amplitude;
the ragged pitch bends and their offsets; the per-file note offsets."""
import ctypes as C

import numpy as np
import pytest

from tests import postsets
from tests.golden_util import edges_case

pytestmark = pytest.mark.gpu

KEYS = ("onset_thresh", "frame_thresh", "min_note_len", "energy_tol", "infer_onsets", "melodia_trick")


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


@pytest.fixture(scope="module")
def edges(golden_dir):
    return dict(np.load(golden_dir / "decode_edges.npz"))


def _set(z, name):
    """The files of a set, checked to be the inputs the fixture was made from, and its parameter grid."""
    files, grid = postsets.get(name)
    for i, f in enumerate(files):
        assert postsets.file_sha(f) == z[f"{name}/sha"][i].tobytes(), f"{name} file {i}: inputs differ from decode_edges.npz"
    return files, grid


def _kw(p):
    kw = {k: p[k] for k in KEYS}
    kw.update(min_pitch_idx=p["lo_col"], max_pitch_idx=p["hi_col"])
    return kw


def _fixture_file(z, key, i):
    """Expected arrays of file i under parameter set `key` ("<set>/p<j>"), in decode_arrays' layout."""
    c = edges_case(z, key)
    a, b = int(c["note_off"][i]), int(c["note_off"][i + 1])
    boff = c["bend_off"]
    return {
        "start": c["start"][a:b], "end": c["end"][a:b], "pitch": c["pitch"][a:b], "amp": c["amp"][a:b],
        "bend_off": boff[a : b + 1] - boff[a], "bends": c["bends"][boff[a] : boff[b]],
    }  # fmt: skip


def _oracle_file(note, onset, contour, p):
    from oracle import decode_ref

    if note.shape[0] == 0:
        wb = []
    else:
        with np.errstate(all="ignore"):
            wb, _ = decode_ref.model_output_to_note_events(
                {"note": np.array(note), "onset": np.array(onset), "contour": np.array(contour)}, p["onset_thresh"],
                p["frame_thresh"], p["infer_onsets"], p["min_note_len"], melodia_trick=p["melodia_trick"],
                energy_tol=p["energy_tol"], lo_col=p["lo_col"], hi_col=p["hi_col"])  # fmt: skip
    bends = [int(v) for e in wb for v in e[4]]
    return {
        "start": np.array([e[0] for e in wb], np.int32), "end": np.array([e[1] for e in wb], np.int32),
        "pitch": np.array([e[2] for e in wb], np.int32), "amp": np.array([e[3] for e in wb], np.float32),
        "bend_off": np.cumsum([0] + [len(e[4]) for e in wb]).astype(np.int32), "bends": np.array(bends, np.int32),
    }  # fmt: skip


def assert_file_equal(got, exp, ctx):
    assert len(got["start"]) == len(exp["start"]), f"{ctx}: {len(got['start'])} notes, expected {len(exp['start'])}"
    for k in ("start", "end", "pitch", "bend_off", "bends"):
        np.testing.assert_array_equal(np.asarray(got[k], np.int64), np.asarray(exp[k], np.int64), err_msg=f"{ctx}: {k}")
    np.testing.assert_array_equal(np.asarray(got["amp"], np.float32).view(np.uint32),
                                  np.asarray(exp["amp"], np.float32).view(np.uint32), err_msg=f"{ctx}: amplitude bytes")


@pytest.mark.parametrize("name", postsets.NAMES)
def test_decode_host_every_set(model, edges, name):
    """bp_decode_host (Model.decode_arrays) on the whole set in one batch and on every file alone, under the set's grid."""
    files, grid = _set(edges, name)
    notes, onsets, contours = ([f[k] for f in files] for k in range(3))
    for j, p in enumerate(grid):
        key = f"{name}/p{j}"
        res = model.decode_arrays(notes, onsets, contours, **_kw(p))
        for i, r in enumerate(res):
            exp = _fixture_file(edges, key, i)
            assert_file_equal(r, exp, f"{key} file {i} (T={files[i][0].shape[0]}) in the batch")
            if len(files) > 1:
                alone = model.decode_arrays([notes[i]], [onsets[i]], [contours[i]], **_kw(p))[0]
                assert_file_equal(alone, exp, f"{key} file {i} alone")
        print(f"{key}: {[len(r['start']) for r in res]} notes")


@pytest.mark.parametrize("name", postsets.NAMES)
def test_decode_device_on_a_side_stream(model, edges, name):
    """bp_decode_device from device tensors on a non-default stream: the bits of the fixture (and of the host call)."""
    import torch

    from basic_pitch_b200 import _lib

    files, grid = _set(edges, name)
    n = len(files)
    foff = np.cumsum([0] + [f[0].shape[0] for f in files]).astype(np.int64)
    dev = f"cuda:{model.device}"
    d = [torch.from_numpy(np.ascontiguousarray(np.concatenate([f[k] for f in files]))).to(dev) for k in range(3)]
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    for j, p in enumerate(grid):
        key = f"{name}/p{j}"
        case = edges_case(edges, key)
        need, need_b = int(case["note_off"][-1]), int(case["bend_off"][-1])
        nt, arrs = model._alloc_notes(n, need + 1, need_b + 1)
        kw = _kw(p)
        params = model._params(kw["onset_thresh"], kw["frame_thresh"], kw["min_note_len"], kw["energy_tol"],
                               kw["infer_onsets"], kw["melodia_trick"], True, kw["min_pitch_idx"], kw["max_pitch_idx"])
        with torch.cuda.stream(stream):
            _lib.load().bp_decode_device(model.handle, d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), foff.ctypes.data,
                                         n, C.byref(params), C.byref(nt), stream.cuda_stream)
        np.testing.assert_array_equal(arrs["note_off"], case["note_off"], err_msg=f"{key}: note_off")
        np.testing.assert_array_equal(arrs["bend_off"][: need + 1], case["bend_off"], err_msg=f"{key}: bend_off")
        for i, r in enumerate(model._split_notes(arrs, n)):
            assert_file_equal(r, _fixture_file(edges, key, i), f"{key} file {i} (bp_decode_device)")


def test_crowded_file_overflows_the_first_slot_allowance(model, edges):
    """The crowded file needs more note slots than the first attempt gives it (min(88 T, 8 T + 64)): the decode runs
    again at full size, reusing the energy / onset maxima / candidate buffers of the first attempt."""
    files, grid = _set(edges, "crowded")
    T = files[1][0].shape[0]
    overflowed = 0
    for j, p in enumerate(grid):
        res = model.decode_arrays([f[0] for f in files], [f[1] for f in files], [f[2] for f in files], **_kw(p))
        counts = [len(r["start"]) for r in res]
        print(f"crowded/p{j}: {counts} notes; first allowance of the crowded file {8 * T + 64}")
        for i, r in enumerate(res):
            assert_file_equal(r, _fixture_file(edges, f"crowded/p{j}", i), f"crowded/p{j} file {i}")
        overflowed += counts[1] > 8 * T + 64
    assert overflowed >= 2


def _need(lib):
    n, b = C.c_int64(0), C.c_int64(0)
    lib.bp_last_required(C.byref(n), C.byref(b))
    return n.value, b.value


def _capacity_checks(model, call, need_n, need_b, ref, ctx):
    """`call(notes)` at note_capacity == need and bend_capacity == need succeeds with `ref`'s arrays; one less of either
    fails with BP_E_CAPACITY and bp_last_required reports the need."""
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    for cap_n, cap_b in ((need_n, need_b + 7), (need_n + 3, need_b)):
        nt, arrs = model._alloc_notes(len(ref["note_off"]) - 1, cap_n, cap_b)
        call(nt)
        for k in ("note_off", "start", "end", "pitch", "bend_off", "bends"):
            m = len(ref[k])
            np.testing.assert_array_equal(arrs[k][:m], ref[k], err_msg=f"{ctx}: {k} at capacity ({cap_n}, {cap_b})")
        np.testing.assert_array_equal(arrs["amp"][: len(ref["amp"])].view(np.uint32), ref["amp"].view(np.uint32))
    for cap_n, cap_b, which in ((need_n - 1, need_b, 0), (need_n, need_b - 1, 1)):
        nt, _ = model._alloc_notes(len(ref["note_off"]) - 1, cap_n, cap_b)
        with pytest.raises(_lib.BpError) as e:
            call(nt)
        assert e.value.code == _lib.BP_E_CAPACITY, (ctx, cap_n, cap_b)
        assert _need(lib)[which] == (need_n, need_b)[which], (ctx, which, _need(lib))


def _concat(arrs, n_notes, n_bends):
    out = {k: arrs[k][:n_notes].copy() for k in ("start", "end", "pitch", "amp")}
    out["note_off"] = arrs["note_off"].copy()
    out["bend_off"] = arrs["bend_off"][: n_notes + 1].copy()
    out["bends"] = arrs["bends"][:n_bends].copy()
    return out


def test_note_and_bend_capacity_at_the_exact_need(model, edges):
    from basic_pitch_b200 import _lib, synth

    lib = _lib.load()
    # bp_decode_host on the crowded batch (the need includes the notes of the retried decode)
    files, grid = _set(edges, "crowded")
    n = len(files)
    cat = [np.ascontiguousarray(np.concatenate([f[k] for f in files])) for k in range(3)]
    foff = np.cumsum([0] + [f[0].shape[0] for f in files]).astype(np.int64)
    kw = _kw(grid[0])
    params = model._params(kw["onset_thresh"], kw["frame_thresh"], kw["min_note_len"], kw["energy_tol"], kw["infer_onsets"],
                           kw["melodia_trick"], True, kw["min_pitch_idx"], kw["max_pitch_idx"])

    def decode(nt):
        lib.bp_decode_host(model.handle, cat[0].ctypes.data, cat[1].ctypes.data, cat[2].ctypes.data, foff.ctypes.data, n,
                           C.byref(params), C.byref(nt))

    case = edges_case(edges, "crowded/p0")
    need_n, need_b = int(case["note_off"][-1]), int(case["bend_off"][-1])
    nt, arrs = model._alloc_notes(n, need_n + 10, need_b + 10)
    decode(nt)
    ref = _concat(arrs, need_n, need_b)
    np.testing.assert_array_equal(ref["note_off"], case["note_off"])
    _capacity_checks(model, decode, need_n, need_b, ref, "bp_decode_host")

    # bp_transcribe_host (host sub-batch path) on audio
    clips = [synth.random_notes_clip(3.0 + 0.7 * i, seed=300 + i) for i in range(5)] + [synth.dense_chords_clip(2.5, seed=9)]
    flat, offs = model._pack_audio(clips)
    n = len(clips)
    p = model._params(0.5, 0.3, 11, 11, True, True, True, 0, 88)
    foff = np.zeros(n + 1, np.int64)

    def transcribe(nt):
        lib.bp_transcribe_host(model.handle, flat.ctypes.data, offs.ctypes.data, n, C.byref(p), None, None, None,
                               foff.ctypes.data, C.byref(nt))

    nt, arrs = model._alloc_notes(n, 100000, 2000000)
    transcribe(nt)
    need_n = int(arrs["note_off"][n])
    need_b = int(arrs["bend_off"][need_n])
    assert need_n > 20
    _capacity_checks(model, transcribe, need_n, need_b, _concat(arrs, need_n, need_b), "bp_transcribe_host")


WHOLE_FILE_PARAMS = [
    dict(energy_tol=33, min_note_len=3),
    dict(melodia_trick=False, infer_onsets=False),
    dict(min_pitch_idx=10, max_pitch_idx=70, onset_thresh=0.3, frame_thresh=0.2),
]


@pytest.mark.parametrize("j", range(len(WHOLE_FILE_PARAMS)))
def test_whole_file_entry_points_under_non_default_params(model, j):
    """bp_transcribe_files_host (transcribe_arrays), bp_transcribe_host and bp_transcribe_device carry the decode
    parameters through every host sub-batch: each call's notes equal the oracle decode of the posteriorgrams that call
    returned, and the three calls agree."""
    import torch

    from basic_pitch_b200 import engine, synth

    lib = model._lib
    base = [synth.random_notes_clip(0.5 + 0.9 * i, seed=500 + i) for i in range(8)]
    base += [synth.dense_chords_clip(1.5 + i, seed=520 + i) for i in range(3)]
    keys = [i % len(base) for i in range(150)]
    keys.insert(77, None)
    clips = [np.zeros(0, np.float32) if k is None else base[k] for k in keys]
    n = len(clips)
    # more than two chunks of windows: at least three host sub-batches
    assert sum(int(lib.bp_num_windows(len(c))) for c in clips) > 2 * int(lib.bp_model_chunk_windows(model.handle))
    kw = dict(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=11, infer_onsets=True, melodia_trick=True,
              min_pitch_idx=0, max_pitch_idx=88)
    kw.update(WHOLE_FILE_PARAMS[j])
    outs, res, frames = model.transcribe_arrays(clips, **kw)
    oracle_p = {k: kw[k] for k in KEYS}
    oracle_p.update(lo_col=kw["min_pitch_idx"], hi_col=kw["max_pitch_idx"])
    seen = {}
    total = 0
    for i, (o, r) in enumerate(zip(outs, res)):
        h = hash((o["note"].tobytes(), o["onset"].tobytes(), o["contour"].tobytes()))
        if h not in seen:
            seen[h] = _oracle_file(o["note"], o["onset"], o["contour"], oracle_p)
        assert_file_equal(r, seen[h], f"transcribe_arrays file {i} {WHOLE_FILE_PARAMS[j]}")
        total += len(r["start"])
    assert total > 100 and len(res[77]["start"]) == 0

    p = model._params(kw["onset_thresh"], kw["frame_thresh"], kw["min_note_len"], kw["energy_tol"], kw["infer_onsets"],
                      kw["melodia_trick"], True, kw["min_pitch_idx"], kw["max_pitch_idx"])
    n_bends = sum(len(r["bends"]) for r in res)
    packed = engine.PackedAudio(clips, pinned=True)
    out_h = engine.NoteBuffers(n, total + 16, n_bends + 16)
    assert engine.transcribe_packed_host(model, packed, out_h, p) == total
    out_d = engine.NoteBuffers(n, total + 16, n_bends + 16)
    d_audio = packed.to_device(model.device)
    assert engine.transcribe_packed_device(model, d_audio, packed.offsets, out_d, p) == total
    torch.cuda.synchronize(model.device)
    for name, out in (("bp_transcribe_host", out_h), ("bp_transcribe_device", out_d)):
        np.testing.assert_array_equal(out.a["frame_off"][: n + 1], np.cumsum([0] + frames), err_msg=name)
        for i, r in enumerate(engine.split_results(out)):
            assert_file_equal(r, res[i], f"{name} file {i} {WHOLE_FILE_PARAMS[j]}")


def test_infer_onsets_entry_point_on_every_length_and_nan_file(model, edges):
    """bp_infer_onsets_host, one file at a time: every length of `lengths`, and the files of `nan_file` (the time-constant
    one is all NaN, the all-zero-onset one is 0 wherever the frames do not rise), against decode_ref.infer_onsets."""
    from oracle import decode_ref

    for name in ("lengths", "nan_file"):
        files, _ = _set(edges, name)
        for i, (note, onset, _contour) in enumerate(files):
            got = model.infer_onsets_array(onset, note)
            if note.shape[0] == 0:
                assert got.shape == (0, 88)
                continue
            with np.errstate(all="ignore"):
                exp = decode_ref.infer_onsets(onset, note)
            assert got.dtype == np.float64 and got.shape == exp.shape
            np.testing.assert_array_equal(np.isnan(got), np.isnan(exp), err_msg=f"{name} file {i}: NaN positions")
            np.testing.assert_array_equal(got, exp, err_msg=f"{name} file {i} (T={note.shape[0]})")
    files, _ = _set(edges, "nan_file")
    assert np.isnan(model.infer_onsets_array(files[1][1], files[1][0])).all()


def test_pitch_bends_entry_point_at_the_clipped_window_edges(model, edges):
    """bp_pitch_bends_host on the notes of pitch_edges (pitches 21 .. 108, tied weighted products, contours < 0 and > 1)
    against the reference's get_pitch_bends (fixture) and decode_ref.pitch_bends."""
    from oracle import decode_ref

    files, _ = _set(edges, "pitch_edges")
    contour = files[0][2]
    notes = postsets.edge_notes()
    st, en, pi = (np.array([n[k] for n in notes], np.int32) for k in range(3))
    off, bends = model.pitch_bends_arrays(contour, st, en, pi)
    np.testing.assert_array_equal(off, np.cumsum([0] + [b - a for a, b, _ in notes]))
    np.testing.assert_array_equal(bends, edges["pitch_edges/direct/bend_flat"])
    exp = decode_ref.pitch_bends(contour, [(a, b, p, 0.5) for a, b, p in notes])
    np.testing.assert_array_equal(bends, [int(v) for e in exp for v in e[4]])
