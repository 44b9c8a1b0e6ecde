"""The note stream on the device (bp_stream_*, Model.note_stream, inference.predict_stream_notes) against its NumPy
restatement (oracle/stream_ref.py) bit for bit, and against the whole-recording decode where the stream is exact."""
import ctypes as C

import numpy as np
import pytest

from oracle import stream_ref
from tests import streamsets
from tests.golden_util import case_params, dequant

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH)


def ev_key(e):
    return (float(e[0]), float(e[1]), int(e[2]), int(np.float32(e[3]).view(np.int32)),
            None if e[4] is None else tuple(int(v) for v in e[4]))  # fmt: skip


def run_stream(model, out, p, sizes, max_seg=0):
    """Push `out` in pieces of the sizes given (cycled), then end; returns (events in order, held frames after each
    push, number of pushes that returned notes)."""
    from basic_pitch_b200.inference import NoteStream

    params = model._params(p["onset_thresh"], p["frame_thresh"], p["min_note_len"], p["energy_tol"], p["infer_onsets"],
                           p["melodia_trick"], p["bends"], p["lo"], p["hi"])  # fmt: skip
    s = NoteStream(model, params, max_seg)
    n, t, k, events, held, early = out["note"].shape[0], 0, 0, [], [], 0
    while t < n:
        u = min(n, t + sizes[k % len(sizes)])
        got = s.push(out["note"][t:u], out["onset"][t:u], out["contour"][t:u] if p["bends"] else None)
        events += got
        early += bool(got)
        held.append(s.held_frames)
        t, k = u, k + 1
    events += s.end()
    assert s.held_frames == 0
    return events, held, early


def oracle_events(out, p, max_seg=0, maxima=None):
    segs, plan = stream_ref.stream_notes(
        out, p["onset_thresh"], p["frame_thresh"], p["infer_onsets"], p["min_note_len"], p["melodia_trick"],
        p["energy_tol"], p["lo"], p["hi"], p["bends"], max_seg, maxima)  # fmt: skip
    return stream_ref.events([x for sg in segs for x in sg], out["note"].shape[0]), plan


def prm(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=11, infer_onsets=True, melodia_trick=True,
        bends=True, lo=0, hi=88):
    return dict(onset_thresh=onset_thresh, frame_thresh=frame_thresh, min_note_len=min_note_len, energy_tol=energy_tol,
                infer_onsets=infer_onsets, melodia_trick=melodia_trick, bends=bends, lo=lo, hi=hi)


def golden_inputs(golden_dir):
    z = np.load(golden_dir / "decode_cases.npz")
    from basic_pitch_b200.note_creation import frequency_to_column_range

    for name in ("notes10s", "chords4s", "fuzz1"):
        out = {k: dequant(z[f"{name}/{k}_q"]) for k in ("note", "onset", "contour")}
        for j in ("p0", "p2"):
            cp = case_params(z, f"{name}/{j}")
            lo, hi = frequency_to_column_range(cp["min_freq"], cp["max_freq"])
            yield f"{name}/{j}", out, prm(cp["onset_thresh"], cp["frame_thresh"], cp["min_note_len"], 11,
                                          cp["infer_onsets"], cp["melodia_trick"], True, lo, hi)


def synthetic_inputs():
    for tol in (11, 3):
        for seed in range(2):
            out = streamsets.gapped(seed, streamsets.gap_lengths(tol) * 2, gap_level=("below", "equal")[seed])
            yield f"gapped tol {tol} seed {seed}", out, prm(0.5, 0.3, 0, tol)
            yield f"gapped tol {tol} seed {seed} b", out, prm(0.3, 0.3, 1, tol, False, True, False, 20, 70)
            yield f"gapped tol {tol} seed {seed} c", out, prm(0.2, 0.3, 11, tol, True, False, True, 0, 40)


@pytest.mark.parametrize("sizes", [[1], [7, 13, 29, 101], [1 << 30]], ids=["one-frame", "odd", "all-at-once"])
def test_stream_equals_the_oracle(model, golden_dir, sizes):
    cuts = 0
    for name, out, p in list(golden_inputs(golden_dir)) + list(synthetic_inputs()):
        got, _, _ = run_stream(model, out, p, sizes)
        exp, plan = oracle_events(out, p)
        cuts += len(plan) - 1
        assert list(map(ev_key, got)) == list(map(ev_key, exp)), name
    assert cuts > 50


def test_exact_cases_equal_the_whole_file_decode(model):
    for tol in (11, 4):
        for out, infer in ((streamsets.gapped(7, streamsets.gap_lengths(tol) * 2), False),
                           (streamsets.gapped(8, streamsets.gap_lengths(tol) * 2, maxima_first=True), True)):
            p = prm(0.5, 0.3, 0, tol, infer)
            got, _, _ = run_stream(model, out, p, [5, 17])
            res = model.decode_arrays([out["note"]], [out["onset"]], [out["contour"]], 0.5, 0.3, 0, tol, infer)[0]
            from basic_pitch_b200.note_creation import note_events_from_arrays

            exp = note_events_from_arrays(res, out["note"].shape[0])
            assert len(stream_ref.plan(stream_ref.quiet_frames(out["note"], 0.3, 0, 88), tol)) > 5
            assert sorted(map(ev_key, got)) == sorted(map(ev_key, exp))


def test_forced_cut_on_dense_chords(model):
    from basic_pitch_b200 import synth

    out = model.run_inference_arrays([synth.dense_chords_clip(20.0)])[0]
    forced = 0
    for m in (64, 200):
        p = prm()
        got, held, _ = run_stream(model, out, p, [23, 41])
        exp, plan = oracle_events(out, p)
        assert list(map(ev_key, got)) == list(map(ev_key, exp))
        got, held, _ = run_stream(model, out, p, [23, 41], max_seg=m)
        exp, plan = oracle_events(out, p, max_seg=m)
        forced += sum(b - a == m for a, b, s, e, r in plan[:-1])
        assert list(map(ev_key, got)) == list(map(ev_key, exp))
        assert max(held) <= m + stream_ref.CTX_BEFORE
    assert forced > 0


def test_predict_stream_notes_end_to_end(model):
    from basic_pitch_b200 import synth
    from basic_pitch_b200.inference import predict_stream_notes, run_inference_stream

    audio = synth.melody_clip(180.0, seed=3)
    blocks = lambda: (audio[i : i + 30011] for i in range(0, len(audio), 30011))  # noqa: E731
    steps = list(predict_stream_notes(blocks(), model, windows_per_step=8))
    ref = list(run_inference_stream(blocks(), model, windows_per_step=8))
    assert len(steps) == len(ref) + 1 and steps[-1][0]["note"].shape[0] == 0
    for (part, _), r in zip(steps, ref):
        for k in ("note", "onset", "contour"):
            np.testing.assert_array_equal(part[k], r[k])
    out = {k: np.concatenate([r[k] for r in ref]) for k in ("note", "onset", "contour")}
    got = [e for _, ev in steps for e in ev]
    exp, plan = oracle_events(out, prm())
    assert list(map(ev_key, got)) == list(map(ev_key, exp))
    assert sum(bool(ev) for _, ev in steps[:-1]) >= 3, "notes must come out before the stream ends"
    # held frames: at most the frames since the last cut, i.e. the longest stretch between cuts plus the frames that
    # confirm the next cut and the context before the segment
    _, held, _ = run_stream(model, out, prm(), [r["note"].shape[0] for r in ref])
    longest = max(b - a for a, b, s, e, r in plan)
    assert len(plan) > 10 and max(held) <= longest + 11 - 1 + stream_ref.CTX_BEFORE
    assert max(held) < out["note"].shape[0] // 4


def test_validation_and_capacity(model):
    from basic_pitch_b200 import _lib
    from basic_pitch_b200.inference import Model, NoteStream

    lib = model._lib
    for bad in (model._params(0.5, -0.1, 11, 11, True, True, True, 0, 88),
                model._params(0.5, 0.3, 11, 0, True, True, True, 0, 88),
                model._params(0.5, float("nan"), 11, 11, True, True, True, 0, 88)):
        with pytest.raises(_lib.BpError) as e:
            NoteStream(model, bad)
        assert e.value.code == _lib.BP_E_INVALID
    with pytest.raises(_lib.BpError) as e:
        NoteStream(model, model._params(0.5, 0.3, 11, 11, True, True, True, 0, 88), -1)
    assert e.value.code == _lib.BP_E_INVALID
    # frame_thresh < 0 without melodia is valid and never cuts
    out = streamsets.gapped(1, streamsets.gap_lengths(11))
    p = prm(0.5, -0.1, 0, melodia_trick=False)
    got, held, early = run_stream(model, out, p, [9])
    assert early == 0 and held[-1] == out["note"].shape[0]
    assert list(map(ev_key, got)) == list(map(ev_key, oracle_events(out, p)[0]))

    s = model.note_stream(0.5, 0.3, 0)
    ptr = lambda a: np.ascontiguousarray(a).ctypes.data  # noqa: E731
    lib.bp_stream_push_host(s._h, ptr(out["note"]), ptr(out["onset"]), ptr(out["contour"]), out["note"].shape[0])
    lib.bp_stream_end(s._h)
    notes, arrs = Model._alloc_notes(1, 0, 0)
    with pytest.raises(_lib.BpError) as e:
        lib.bp_stream_take(s._h, C.byref(notes))
    assert e.value.code == _lib.BP_E_CAPACITY
    need_n, need_b = C.c_int64(0), C.c_int64(0)
    lib.bp_last_required(C.byref(need_n), C.byref(need_b))
    assert need_n.value > 0 and need_b.value > 0
    notes, arrs = Model._alloc_notes(1, need_n.value, need_b.value)
    lib.bp_stream_take(s._h, C.byref(notes))
    assert arrs["note_off"][1] == need_n.value and arrs["bend_off"][need_n.value] == need_b.value
    exp, _ = oracle_events(out, prm(0.5, 0.3, 0))
    from basic_pitch_b200.note_creation import frame_index_to_time

    assert list(frame_index_to_time(arrs["start"].astype(np.int64))) == [e[0] for e in exp]
    with pytest.raises(_lib.BpError) as e:
        s.push(out["note"][:3], out["onset"][:3], out["contour"][:3])
    assert e.value.code == _lib.BP_E_INVALID
    with pytest.raises(_lib.BpError) as e:
        s.end()
    assert e.value.code == _lib.BP_E_INVALID
