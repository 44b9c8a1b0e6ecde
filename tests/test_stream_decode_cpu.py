"""The cut property of the note stream (oracle/stream_ref.py, DESIGN.md §4.5) on the CPU: decoded segment by segment with
the whole recording's maxima, the stream gives exactly the notes of the whole-recording decode (oracle/decode_ref.py),
and with its running maxima each segment is the direct decode of its range under those maxima."""
import numpy as np
import pytest

from oracle import decode_ref, stream_ref
from tests import streamsets
from tests.golden_util import case_params, dequant

PARAMS = [
    dict(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, infer_onsets_flag=True, melodia_trick=True),
    dict(onset_thresh=0.5, frame_thresh=0.3, min_note_len=1, infer_onsets_flag=True, melodia_trick=False),
    dict(onset_thresh=0.3, frame_thresh=0.3, min_note_len=0, infer_onsets_flag=False, melodia_trick=True),
    dict(onset_thresh=0.2, frame_thresh=0.3, min_note_len=11, infer_onsets_flag=True, melodia_trick=True),
]
RANGES = [(0, 88), (20, 70), (0, 40)]


def note_key(n):
    a, b, p, amp, bends = n
    return (int(a), int(b), int(p), int(np.float32(amp).view(np.int32)), None if bends is None else tuple(int(v) for v in bends))


def whole(out, p, tol, lo, hi):
    with np.errstate(all="ignore"):
        wb, ev = decode_ref.model_output_to_note_events(
            {k: np.array(v) for k, v in out.items()}, p["onset_thresh"], p["frame_thresh"], p["infer_onsets_flag"],
            p["min_note_len"], melodia_trick=p["melodia_trick"], energy_tol=tol, lo_col=lo, hi_col=hi)  # fmt: skip
    return wb, ev


def assert_cut_property(out, p, tol, lo, hi, min_cuts=0):
    wb, ev = whole(out, p, tol, lo, hi)
    segs, plan = stream_ref.stream_notes(out, energy_tol=tol, lo_col=lo, hi_col=hi,
                                         maxima=stream_ref.whole_maxima(out, lo, hi), **p)
    got = [n for s in segs for n in s]
    assert len(plan) - 1 >= min_cuts
    assert sorted(map(note_key, got)) == sorted(map(note_key, wb)), (p, tol, lo, hi)
    n = out["note"].shape[0]
    key_t = lambda e: (float(e[0]), float(e[1]), int(e[2]), note_key((0, 0, 0, e[3], e[4]))[3:])  # noqa: E731
    assert sorted(map(key_t, stream_ref.events(got, n))) == sorted(map(key_t, ev))


@pytest.mark.parametrize("name", ["notes10s", "chords4s", "constant", "fuzz0", "fuzz1", "fuzz2", "tiny1", "tiny25"])
def test_cut_property_on_golden_posteriorgrams(golden_dir, name):
    z = np.load(golden_dir / "decode_cases.npz")
    out = {k: dequant(z[f"{name}/{k}_q"]) for k in ("note", "onset", "contour")}
    from basic_pitch_b200.note_creation import frequency_to_column_range

    for j in sorted({k.split("/")[1] for k in z.keys() if k.startswith(f"{name}/p")}):
        cp = case_params(z, f"{name}/{j}")
        lo, hi = frequency_to_column_range(cp["min_freq"], cp["max_freq"])
        p = dict(onset_thresh=cp["onset_thresh"], frame_thresh=cp["frame_thresh"], min_note_len=cp["min_note_len"],
                 infer_onsets_flag=cp["infer_onsets"], melodia_trick=cp["melodia_trick"])
        for tol in (11, 3):
            assert_cut_property(out, p, tol, lo, hi)


def test_cut_property_on_the_edge_posteriorgrams():
    from tests import postsets

    for name in ("runs", "ties", "nan_file"):
        files, grid = postsets.get(name)
        for f in files:
            out = {"note": f[0], "onset": f[1], "contour": f[2]}
            for q in grid[:3]:
                p = dict(onset_thresh=q["onset_thresh"], frame_thresh=q["frame_thresh"], min_note_len=q["min_note_len"],
                         infer_onsets_flag=q["infer_onsets"], melodia_trick=q["melodia_trick"])
                assert_cut_property(out, p, q["energy_tol"], q["lo_col"], q["hi_col"])


@pytest.mark.parametrize("tol", [11, 1, 2, 5, 20])
@pytest.mark.parametrize("level", ["below", "zero", "equal"])
def test_cut_property_on_gaps_of_the_minimum_length(tol, level):
    for seed in range(3):
        out = streamsets.gapped(seed, streamsets.gap_lengths(tol), gap_level=level)
        for p in PARAMS:
            for lo, hi in RANGES:
                assert_cut_property(out, p, tol, lo, hi)


@pytest.mark.parametrize("tol", [11, 4])
def test_cuts_fall_on_quiet_runs_of_the_minimum_length_only(tol):
    gaps = streamsets.gap_lengths(tol)
    out = streamsets.gapped(5, gaps, gap_level="zero", gap_onset_peaks=False)
    quiet = stream_ref.quiet_frames(out["note"], 0.3, 0, 88)
    plan = stream_ref.plan(quiet, tol)
    # the bursts are never quiet at both ends (a plateau may sit anywhere), so count the runs directly
    runs, t = [], 0
    while t < len(quiet):
        if quiet[t]:
            u = t
            while u < len(quiet) and quiet[u]:
                u += 1
            runs.append((t, u))
            t = u
        else:
            t += 1
    expect = [q0 + stream_ref.LB for q0, q1 in runs if q1 - q0 >= tol + stream_ref.LB]
    assert [s[1] for s in plan[:-1]] == expect
    assert len(expect) >= 4
    for a, b, s, e, r in plan[:-1]:
        assert quiet[b - stream_ref.LB : b + tol].all() and (b - stream_ref.LB == 0 or not quiet[b - stream_ref.LB - 1])
        assert e == b + stream_ref.ctx_after(tol) and s == (a if a == r else a - stream_ref.CTX_BEFORE)
    # a value equal to frame_thresh is not quiet, and frame_thresh <= 0 never cuts
    eq = np.array(out["note"])
    cuts = [s[1] for s in plan[:-1]]
    eq[cuts, 7] = np.float32(0.3)
    assert not stream_ref.quiet_frames(eq, 0.3, 0, 88)[cuts].any()
    assert len(stream_ref.plan(stream_ref.quiet_frames(eq, 0.3, 0, 88), tol)) < len(plan)
    eq[cuts, 7] = np.nextafter(np.float32(0.3), np.float32(0))
    assert stream_ref.plan(stream_ref.quiet_frames(eq, 0.3, 0, 88), tol) == plan
    assert len(stream_ref.plan(stream_ref.quiet_frames(out["note"], 0.0, 0, 88), tol)) == 1


def test_running_maxima_segments_are_direct_decodes():
    for seed in range(3):
        out = streamsets.gapped(seed, streamsets.gap_lengths(11))
        for p in PARAMS:
            segs, plan = stream_ref.stream_notes(out, **p)
            nc = stream_ref.constrained(out["note"], 0, 88)
            oc = stream_ref.constrained(out["onset"], 0, 88)
            for notes, (a, b, s, e, r) in zip(segs, plan):
                mo = oc[:e].max()
                mf = stream_ref.frame_diff(nc, [0])[:e].max()
                seg = {"note": nc[s:e], "onset": oc[s:e], "contour": out["contour"][s:e]}
                on = stream_ref.infer_onsets_with(seg["onset"], seg["note"], mo, mf) if p["infer_onsets_flag"] else seg["onset"]
                with np.errstate(all="ignore"):
                    local = decode_ref.output_to_notes_polyphonic(
                        np.array(seg["note"]), on, p["onset_thresh"], p["frame_thresh"], p["min_note_len"], False, None,
                        None, p["melodia_trick"], 11)  # fmt: skip
                wb = decode_ref.pitch_bends(seg["contour"], [x for x in local if a <= s + x[0] < b])
                assert list(map(note_key, notes)) == [note_key((s + x[0], s + x[1], *x[2:])) for x in wb]


def test_maxima_in_the_first_segment_make_the_running_maxima_exact():
    out = streamsets.gapped(2, streamsets.gap_lengths(11), maxima_first=True)
    for p in PARAMS:
        wb, _ = whole(out, p, 11, 0, 88)
        segs, plan = stream_ref.stream_notes(out, **p)
        assert len(plan) > 3
        assert sorted(map(note_key, [n for s in segs for n in s])) == sorted(map(note_key, wb))


def test_forced_cuts_decode_each_part_as_a_file():
    out = streamsets.gapped(3, [4] * 6)
    out["note"][::4, 3] = 0.5  # no quiet run long enough: only forced cuts
    p = PARAMS[0]
    segs, plan = stream_ref.stream_notes(out, max_segment_frames=40, **p)
    n = out["note"].shape[0]
    assert [s[1] for s in plan[:-1]] == list(range(40, n, 40))[: len(plan) - 1] and plan[-1][1] == n
    for notes, (a, b, s, e, r) in zip(segs, plan):
        assert s == a == r and e == b
        assert all(a <= x[0] < b and x[1] <= b for x in notes)
