"""The note stream's adversarial inputs on the CPU (tests/streamsets.py, oracle/stream_ref.py; DESIGN.md §4.5): the cut
property on every carved decode edge set, the push schedule (which push returns each segment, how many frames are held
after each push) on hand-worked cases, the scan geometry the device inputs reach, and a NumPy model of the quiet scan's
last-CTA walk (csrc/stream.cu) that must cut where the sequential rule does."""
import numpy as np
import pytest

from oracle import stream_ref
from tests import postsets, streamsets
from tests.test_stream_decode_cpu import note_key, whole

NO_RUN = -(1 << 60)  # no cut-eligible quiet run in progress (csrc/kernels.cuh kStreamNoRun)


def ref_params(q):
    return dict(onset_thresh=q["onset_thresh"], frame_thresh=q["frame_thresh"], min_note_len=q["min_note_len"],
                infer_onsets_flag=q["infer_onsets"], melodia_trick=q["melodia_trick"])


@pytest.mark.parametrize("name", postsets.NAMES)
def test_cut_property_on_every_carved_set(name):
    """Decoded segment by segment with the whole recording's maxima, every carved file under every setting of its grid
    gives exactly the whole-recording decode's notes."""
    cases = cuts = 0
    for label, out, q in streamsets.carved_cases(name):
        tol, lo, hi = q["energy_tol"], q["lo_col"], q["hi_col"]
        wb, _ = whole(out, ref_params(q), tol, lo, hi)
        segs, plan = stream_ref.stream_notes(out, energy_tol=tol, lo_col=lo, hi_col=hi,
                                             maxima=stream_ref.whole_maxima(out, lo, hi), **ref_params(q))
        assert sorted(map(note_key, [n for s in segs for n in s])) == sorted(map(note_key, wb)), label
        cases, cuts = cases + 1, cuts + len(plan) - 1
    assert cuts >= 10, (name, cuts)  # the carving makes every set cut (the sets alone rarely do)
    print(f"{name}: {cases} cases, {cuts} cuts")


def test_push_schedule_on_hand_worked_plans():
    # energy_tol 2 (LA 2, w 5, ctx_after 1); loud frames 0 and 10: cuts at 4 (confirmed at 5) and 14 (at 15)
    quiet = np.ones(20, bool)
    quiet[[0, 10]] = False
    segs = stream_ref.plan(quiet, 2)
    assert segs == [(0, 4, 0, 5, 0), (4, 14, 1, 15, 0), (14, 20, 11, 20, 0)]
    assert stream_ref.confirmations(segs, 2) == [(5, False), (15, False)]
    closed_by, held = stream_ref.push_schedule(segs, 2, [3, 5, 6, 6, 15, 16, 20])
    assert closed_by == [2, 5, 7]  # frame 5 arrives with push 2, frame 15 with push 5; the rest at the end
    assert held == [3, 5, 5, 5, 14, 5, 9]
    closed_by, held = stream_ref.push_schedule(segs, 2, [20])
    assert closed_by == [0, 0, 1] and held == [9]
    closed_by, held = stream_ref.push_schedule(segs, 2, [0, 0])
    assert closed_by == [2, 2, 2] and held == [0, 0]

    # no quiet frame, M = 6: forced cuts at 6, 12, 18, each confirmed by the frame before it; no context at a forced cut
    segs = stream_ref.plan(np.zeros(20, bool), 2, 6)
    assert segs == [(0, 6, 0, 6, 0), (6, 12, 6, 12, 6), (12, 18, 12, 18, 12), (18, 20, 18, 20, 18)]
    assert stream_ref.confirmations(segs, 2) == [(5, True), (11, True), (17, True)]
    assert stream_ref.push_schedule(segs, 2, [5, 6, 12, 20]) == ([1, 2, 3, 4], [5, 0, 0, 2])

    # M = 6 with loud frame 0: the quiet cut confirmed at 5 = a + M - 1 wins; then forced at 4 + 6 = 10, a quiet cut
    # confirmed at 14 (the forced part's start counts as the run's start: cut at 13), forced at 19
    quiet = np.ones(20, bool)
    quiet[0] = False
    segs = stream_ref.plan(quiet, 2, 6)
    assert segs == [(0, 4, 0, 5, 0), (4, 10, 1, 10, 0), (10, 13, 10, 14, 10), (13, 19, 10, 19, 10), (19, 20, 19, 20, 19)]
    assert stream_ref.confirmations(segs, 2) == [(5, False), (9, True), (14, False), (18, True)]
    assert stream_ref.push_schedule(segs, 2, [9, 10, 15, 19]) == ([0, 1, 2, 3, 4], [8, 0, 5, 0])
    # M = 5: the forced cut at 5 comes first (a quiet cut confirmed at a + M is too late)
    assert stream_ref.plan(quiet, 2, 5)[:2] == [(0, 5, 0, 5, 0), (5, 8, 5, 9, 5)]


def walk(quiet, start, last, w, carry=True):
    """The quiet scan's last CTA: from row `start` in chunks of 256 rows, the inclusive prefix maximum of the loud rows
    (within the chunk, then `last` carried from the chunks before), and the first quiet row t with t - L == w.
    Returns (t or -1, the carried L after the chunk that holds t / after the last chunk)."""
    n, L, chunk = len(quiet), last, streamsets.SCAN_CHUNK
    for base in range(start, n, chunk):
        q = quiet[base : base + chunk]
        rows = np.arange(base, base + len(q))
        m = np.maximum.accumulate(np.where(q, NO_RUN, rows))
        lt = np.maximum(L, m)
        hit = np.flatnonzero(q & (rows - lt == w))
        if carry:
            L = max(L, int(m[-1]))
        if len(hit):
            return int(rows[hit[0]]), L
    return -1, L


def scanned_cuts(quiet, energy_tol, ends, max_seg=0, carry=True):
    """bp_stream_push_host's loop over pushes ending at `ends`, with `walk` as the scan: [(b, forced)] of every cut."""
    la, w = stream_ref.cut_after(energy_tol), stream_ref.cut_after(energy_tol) + stream_ref.LB
    a, last, scan_from, n, cuts = 0, -1, 0, 0, []
    for end in ends:
        if end == n:
            continue
        n = end
        while True:
            t, L = walk(quiet[:n], scan_from, last, w, carry) if scan_from < n else (-1, last)
            if t >= 0 and (max_seg == 0 or t < a + max_seg):
                a, last, scan_from = t - la + 1, NO_RUN, t + 1
                cuts.append((a, False))
            elif max_seg > 0 and n >= a + max_seg:
                a = a + max_seg
                last, scan_from = a - 1, a
                cuts.append((a, True))
            else:
                last, scan_from = L, n
                break
    return cuts


def plan_cuts(segs):
    return [(b, e == b) for a, b, s, e, r in segs[:-1]]


def schedules(n, confirms):
    """The push schedules of the device tests, as cumulative frame counts."""
    def sizes(sz):
        ends, t, k = [], 0, 0
        while t < n:
            t = min(n, t + sz[k % len(sz)])
            ends.append(t)
            k += 1
        return ends

    at = lambda d: sorted({min(n, max(0, t + d)) for t in confirms} | {n})  # noqa: E731
    return {"one": sizes([1]), "7-8-9": sizes([7, 8, 9]), "255-256-257-31": sizes([255, 256, 257, 31]),
            "to t": at(1), "to t + 1": at(2), "to t - 1": at(0), "to t - 2": at(-1), "whole": [n]}  # fmt: skip


def scan_starts(segs, energy_tol, ends):
    """(confirming frame, scan start) of every quiet cut under a push schedule: the scan that finds a cut starts at the
    first frame of its push or after the confirming frame of the cut before, whichever is later."""
    out, prev = [], 0
    for t, forced in stream_ref.confirmations(segs, energy_tol):
        j = next(j for j, e in enumerate(ends) if e > t)
        if not forced:
            out.append((t, max(ends[j - 1] if j else 0, prev)))
        prev = t + 1
    return out


def test_scan_model_equals_the_sequential_rule():
    """On the geometry inputs (and the long stream) under every schedule of the device tests, the chunked walk with the
    carried L cuts exactly where `plan` does; without the carry it does not (the inputs reach the carry)."""
    cases = [(label, out, q["energy_tol"], q["frame_thresh"]) for label, out, q in streamsets.geometry_cases()]
    long = streamsets.long_stream()
    cases.append(("long", long, streamsets.LONG_SETTING["energy_tol"], streamsets.LONG_SETTING["frame_thresh"]))
    missed_without_carry = 0
    for label, out, tol, ft in cases:
        quiet = stream_ref.quiet_frames(out["note"], ft, 0, 88)
        for m in (0, 64):
            segs = stream_ref.plan(quiet, tol, m)
            conf = [t for t, _ in stream_ref.confirmations(segs, tol)]
            for name, ends in schedules(len(quiet), conf).items():
                if label == "long" and name in ("one", "7-8-9"):
                    continue
                assert scanned_cuts(quiet, tol, ends, m) == plan_cuts(segs), (label, m, name)
                if m == 0 and name == "whole":
                    missed_without_carry += scanned_cuts(quiet, tol, ends, m, carry=False) != plan_cuts(segs)
    assert missed_without_carry >= 3


def test_geometry_inputs_reach_the_scan_corners():
    """Confirming frames 0, 1, 255, 256 and 257 rows after the scan start; last loud rows on the last row of a warp and of
    a chunk with the cut confirmed in a later warp / chunk; a quiet run longer than a chunk; one push of more than
    4 096 CTAs x 8 rows (the flag loop's grid stride)."""
    offsets, warp_end, chunk_end, long_runs = set(), 0, 0, 0
    for label, out, q in streamsets.geometry_cases():
        tol = q["energy_tol"]
        segs = stream_ref.plan(stream_ref.quiet_frames(out["note"], q["frame_thresh"], 0, 88), tol)
        conf = [t for t, _ in stream_ref.confirmations(segs, tol)]
        for name, ends in schedules(out["note"].shape[0], conf).items():
            for t, s0 in scan_starts(segs, tol, ends):
                offsets.add(t - s0)
                lo = t - tol - 3 - s0  # the last loud row, relative to the scan start
                if lo >= 0 and name == "whole":
                    warp_end += lo % 32 == 31 and (t - s0) // 32 > lo // 32
                    chunk_end += lo % 256 == 255 and (t - s0) // 256 > lo // 256
                    long_runs += (t - s0) // 256 > lo // 256 and tol + 3 > 256
        # every cut frame carries an onset peak (a note that starts exactly at the cut)
        assert all(out["onset"][b, 40] == 0.75 for a, b, s, e, r in segs[:-1]), label
    assert {0, 1, 255, 256, 257} <= offsets, sorted(offsets)
    assert warp_end >= 2 and chunk_end >= 2 and long_runs >= 2, (warp_end, chunk_end, long_runs)
    assert streamsets.long_stream()["note"].shape[0] > 2 * streamsets.SCAN_MAX_CTAS * streamsets.SCAN_ROWS_PER_CTA
