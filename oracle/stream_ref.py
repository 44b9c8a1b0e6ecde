"""ORACLE (test infrastructure, not product code): NumPy restatement of the streamed note decode (bp_stream_*,
include/bp_b200.h; DESIGN.md §4.5) on top of `oracle/decode_ref.py`.

Only `tests/` and tools that check the library against it may import this module.

The stream cuts a recording at quiet stretches and decodes each segment, with a few frames of context, on its own:

  * quiet frame   every column of the pitch range [lo, hi) has a note value strictly below frame_thresh (float64
                  compare, NaN is not quiet); columns outside the range count as 0, so frame_thresh <= 0 never gives one
  * cut           at frame c when frames [c - LB, c + LA) are quiet and frame c - LB - 1 is not (or c - LB is where the
                  recording, or the part after a forced cut, starts): one cut per quiet run of at least LA + LB frames,
                  LA = energy_tol, LB = 3.  It is known once frame c + LA - 1 has arrived.
  * segment       frames [a, b) between two cuts, decoded over [a - CTX_BEFORE, b + ctx_after(energy_tol)) (no context
                  before the start of the recording or of a forced part); only notes starting in [a, b) are kept
  * maxima        segment k infers its onsets with max(onsets) and max(frame_diff) over stream frames [0, e_k), e_k the
                  end of its decode range; frame_diff is zero on the first two frames of the recording and of every
                  forced part (as at the start of a file)
  * forced cut    with max_segment_frames = M > 0: when M frames have arrived since the segment's start a without a
                  cut known within them, the stream cuts at a + M as at a file boundary
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from oracle import decode_ref

LB = 3  # quiet frames before a cut: the peak pick at the cut reads frame c - 1, whose inferred onset reads c - 3
CTX_BEFORE = 3  # decode context before a segment that starts at a cut


def cut_after(energy_tol: int) -> int:
    """LA: quiet frames from a cut on (a candidate on the last quiet frame before the cut scans energy_tol frames)."""
    return int(energy_tol)


def ctx_after(energy_tol: int) -> int:
    """Decode context after a segment that ends at a cut: a track whose last loud frame is c - LB - 1 reads up to
    c - LB - 1 + energy_tol, which the scan's `i < n_frames - 1` bound must admit; the peak pick at c - 1 reads frame c."""
    return max(1, int(energy_tol) - 2)


def quiet_frames(note: np.ndarray, frame_thresh: float, lo: int, hi: int) -> np.ndarray:
    n = note.shape[0]
    if not frame_thresh > 0:
        return np.zeros(n, bool)
    with np.errstate(invalid="ignore"):
        return np.all(note[:, lo:hi].astype(np.float64) < frame_thresh, axis=1)


def constrained(m: np.ndarray, lo: int, hi: int) -> np.ndarray:
    out = np.array(m, dtype=np.float32, copy=True)
    out[:, :lo] = 0
    out[:, hi:] = 0
    return out


def frame_diff(note_c: np.ndarray, starts) -> np.ndarray:
    """float64 (T,88) positive part of min(n[t] - n[t-1], n[t] - n[t-2]), zero on the first two frames after each start."""
    f64 = note_c.astype(np.float64)
    d = np.zeros_like(f64)
    if f64.shape[0] > 2:
        d[2:] = np.minimum(f64[2:] - f64[1:-1], f64[2:] - f64[:-2])
    d[d < 0] = 0
    for s in starts:
        d[s : s + 2] = 0
    return d


def infer_onsets_with(onsets: np.ndarray, frames: np.ndarray, max_onset, max_fd) -> np.ndarray:
    """decode_ref.infer_onsets on one decode range, with the two maxima passed in instead of taken over the range."""
    n_t, n_f = frames.shape
    f64 = frames.astype(np.float64)
    diff = None
    for n in range(1, 3):
        lagged = np.concatenate([np.zeros((n, n_f)), f64])[:n_t]
        d = f64 - lagged
        diff = d if diff is None else np.minimum(diff, d)
    diff[diff < 0] = 0
    diff[:2, :] = 0
    with np.errstate(invalid="ignore", divide="ignore"):
        diff = max_onset * diff / max_fd
    return np.maximum(onsets.astype(np.float64), diff)


def plan(quiet: np.ndarray, energy_tol: int, max_segment_frames: int = 0) -> List[Tuple[int, int, int, int, int]]:
    """Segments of a stream of len(quiet) frames, in order: (a, b, s, e, r) = kept frames [a, b), decode range [s, e),
    start r of the recording or forced part the segment belongs to."""
    n = len(quiet)
    la, w = cut_after(energy_tol), cut_after(energy_tol) + LB
    after = ctx_after(energy_tol)
    m = int(max_segment_frames)
    segs = []
    r, a = 0, 0
    last = -1  # the frame before the current cut-eligible quiet run (None: the run already gave a cut)

    def start(a_, r_):
        return a_ if a_ == r_ else a_ - CTX_BEFORE

    for t in range(n):
        if m > 0 and t == a + m:  # forced cut: no cut became known within the segment's first m frames
            segs.append((a, t, start(a, r), t, r))
            r = a = t
            last = t - 1
        if not quiet[t]:
            last = t
        elif last is not None and t - last == w:
            c = t - la + 1
            segs.append((a, c, start(a, r), c + after, r))
            a, last = c, None
    if m > 0 and n == a + m:  # the last m frames pushed complete a part: the forced cut is known with frame n - 1
        segs.append((a, n, start(a, r), n, r))
        r = a = n
    segs.append((a, n, start(a, r), n, r))
    return segs


def confirmations(segs, energy_tol: int) -> List[Tuple[int, bool]]:
    """(confirming frame, forced) of every cut of a plan: frame c + LA - 1 for a quiet cut at c, a + M - 1 for a forced
    cut at a + M (a forced cut ends its decode range at the cut, a quiet one ctx_after frames later)."""
    return [(b - 1, True) if e == b else (b + cut_after(energy_tol) - 1, False) for a, b, s, e, r in segs[:-1]]


def push_schedule(segs, energy_tol: int, ends) -> Tuple[List[int], List[int]]:
    """For pushes that end at the stream frames `ends` (cumulative frame counts, nondecreasing; a 0-frame push repeats
    the previous end): closed_by[k] = the push that returns segment k's notes, the first whose frames include the cut's
    confirming frame (len(ends): the end of the stream); held[j] = held frames after push j, n_j - (a if a == r else
    a - 3) for the segment [a, ..) still open then (its decode start)."""
    conf = [t for t, _ in confirmations(segs, energy_tol)]
    closed_by = [next((j for j, n in enumerate(ends) if n > t), len(ends)) for t in conf] + [len(ends)]
    held = []
    for n in ends:
        k = next((i for i, t in enumerate(conf) if t >= n), len(conf))
        held.append(int(n) - segs[k][2])
    return closed_by, held


def stream_notes(output: Dict[str, np.ndarray], onset_thresh: float, frame_thresh: float, infer_onsets_flag: bool = True,
                 min_note_len: int = 11, melodia_trick: bool = True, energy_tol: int = 11, lo_col: int = 0,
                 hi_col: int = 88, include_pitch_bends: bool = True, max_segment_frames: int = 0,
                 maxima: Optional[Tuple[float, float]] = None, decoded: Optional[list] = None):
    """The stream's output, one list per segment of (start, end, pitch, amp, bends) frame-indexed notes (global frames)
    in the reference's generation order for that segment, plus the plan.  `maxima` = (max onset, max frame_diff) replaces
    the running maxima (the whole file's make the decode exact).  `decoded`, a list, receives per segment the number of
    notes its decode range yields before the start filter."""
    note, onset, contour = output["note"], output["onset"], output["contour"]
    n = note.shape[0]
    lo, hi = int(lo_col), int(hi_col)
    nc, oc = constrained(note, lo, hi), constrained(onset, lo, hi)
    segs = plan(quiet_frames(note, frame_thresh, lo, hi), energy_tol, max_segment_frames)
    fd = frame_diff(nc, sorted({s[4] for s in segs}))
    out = []
    for a, b, s, e, _r in segs:
        if e <= s:
            out.append([])
            if decoded is not None:
                decoded.append(0)
            continue
        if maxima is None:
            mo, mf = oc[:e].max(), fd[:e].max()
        else:
            mo, mf = maxima
        on = infer_onsets_with(oc[s:e], nc[s:e], mo, mf) if infer_onsets_flag else oc[s:e]
        with np.errstate(invalid="ignore"):
            local = decode_ref.output_to_notes_polyphonic(
                np.array(nc[s:e]), np.array(on), onset_thresh, frame_thresh, min_note_len, False, None, None,
                melodia_trick, energy_tol, lo, hi)  # fmt: skip
        if decoded is not None:
            decoded.append(len(local))
        local = [x for x in local if a <= s + x[0] < b]
        if include_pitch_bends:
            wb = decode_ref.pitch_bends(contour[s:e], local)
        else:
            wb = [(t0, t1, p, amp, None) for t0, t1, p, amp in local]
        out.append([(s + t0, s + t1, p, amp, bd) for t0, t1, p, amp, bd in wb])
    return out, segs


def whole_maxima(output: Dict[str, np.ndarray], lo_col: int = 0, hi_col: int = 88) -> Tuple[float, float]:
    """max(onsets) and max(frame_diff) of the whole recording, as the whole-file decode takes them."""
    nc, oc = constrained(output["note"], lo_col, hi_col), constrained(output["onset"], lo_col, hi_col)
    return (oc.max(), frame_diff(nc, [0]).max()) if oc.shape[0] else (np.float32(0), 0.0)


def events(notes, n_frames: int):
    """Frame-indexed notes -> the reference's (start_s, end_s, pitch, amp, bends) with times at the global frames."""
    times = decode_ref.frames_to_time(n_frames + 1)
    return [(times[a], times[b], p, amp, bd) for a, b, p, amp, bd in notes]
