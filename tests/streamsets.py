"""Posteriorgrams for the note stream (CPU only: plain NumPy, deterministic): bursts of notes separated by quiet gaps
of chosen lengths, so that the stream's cuts (oracle/stream_ref.py) fall where a test wants them."""
from __future__ import annotations

from typing import Dict, Sequence

import numpy as np

N_PITCH, N_BINS = 88, 264


def _q(x) -> np.ndarray:
    return (np.round(np.asarray(x, np.float64) * 64) / 64).astype(np.float32)


def gapped(seed: int, gaps: Sequence[int], frame_thresh: float = 0.3, gap_level: str = "below",
           gap_onset_peaks: bool = True, maxima_first: bool = False) -> Dict[str, np.ndarray]:
    """One burst of random plateaus (values on a 1/64 grid, at most 63/64) before each gap, one after the last.
    gap_level: "below" fills the gaps with values under frame_thresh, "equal" puts one cell equal to it in the middle of
    every gap (such a frame is not quiet), "zero" leaves them 0.  gap_onset_peaks puts isolated onset peaks inside the
    gaps.  maxima_first: the file's max(onsets) and max(frame_diff) (both 1.0) fall in the first burst."""
    rng = np.random.default_rng(seed)
    parts, onsets = [], []
    for k in range(len(gaps) + 1):
        n = int(rng.integers(8, 48))
        b = np.zeros((n, N_PITCH), np.float32)
        for _ in range(int(rng.integers(1, 6))):
            f, t0 = int(rng.integers(0, N_PITCH)), int(rng.integers(0, n))
            b[t0 : t0 + int(rng.integers(1, n - t0 + 1)), f] = rng.uniform(0.3, 63 / 64)
        parts.append(_q(b))
        onsets.append(_q(rng.uniform(0, 1, (n, N_PITCH)) ** 8 * (63 / 64)))
        if k == len(gaps):
            break
        g = int(gaps[k])
        gap = np.zeros((g, N_PITCH), np.float32)
        if gap_level != "zero":
            gap = _q(rng.uniform(0, frame_thresh, (g, N_PITCH)))
            gap[gap >= frame_thresh] = 0
        if gap_level == "equal" and g:
            gap[g // 2, int(rng.integers(0, N_PITCH))] = frame_thresh
        parts.append(gap)
        o = np.zeros((g, N_PITCH), np.float32)
        if gap_onset_peaks:
            for t in range(1, g - 1, 3):
                o[t, int(rng.integers(0, N_PITCH))] = 0.75
        onsets.append(o)
    note, onset = np.concatenate(parts), np.concatenate(onsets)
    if maxima_first:
        note[:4, 40] = 0
        note[4:9, 40] = 1.0
        onset[5, 10] = 1.0
    contour = rng.uniform(0, 1, (note.shape[0], N_BINS)).astype(np.float32)
    return {"note": note, "onset": onset, "contour": contour}


def gap_lengths(energy_tol: int) -> list:
    """Quiet runs of exactly the minimum length (energy_tol + 3), one frame shorter (no cut), longer, and twice it."""
    w = int(energy_tol) + 3
    return [w, w - 1, w + 1, 2 * w, w, w - 1, 3 * w]


def carved(file, setting: Dict, seed: int, columns: str = "all") -> Dict[str, np.ndarray]:
    """A file of tests/postsets.py (note, onset, contour) with quiet runs of w - 1, w, w + 1 and w + 2 frames carved into
    it in turn (w = energy_tol + 3: the shortest run that cuts), a random 1 .. 2 w + 23 frames apart: in each run every
    note cell at or above the setting's frame_thresh becomes nextafter(frame_thresh, 0), in all 88 columns
    (columns="all") or in the setting's pitch range [lo_col, hi_col) only ("range", so loud cells outside the range sit
    inside the runs).  The onsets stay as they were (peaks inside the runs make 1-frame notes at min_note_len 0).  No run
    is carved when frame_thresh <= 0 (no frame is ever quiet) or w exceeds the file."""
    note, onset, contour = (np.array(a, dtype=np.float32, copy=True) for a in file)
    n, tol = note.shape[0], int(setting["energy_tol"])
    ft = np.float32(setting["frame_thresh"])
    lo, hi = (0, N_PITCH) if columns == "all" else (int(setting["lo_col"]), int(setting["hi_col"]))
    rng = np.random.default_rng(seed)
    if ft > 0 and tol + 3 <= n:
        w, below, k = tol + 3, np.nextafter(ft, np.float32(0)), 0
        t = int(rng.integers(0, w))
        while t + w - 1 + k % 4 <= n:
            run = note[t : t + w - 1 + k % 4, lo:hi]
            run[run >= ft] = below
            t += w - 1 + k % 4 + int(rng.integers(1, 2 * w + 24))
            k += 1
    return {"note": note, "onset": onset, "contour": contour}


def placed(n: int, loud: Sequence[int], onset_peaks: Sequence[int] = (), column: int = 40, seed: int = 0,
           frame_thresh: float = 0.3) -> Dict[str, np.ndarray]:
    """n frames of quiet background (values on the 1/64 grid below frame_thresh) with one cell of 0.5 in `column` at each
    frame of `loud`, and onset peaks of 0.75 in that column at the frames of `onset_peaks`: a quiet run cuts exactly when
    w = energy_tol + 3 frames follow a loud frame, so cuts, their confirming frames and forced-cut positions fall where a
    test puts them."""
    rng = np.random.default_rng(seed)
    note = _q(rng.uniform(0, frame_thresh, (n, N_PITCH)))
    note[note >= frame_thresh] = 0
    onset = _q(rng.uniform(0, 0.4, (n, N_PITCH)))
    loud, peaks = np.asarray(loud, np.int64), np.asarray(onset_peaks, np.int64)
    note[loud, column] = 0.5
    onset[peaks, column] = 0.75
    contour = _q(rng.uniform(0, 1, (n, N_BINS)))
    return {"note": note, "onset": onset, "contour": contour}


def maxima_prefix(out: Dict[str, np.ndarray], lo: int = 0, hi: int = N_PITCH) -> Dict[str, np.ndarray]:
    """Four frames before the recording that hold its largest onset (frame 0) and a 0 -> v step (frame 3), v at least
    the recording's largest note value and frame difference, in column lo of the pitch range [lo, hi): both maxima of the
    inferred onsets then arrive in the first segment, so the running maxima are the whole recording's.  Only valid where
    the recording has no NaN note or onset cell (callers check)."""
    from oracle import stream_ref

    note, onset, contour = out["note"], out["onset"], out["contour"]
    mo, mf = stream_ref.whole_maxima(out, lo, hi)
    v = np.float32(max(1.0, float(mf), float(stream_ref.constrained(note, lo, hi).max(initial=0.0))))
    pn, po = np.zeros((4, N_PITCH), np.float32), np.zeros((4, N_PITCH), np.float32)
    if hi > lo:
        pn[3, lo] = v
        po[0, lo] = max(np.float32(mo), np.float32(0))
    pc = np.zeros((4, N_BINS), np.float32)
    return {"note": np.concatenate([pn, note]), "onset": np.concatenate([po, onset]), "contour": np.concatenate([pc, contour])}


LONG_SETTING = dict(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, energy_tol=11, infer_onsets=False,
                    melodia_trick=True, lo_col=0, hi_col=N_PITCH)


def long_stream(min_frames: int = 70_000) -> Dict[str, np.ndarray]:
    """Carved long_notes and ties files (tests/postsets.py) end to end, under LONG_SETTING's energy_tol and frame_thresh,
    until more than min_frames frames: the quiet scan then needs its grid-stride loop (more than 4 096 CTAs of 8 rows)
    when the whole stream arrives in one push."""
    from tests import postsets

    parts, total, k = [], 0, 0
    files = postsets.get("long_notes")[0] + postsets.get("ties")[0]
    while total <= min_frames:
        part = carved(files[k % len(files)], LONG_SETTING, 1000 + k)
        parts.append(part)
        total += part["note"].shape[0]
        k += 1
    return {key: np.concatenate([p[key] for p in parts]) for key in ("note", "onset", "contour")}


def carved_cases(name: str):
    """(label, carved input, setting) for every file of a tests/postsets.py set under every setting of its grid (the
    0-frame file of `lengths` left out); columns="range" on every other case."""
    from tests import postsets

    files, grid = postsets.get(name)
    k = 0
    for i, f in enumerate(files):
        if f[0].shape[0] == 0:
            continue
        for j, p in enumerate(grid):
            cols = ("all", "range")[k % 2]
            yield f"{name}[{i}] setting {j} {cols}", carved(f, p, 100 * i + j, cols), p
            k += 1


# the quiet scan of csrc/stream.cu: 8 rows (one per warp) per CTA when flagging, at most 4 096 CTAs, and a last CTA that
# walks the flags in chunks of 256 rows (32-row warps) from the scan start, carrying the last loud row between chunks
SCAN_ROWS_PER_CTA, SCAN_MAX_CTAS, SCAN_CHUNK, SCAN_WARP = 8, 4096, 256, 32


def dense_cuts(spans: Sequence[int], energy_tol: int, n_tail: int = 40, peaks_at_cuts: bool = True):
    """Loud frames (one cell each) filling [s, s + x] for each x of `spans`, s the frame after the previous cut's
    confirming frame (0 first): the quiet run after them is confirmed as a cut at s + x + w (w = energy_tol + 3), so the
    last loud row sits x rows and the confirming frame x + w rows after the scan start.  Returns (n, loud, confirming
    frames, onset peaks on the cut frames)."""
    w = int(energy_tol) + 3
    loud, confirms, s = [], [], 0
    for x in spans:
        loud += list(range(s, s + x + 1))
        confirms.append(s + x + w)
        s = s + x + w + 1
    peaks = [t - int(energy_tol) + 1 for t in confirms] if peaks_at_cuts else []
    return s + n_tail, loud, confirms, peaks


def geometry_cases():
    """(label, input, setting) whose cuts reach the corners of the quiet scan when pushed as the tests push them: last
    loud rows on the last row of a warp and of a chunk, confirming frames 255 / 256 / 257 rows after the scan start and in
    the chunk after the last loud row, quiet runs longer than a chunk (energy_tol 300), with onset peaks on the cut
    frames (min_note_len 0: 1-frame notes that start exactly at a cut)."""
    base = dict(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, energy_tol=11, infer_onsets=False,
                melodia_trick=True, lo_col=0, hi_col=N_PITCH)
    out = []
    for tol, spans in ((11, [241, 242, 243, 31, 255, 511, 0, 3, 30, 32, 254, 256, 767]), (300, [100, 0, 255, 600]),
                       (2, [31, 255, 253, 0, 1, 2, 223])):
        n, loud, _, peaks = dense_cuts(spans, tol)
        p = dict(base, energy_tol=tol)
        out.append((f"dense tol {tol}", placed(n, loud, peaks, seed=tol), p))
    return out


def precedence(max_seg: int, energy_tol: int, d: int, reps: int = 4) -> Dict[str, np.ndarray]:
    """Loud frames that put each segment's first quiet-cut confirmation at a + max_seg + d (a: the segment's start),
    `reps` times: with d < 0 every cut is a quiet one, with d >= 0 the forced cut at a + max_seg comes first (needs
    max_seg + d >= 2 (energy_tol + 3))."""
    w, loud, a, s = int(energy_tol) + 3, [], 0, 0
    for _ in range(reps):
        t = a + max_seg + d
        loud += list(range(s, t - w + 1))
        if d < 0:
            a, s = t - int(energy_tol) + 1, t + 1
        else:
            a = a + max_seg
            s = a + 1
    return placed(s + max_seg + 8, loud, seed=max_seg + d)
