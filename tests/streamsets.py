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
