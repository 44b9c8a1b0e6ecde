"""Note-level transcription scores (addition; no reference counterpart).

The library counts, per (setting, file) or item, the reference notes, the estimated notes and the size of a maximum
matching with and without the offset test (`Model.score_grid`, `Model.score_notes`, `inference.evaluate_grid`;
include/bp_b200.h, bp_score_*).  This module turns the counts into the precision, recall and F-measure of
mir_eval.transcription.precision_recall_f1_overlap (0.7, beta = 1, strict=False), by its formulas.
"""
from __future__ import annotations

from typing import Dict

import numpy as np

# mir_eval.transcription's defaults: onset within 50 ms, pitch within 50 cents, offset within
# max(0.2 x reference duration, 50 ms)
TOLERANCES = dict(onset_tolerance=0.05, pitch_tolerance=50.0, offset_ratio=0.2, offset_min_tolerance=0.05)

# log2(Hz) of MIDI numbers 0..127, the pitch of an estimated note as mir_eval sees it: np.log2 of
# `note_creation.midi_to_hz`
EST_LOG2_HZ = np.ascontiguousarray(np.log2(440.0 * 2.0 ** ((np.arange(128, dtype=np.float64) - 69.0) / 12.0)))

FIELDS = ("n_ref", "n_est", "matched_no_offset", "matched")


def note_scores(counts) -> Dict[str, np.ndarray]:
    """counts (..., 4) as `Model.score_grid` / `score_notes` return them -> dict of float64 arrays of shape counts.shape[:-1]:
    precision, recall, f_measure (with offsets) and precision_no_offset, recall_no_offset, f_measure_no_offset.
    P = m / n_est, R = m / n_ref, F = 2 P R / (P + R) (0 when P = R = 0); all three 0 when either side is empty.
    "mean" holds the same six names averaged over the last axis (over files for a grid: one value per setting; 0 where
    that axis is empty)."""
    c = np.asarray(counts, np.int64)
    if c.ndim < 1 or c.shape[-1] != 4:
        raise ValueError(f"counts must have shape (..., 4), got {c.shape}")
    n_ref, n_est = c[..., 0], c[..., 1]
    empty = (n_ref == 0) | (n_est == 0)
    out: Dict[str, np.ndarray] = {}
    for suffix, m in (("", c[..., 3]), ("_no_offset", c[..., 2])):
        with np.errstate(divide="ignore", invalid="ignore"):
            p = np.where(empty, 0.0, m / n_est)
            r = np.where(empty, 0.0, m / n_ref)
            f = np.where((p == 0) & (r == 0), 0.0, 2.0 * p * r / (p + r))
        out["precision" + suffix], out["recall" + suffix], out["f_measure" + suffix] = p, r, f
    if c.ndim >= 2:
        n = c.shape[-2]
        out["mean"] = {k: (v.mean(axis=-1) if n else np.zeros(v.shape[:-1])) for k, v in out.items()}
    else:
        out["mean"] = {k: (v.mean() if v.size else np.float64(0.0)) for k, v in out.items()}
    return out
