"""NumPy / SciPy restatement of mir_eval.transcription 0.7's note matching (tests only).

`hit_matrices` builds the (n_ref, n_est) hit matrices exactly as mir_eval.transcription.match_notes does (float64,
np.subtract.outer, np.around(., 4)); `max_matching` takes the size of a maximum bipartite matching with SciPy
(mir_eval runs Hopcroft-Karp; the maximum size is unique).  `counts` returns what the library's bp_score_* return per
(setting, file) or item: [n_ref, n_est, matched without offsets, matched].
"""
from __future__ import annotations

import numpy as np
import scipy.sparse
from scipy.sparse.csgraph import maximum_bipartite_matching

TOLERANCES = dict(onset_tolerance=0.05, pitch_tolerance=50.0, offset_ratio=0.2, offset_min_tolerance=0.05)


def hit_matrices(ref_intervals, ref_log2, est_intervals, est_log2, onset_tolerance=0.05, pitch_tolerance=50.0,
                 offset_ratio=0.2, offset_min_tolerance=0.05):
    """-> (hits without the offset test, hits with it), bool (n_ref, n_est).  *_log2 are np.log2 of the pitches in Hz."""
    ref_intervals = np.asarray(ref_intervals, np.float64).reshape(-1, 2)
    est_intervals = np.asarray(est_intervals, np.float64).reshape(-1, 2)
    onset_distances = np.around(np.abs(np.subtract.outer(ref_intervals[:, 0], est_intervals[:, 0])), decimals=4)
    onset_hit = onset_distances <= onset_tolerance
    pitch_distances = np.abs(1200 * np.subtract.outer(np.asarray(ref_log2, np.float64), np.asarray(est_log2, np.float64)))
    pitch_hit = pitch_distances <= pitch_tolerance
    note_hit = np.logical_and(onset_hit, pitch_hit)
    offset_distances = np.around(np.abs(np.subtract.outer(ref_intervals[:, 1], est_intervals[:, 1])), decimals=4)
    ref_durations = np.abs(np.diff(ref_intervals, axis=-1)).flatten()
    offset_tolerances = np.maximum(offset_ratio * ref_durations, offset_min_tolerance)
    offset_hit = offset_distances <= offset_tolerances.reshape(-1, 1)
    return note_hit, np.logical_and(note_hit, offset_hit)


def max_matching(hits) -> int:
    hits = np.asarray(hits, bool)
    if hits.size == 0 or not hits.any():
        return 0
    m = maximum_bipartite_matching(scipy.sparse.csr_matrix(hits), perm_type="column")
    return int((m >= 0).sum())


def counts(ref_intervals, ref_pitches_hz, est_intervals, est_pitches_hz, **tolerances):
    """[n_ref, n_est, matched without offsets, matched] of one file (0 matches when either side is empty)."""
    tol = {**TOLERANCES, **tolerances}
    n_ref, n_est = len(ref_pitches_hz), len(est_pitches_hz)
    if n_ref == 0 or n_est == 0:
        return [n_ref, n_est, 0, 0]
    no_off, with_off = hit_matrices(ref_intervals, np.log2(np.asarray(ref_pitches_hz, np.float64)), est_intervals,
                                    np.log2(np.asarray(est_pitches_hz, np.float64)), **tol)
    return [n_ref, n_est, max_matching(no_off), max_matching(with_off)]
