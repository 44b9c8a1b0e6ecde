"""Plain-NumPy restatement of mir_eval 0.7's onset-only and offset-only note scores and of transcription.evaluate
(tests only).

mir_eval is not a dependency of this project; this module restates, from the specification in include/bp_b200.h
(bp_score_onset_offset_*), what mir_eval.transcription.match_note_onsets / match_note_offsets (strict=False),
onset_precision_recall_f1 / offset_precision_recall_f1 and evaluate compute.  The matching is
oracle/note_matching_ref.py's restatement of util._bipartite_match; the note-level values come from
oracle/transcription_ref.py's hit matrices through note_matching_ref.
"""
from __future__ import annotations

import collections

import numpy as np

from oracle import note_matching_ref as nm
from oracle import transcription_ref as tr


def _intervals(iv):
    return np.asarray(iv, np.float64).reshape(-1, 2)


def onset_hits(ref_intervals, est_intervals, onset_tolerance=0.05):
    """bool (n_ref, n_est) hit matrix of match_note_onsets."""
    ref_intervals, est_intervals = _intervals(ref_intervals), _intervals(est_intervals)
    onset_distances = np.abs(np.subtract.outer(ref_intervals[:, 0], est_intervals[:, 0]))
    onset_distances = np.around(onset_distances, decimals=4)
    return np.less_equal(onset_distances, onset_tolerance)


def offset_hits(ref_intervals, est_intervals, offset_ratio=0.2, offset_min_tolerance=0.05):
    """bool (n_ref, n_est) hit matrix of match_note_offsets."""
    ref_intervals, est_intervals = _intervals(ref_intervals), _intervals(est_intervals)
    offset_distances = np.abs(np.subtract.outer(ref_intervals[:, 1], est_intervals[:, 1]))
    offset_distances = np.around(offset_distances, decimals=4)
    ref_durations = np.abs(np.diff(ref_intervals, axis=-1)).flatten()
    offset_tolerances = np.maximum(offset_ratio * ref_durations, offset_min_tolerance)
    return np.less_equal(offset_distances, offset_tolerances.reshape(-1, 1))


def match_hits(hits):
    """sorted(util._bipartite_match(G).items()) with G keyed by estimate, as match_note_onsets / _offsets build it."""
    return sorted(nm.bipartite_match(nm.match_graph(hits)).items())


def match_note_onsets(ref_intervals, est_intervals, onset_tolerance=0.05):
    return match_hits(onset_hits(ref_intervals, est_intervals, onset_tolerance))


def match_note_offsets(ref_intervals, est_intervals, offset_ratio=0.2, offset_min_tolerance=0.05):
    return match_hits(offset_hits(ref_intervals, est_intervals, offset_ratio, offset_min_tolerance))


def _prf(n_matched, n_ref, n_est):
    precision = float(n_matched) / n_est
    recall = float(n_matched) / n_ref
    return precision, recall, nm.f_measure(precision, recall)


def onset_precision_recall_f1(ref_intervals, est_intervals, onset_tolerance=0.05):
    ref_intervals, est_intervals = _intervals(ref_intervals), _intervals(est_intervals)
    if len(ref_intervals) == 0 or len(est_intervals) == 0:
        return 0.0, 0.0, 0.0
    matching = match_note_onsets(ref_intervals, est_intervals, onset_tolerance)
    return _prf(len(matching), len(ref_intervals), len(est_intervals))


def offset_precision_recall_f1(ref_intervals, est_intervals, offset_ratio=0.2, offset_min_tolerance=0.05):
    ref_intervals, est_intervals = _intervals(ref_intervals), _intervals(est_intervals)
    if len(ref_intervals) == 0 or len(est_intervals) == 0:
        return 0.0, 0.0, 0.0
    matching = match_note_offsets(ref_intervals, est_intervals, offset_ratio, offset_min_tolerance)
    return _prf(len(matching), len(ref_intervals), len(est_intervals))


def counts(ref_intervals, est_intervals, onset_tolerance=0.05, offset_ratio=0.2, offset_min_tolerance=0.05, **_):
    """[n_ref, n_est, onsets matched, offsets matched] of one file or item, as bp_score_onset_offset_* return them."""
    ref_intervals, est_intervals = _intervals(ref_intervals), _intervals(est_intervals)
    n_ref, n_est = len(ref_intervals), len(est_intervals)
    if n_ref == 0 or n_est == 0:
        return [n_ref, n_est, 0, 0]
    return [n_ref, n_est, len(match_note_onsets(ref_intervals, est_intervals, onset_tolerance)),
            len(match_note_offsets(ref_intervals, est_intervals, offset_ratio, offset_min_tolerance))]


def precision_recall_f1_overlap(ref_intervals, ref_pitches_hz, est_intervals, est_pitches_hz, with_offsets=True,
                                **tolerances):
    """transcription.precision_recall_f1_overlap (offset_ratio=None when not with_offsets)."""
    ref_intervals, est_intervals = _intervals(ref_intervals), _intervals(est_intervals)
    if len(ref_pitches_hz) == 0 or len(est_pitches_hz) == 0:
        return 0.0, 0.0, 0.0, 0.0
    matching = nm.match_notes(ref_intervals, np.log2(np.asarray(ref_pitches_hz, np.float64)), est_intervals,
                              np.log2(np.asarray(est_pitches_hz, np.float64)), with_offsets, **tolerances)
    p, r, f = _prf(len(matching), len(ref_pitches_hz), len(est_pitches_hz))
    return p, r, f, nm.average_overlap_ratio(ref_intervals, est_intervals, matching)


def evaluate(ref_intervals, ref_pitches_hz, est_intervals, est_pitches_hz, **tolerances):
    """transcription.evaluate: the 14 values in its key order."""
    tol = {**tr.TOLERANCES, **tolerances}
    scores = collections.OrderedDict()
    (scores["Precision"], scores["Recall"], scores["F-measure"],
     scores["Average_Overlap_Ratio"]) = precision_recall_f1_overlap(ref_intervals, ref_pitches_hz, est_intervals,
                                                                    est_pitches_hz, True, **tol)
    (scores["Precision_no_offset"], scores["Recall_no_offset"], scores["F-measure_no_offset"],
     scores["Average_Overlap_Ratio_no_offset"]) = precision_recall_f1_overlap(ref_intervals, ref_pitches_hz,
                                                                              est_intervals, est_pitches_hz, False,
                                                                              **tol)
    (scores["Onset_Precision"], scores["Onset_Recall"],
     scores["Onset_F-measure"]) = onset_precision_recall_f1(ref_intervals, est_intervals, tol["onset_tolerance"])
    (scores["Offset_Precision"], scores["Offset_Recall"],
     scores["Offset_F-measure"]) = offset_precision_recall_f1(ref_intervals, est_intervals, tol["offset_ratio"],
                                                              tol["offset_min_tolerance"])
    return scores
