"""Plain-Python restatement of mir_eval 0.7's note matching and the scores that depend on its pairs (tests only).

mir_eval is not a dependency of this project; this module restates, from the specification in include/bp_b200.h
(bp_match_*), what mir_eval.transcription.match_notes, util._bipartite_match (Hopcroft-Karp after Eppstein's PADS, with
Python dicts walked in insertion order), transcription.average_overlap_ratio and transcription_velocity.match_notes /
precision_recall_f1_overlap compute.  Hits come from oracle/transcription_ref.py (hit_matrices).
"""
from __future__ import annotations

import numpy as np

from oracle import transcription_ref as tr


def match_graph(hits):
    """G = {estimate: [references it hits]} from a bool (n_ref, n_est) hit matrix, built as match_notes builds it: the
    row-major np.where fixes the key order (first reference, then j) and each list is in ascending reference order."""
    G = {}
    for ref_i, est_i in zip(*np.where(np.asarray(hits, bool))):
        G.setdefault(int(est_i), []).append(int(ref_i))
    return G


def bipartite_match(graph, stats=None):
    """{reference: estimate} of util._bipartite_match(graph).  stats (a dict, optional) receives the number of phases
    that augmented ("phases") and of recursions that returned False ("dead")."""
    matching = {}
    for u in graph:
        for v in graph[u]:
            if v not in matching:
                matching[v] = u
                break
    if stats is not None:
        stats.update(phases=0, dead=0)
    while True:
        preds = {}
        unmatched = []
        pred = {u: unmatched for u in graph}
        for v in matching:
            del pred[matching[v]]
        layer = list(pred)
        while layer and not unmatched:
            new_layer = {}
            for u in layer:
                for v in graph[u]:
                    if v not in preds:
                        new_layer.setdefault(v, []).append(u)
            layer = []
            for v in new_layer:
                preds[v] = new_layer[v]
                if v in matching:
                    layer.append(matching[v])
                    pred[matching[v]] = v
                else:
                    unmatched.append(v)
        if not unmatched:
            return matching
        if stats is not None:
            stats["phases"] += 1

        def recurse(v):
            if v in preds:
                L = preds.pop(v)
                for u in L:
                    if u in pred:
                        pu = pred.pop(u)
                        if pu is unmatched or recurse(pu):
                            matching[v] = u
                            return True
                if stats is not None:
                    stats["dead"] += 1
            return False

        for v in unmatched:
            recurse(v)


def match_notes(ref_intervals, ref_log2, est_intervals, est_log2, with_offsets=True, **tolerances):
    """sorted(matching.items()) of one file: [(reference index, estimate index)] in ascending reference order."""
    tol = {**tr.TOLERANCES, **tolerances}
    if len(ref_log2) == 0 or len(est_log2) == 0:
        return []
    no_off, with_off = tr.hit_matrices(ref_intervals, ref_log2, est_intervals, est_log2, **tol)
    return sorted(bipartite_match(match_graph(with_off if with_offsets else no_off)).items())


def match_array(pairs, n_ref):
    """[(reference, estimate)] -> int32 (n_ref,) estimate per reference, -1 where unmatched (the library's layout)."""
    out = np.full(n_ref, -1, np.int32)
    for r, e in pairs:
        out[r] = e
    return out


def average_overlap_ratio(ref_intervals, est_intervals, matching):
    ratios = []
    for r, e in matching:
        ref_int, est_int = ref_intervals[r], est_intervals[e]
        ratios.append((min(ref_int[1], est_int[1]) - max(ref_int[0], est_int[0])) /
                      (max(ref_int[1], est_int[1]) - min(ref_int[0], est_int[0])))
    return 0 if len(ratios) == 0 else np.mean(ratios)


def velocity_matching(ref_velocities, est_velocities, matching, velocity_tolerance=0.1):
    """transcription_velocity.match_notes after the note matching: the pairs whose rescaled velocity is within tolerance."""
    ref_velocities = np.asarray(ref_velocities)
    est_velocities = np.asarray(est_velocities)
    min_velocity, max_velocity = np.min(ref_velocities), np.max(ref_velocities)
    velocity_range = max(1, max_velocity - min_velocity)
    ref_velocities = (ref_velocities - min_velocity) / float(velocity_range)
    matching = np.array(matching)
    if matching.size == 0:
        return []
    ref_matched = ref_velocities[matching[:, 0]]
    est_matched = est_velocities[matching[:, 1]]
    slope, intercept = np.linalg.lstsq(np.vstack([est_matched, np.ones(len(est_matched))]).T, ref_matched)[0]
    est_matched = slope * est_matched + intercept
    within = np.abs(est_matched - ref_matched) < velocity_tolerance
    return [tuple(x) for x in matching[within]]


def f_measure(precision, recall):
    if precision == 0 and recall == 0:
        return 0.0
    return 2 * precision * recall / (precision + recall)


def velocity_scores(ref_intervals, ref_velocities, est_intervals, est_velocities, matching, velocity_tolerance=0.1):
    """(precision, recall, f_measure, average_overlap_ratio) of transcription_velocity.precision_recall_f1_overlap,
    given the note matching of the same pass."""
    if len(ref_velocities) == 0 or len(est_velocities) == 0:
        return 0.0, 0.0, 0.0, 0.0
    kept = velocity_matching(ref_velocities, est_velocities, matching, velocity_tolerance)
    p = float(len(kept)) / len(est_velocities)
    r = float(len(kept)) / len(ref_velocities)
    return p, r, f_measure(p, r), average_overlap_ratio(ref_intervals, est_intervals, kept)
