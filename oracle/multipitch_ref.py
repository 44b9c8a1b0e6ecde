"""NumPy / SciPy restatement of mir_eval.multipitch 0.7's metrics (tests only).

`resample_index` maps reference frames to estimate frames as mir_eval.multipitch.resample_multipitch does, through
scipy.interpolate.interp1d itself; `hit_matrix` builds a frame's hit matrix as util._fast_hit_windows (plain) or
util._outer_distance_mod_n (chroma) does; `max_matching` takes the size of a maximum bipartite matching with SciPy
(mir_eval runs Hopcroft-Karp; the maximum size is unique).  `counts` returns what the library's frame scorers return
per (setting, file) or item (include/bp_b200.h, rule 4), and `metrics` the 14 floats as mir_eval computes them.
"""
from __future__ import annotations

import numpy as np
import scipy.interpolate
import scipy.sparse
from scipy.sparse.csgraph import maximum_bipartite_matching


def values(hz):
    """frequencies_to_midi, and midi_to_chroma followed by the np.mod of _outer_distance_mod_n."""
    midi = 69.0 + 12.0 * np.log2(np.asarray(hz, np.float64) / 440.0)
    return midi, np.mod(np.mod(midi, 12), 12)


def resample_index(est_time, ref_time):
    """Estimate frame read by each reference frame, -1 for an empty one."""
    est_time, ref_time = np.asarray(est_time, np.float64), np.asarray(ref_time, np.float64)
    n = len(est_time)
    if n == 0:
        return np.full(len(ref_time), -1, np.int64)
    if n == len(ref_time) and np.allclose(est_time, ref_time):
        return np.arange(n, dtype=np.int64)
    idx = scipy.interpolate.interp1d(est_time, np.arange(n), kind="nearest", bounds_error=False, fill_value=n,
                                     assume_sorted=True)(ref_time).astype(np.int64)
    idx[idx == n] = -1
    return idx


def hit_matrix(ref, est, window, chroma):
    """bool (n_ref, n_est): midi values (plain) or chroma values."""
    ref, est = np.asarray(ref, np.float64), np.asarray(est, np.float64)
    if chroma:
        d = np.abs(np.subtract.outer(np.mod(ref, 12), np.mod(est, 12)))
        return np.minimum(d, 12 - d) <= window
    return (ref[:, None] >= (est - window)[None, :]) & (ref[:, None] <= (est + window)[None, :])


def max_matching(hits) -> int:
    hits = np.asarray(hits, bool)
    if hits.size == 0 or not hits.any():
        return 0
    m = maximum_bipartite_matching(scipy.sparse.csr_matrix(hits), perm_type="column")
    return int((m >= 0).sum())


def frame_arrays(ref_time, ref_vals, est_time, est_vals, window=0.5):
    """Per reference frame: |R_k|, |E_k|, tp_k, tp_chroma_k (int64 arrays).  *_vals: [(midi, chroma) per frame]."""
    idx = resample_index(est_time, ref_time)
    empty = (np.zeros(0), np.zeros(0))
    K = len(ref_vals)
    out = np.zeros((4, K), np.int64)
    for k in range(K):
        rm, rc = ref_vals[k]
        em, ec = est_vals[idx[k]] if idx[k] >= 0 else empty
        out[0, k], out[1, k] = len(rm), len(em)
        if len(rm) and len(em):
            out[2, k] = max_matching(hit_matrix(rm, em, window, False))
            out[3, k] = max_matching(hit_matrix(rc, ec, window, True))
    return out


def counts_values(ref_time, ref_vals, est_time, est_vals, window=0.5):
    """[n_ref, n_est, tp, tp_chroma, n_min, miss, fa] of one series pair given as (midi, chroma) values per frame."""
    r, e, tp, tpc = frame_arrays(ref_time, ref_vals, est_time, est_vals, window)
    return [int(r.sum()), int(e.sum()), int(tp.sum()), int(tpc.sum()), int(np.minimum(r, e).sum()),
            int(np.maximum(r - e, 0).sum()), int(np.maximum(e - r, 0).sum())]


def counts(ref_time, ref_freqs, est_time, est_freqs, window=0.5):
    """As counts_values, from frequencies in Hz per frame."""
    return counts_values(ref_time, [values(f) for f in ref_freqs], est_time, [values(f) for f in est_freqs], window)


def metrics(ref_time, ref_freqs, est_time, est_freqs, window=0.5):
    """The 14 floats of mir_eval.multipitch.metrics, by its compute_accuracy / compute_err_score."""
    r, e, tp, tpc = frame_arrays(ref_time, [values(f) for f in ref_freqs], est_time, [values(f) for f in est_freqs],
                                 window)
    out = {}
    for prefix, t in (("", tp.astype(np.float64)), ("chroma_", tpc.astype(np.float64))):
        tp_sum = float(t.sum())
        n_est_sum, n_ref_sum = e.sum(), r.sum()
        acc_denom = (e + r - t).sum()
        out[prefix + "precision"] = tp_sum / n_est_sum if n_est_sum > 0 else 0.0
        out[prefix + "recall"] = tp_sum / n_ref_sum if n_ref_sum > 0 else 0.0
        out[prefix + "accuracy"] = tp_sum / acc_denom if acc_denom > 0 else 0.0
        n_ref_f = float(n_ref_sum)
        if n_ref_f == 0:
            errs = (0.0, 0.0, 0.0, 0.0)
        else:
            miss = r - e
            miss[miss < 0] = 0
            fa = e - r
            fa[fa < 0] = 0
            errs = ((np.min([r, e], axis=0) - t).sum() / n_ref_f, miss.sum() / n_ref_f, fa.sum() / n_ref_f,
                    (np.max([r, e], axis=0) - t).sum() / n_ref_f)
        for name, v in zip(("substitution_error", "miss_error", "false_alarm_error", "total_error"), errs):
            out[prefix + name] = v
    return out
