"""CPU: the facts the onset / offset kernel (csrc/score.cu, onset_offset_kernel) rests on, the oracle it is checked
against (oracle/onset_offset_ref.py), and the host side of the scores (evaluate.onset_offset_scores,
evaluate.TRANSCRIPTION_KEYS).

The kernel needs two facts, established here on random and adversarial note sets: (1) with the estimates in ascending
order of the tested time, every reference's row of the onset and offset hit matrices is one contiguous run; (2) taking
the references by ascending run end, each matched to the smallest free estimate of its run, gives a maximum matching.
`kernel_counts` restates the kernel's steps in Python; it must equal the oracle everywhere."""
import numpy as np
import pytest
import scipy.sparse
from scipy.sparse.csgraph import maximum_bipartite_matching

from oracle import onset_offset_ref as oo

TOL = dict(onset_tolerance=0.05, offset_ratio=0.2, offset_min_tolerance=0.05)


def _around4(x):
    return np.around(np.float64(x), 4)


def _limits(ref_iv, test, tol):
    if test == 0:
        return np.full(len(ref_iv), tol["onset_tolerance"])
    return np.maximum(tol["offset_ratio"] * np.abs(np.diff(ref_iv, axis=-1)).flatten(), tol["offset_min_tolerance"])


def kernel_counts(ref_iv, est_iv, tol=TOL):
    """The kernel's steps per test: sort the estimates' tested times, find each reference's run by two binary searches
    with the exact predicate, counting-sort the references by run end, give each the smallest free estimate of its run
    (next-free array, path halving).  -> [n_ref, n_est, onsets matched, offsets matched]."""
    ref_iv, est_iv = np.asarray(ref_iv, np.float64).reshape(-1, 2), np.asarray(est_iv, np.float64).reshape(-1, 2)
    n_ref, n = len(ref_iv), len(est_iv)
    out = [n_ref, n]
    for test in (0, 1):
        if n_ref == 0 or n == 0:
            out.append(0)
            continue
        t = np.sort(est_iv[:, test])
        lim = _limits(ref_iv, test, tol)
        runs = []
        for r in range(n_ref):
            tr = ref_iv[r, test]

            def miss(j):
                return not (_around4(abs(tr - t[j])) <= lim[r])

            a, length = 0, n
            while length > 0:  # lo: estimates before the reference that miss it
                h = length >> 1
                if t[a + h] < tr and miss(a + h):
                    a, length = a + h + 1, length - h - 1
                else:
                    length = h
            lo, length = a, n - a
            while length > 0:  # end: first estimate after the reference that misses it
                h = length >> 1
                if not (t[a + h] > tr and miss(a + h)):
                    a, length = a + h + 1, length - h - 1
                else:
                    length = h
            runs.append((lo, a))
        cnt = [0] * (n + 1)
        for lo, end in runs:
            if lo < end:
                cnt[end] += 1
        s = 0
        for k in range(n + 1):
            cnt[k], s = s, s + cnt[k]
        order = [None] * s
        for r, (lo, end) in enumerate(runs):
            if lo < end:
                order[cnt[end]] = r
                cnt[end] += 1
        nf = list(range(n + 1))
        matched = 0
        for r in order:
            x = runs[r][0]
            while nf[x] != x:
                nf[x] = nf[nf[x]]
                x = nf[x]
            if x < runs[r][1]:
                nf[x] = x + 1
                matched += 1
        out.append(matched)
    return out


def _scipy_size(hits):
    hits = np.asarray(hits, bool)
    if not hits.any():
        return 0
    return int((maximum_bipartite_matching(scipy.sparse.csr_matrix(hits), perm_type="column") >= 0).sum())


# ------------------------------------------------------------------------------------------------ note sets
def _frame_times(n):
    from basic_pitch_b200.note_creation import model_frames_to_time

    return model_frames_to_time(n)


def _random_set(rng, grid, n_max=24, span=1.0):
    """References and estimates with times on `grid` (seconds; None: model frame times), many of them near one
    another so that distances fall on and around the tolerances."""
    nr, ne = (int(x) for x in rng.integers(0, n_max, 2))
    frames = _frame_times(int(span * 90) + 400)

    def snap(x):
        if grid is None:
            return frames[np.clip(np.searchsorted(frames, x), 0, len(frames) - 1)]
        return np.round(x / grid) * grid

    def notes(k, base):
        on = snap(base[rng.integers(0, len(base), k)] + rng.choice([0.0, 0.05, -0.05, 0.0501, 0.04995, 0.1], k)
                  + rng.normal(0, 0.01, k) * rng.integers(0, 2, k))
        on = np.maximum(on, 0.0)
        dur = snap(rng.choice([0.01, 0.1, 0.2, 0.25, 0.2505, 0.2495, 0.5, 1.0], k) + rng.uniform(0, 0.02, k) *
                   rng.integers(0, 2, k))
        off = np.maximum(snap(on + dur), on + (grid or 0.02))
        return np.stack([on, off], 1)

    base = np.maximum(rng.uniform(0, span, 6), 0.0)
    return notes(nr, base), notes(ne, base)


def _boundary_sets():
    """Hand-made adversarial sets: half-even ties from 0 s, just-below-half distances between nonzero times, equal
    times, durations on both sides of offset_min_tolerance / offset_ratio = 0.25 s."""
    sets = []
    z = np.array([[0.0, 1.0]])
    for d in (0.05005, 0.05015, 0.05, 0.0501, 0.04995):
        sets.append((np.array([[d, 1.0 + d]]), z))  # ties from an estimate at 0 s (onsets and offsets)
        sets.append((np.array([[1.0 + d, 2.0 + d], [1.0, 2.0]]), np.array([[1.0, 2.0], [1.0 + 2 * d, 2.0 + 2 * d]])))
    on = np.array([1.05005, 1.05015, 1.0, 1.1, 0.95, 0.94995])
    sets.append((np.stack([on, on + 0.5], 1), np.array([[1.0, 1.5]] * 3)))  # duplicate estimates
    sets.append((np.array([[1.0, 1.5]] * 4), np.array([[1.0, 1.5]] * 2 + [[1.05, 1.55]])))  # equal times
    for dur in (0.2499, 0.25, 0.2501, 0.3, 0.1):
        ref = np.array([[2.0, 2.0 + dur]])
        lim = max(0.2 * dur, 0.05)
        est = np.array([[2.0, 2.0 + dur + lim], [2.0, 2.0 + dur - lim], [2.0, 2.0 + dur + lim + 1e-4]])
        sets.append((ref, est))
    # a chord: one shared onset, offsets apart
    sets.append((np.array([[3.0, 3.5], [3.0, 3.8], [3.0, 4.0]]), np.array([[3.0, 3.52], [3.01, 3.9], [3.02, 3.45]])))
    return sets


def _tolerance_sets():
    return [TOL, dict(onset_tolerance=0.0, offset_ratio=0.0, offset_min_tolerance=0.0),  # zero tolerance
            dict(onset_tolerance=100.0, offset_ratio=0.2, offset_min_tolerance=100.0),  # complete graphs
            dict(onset_tolerance=0.02, offset_ratio=5.0, offset_min_tolerance=0.0)]


def _all_cases():
    rng = np.random.default_rng(2026)
    cases = [(r, e, TOL) for r, e in _boundary_sets()]
    for tol in _tolerance_sets():
        for r, e in _boundary_sets():
            cases.append((r, e, tol))
    for grid in (1e-4, 5e-5, 1e-3, None):
        for k in range(120):
            r, e = _random_set(rng, grid, span=0.3 if k % 2 else 2.0)
            cases.append((r, e, _tolerance_sets()[k % 4] if k % 5 == 0 else TOL))
    return cases


CASES = _all_cases()


# ------------------------------------------------------------------------------------------------ tests
def test_oracle_matching_is_maximum_on_random_graphs():
    """The restated mir_eval matching has SciPy's maximum size on > 1 000 random graphs (dense, sparse, skewed) and on
    the hit matrices of every case below."""
    rng = np.random.default_rng(5)
    n = 0
    for _ in range(1100):
        nr, ne = (int(x) for x in rng.integers(0, 14, 2))
        hits = rng.random((nr, ne)) < rng.choice([0.05, 0.2, 0.5, 0.9])
        assert len(oo.match_hits(hits)) == _scipy_size(hits)
        n += 1
    for ref, est, tol in CASES[::3]:
        for hits in (oo.onset_hits(ref, est, tol["onset_tolerance"]),
                     oo.offset_hits(ref, est, tol["offset_ratio"], tol["offset_min_tolerance"])):
            assert len(oo.match_hits(hits)) == _scipy_size(hits)
            n += 1
    assert n > 1000


def test_rounding_boundary_facts():
    """From an estimate at 0 s, 0.05005 and 0.05015 s are exact half-even ties (a hit, then a miss); between nonzero
    times the same distances land just below the half and round down."""
    z = np.array([[0.0, 1.0]])
    assert oo.onset_hits([[0.05005, 1.0]], z)[0, 0] and not oo.onset_hits([[0.05015, 1.0]], z)[0, 0]
    assert 0.05005 * 10000 == 500.5 and 0.05015 * 10000 == 501.5
    assert (1.05005 - 1.0) * 10000 < 500.5 and (1.05015 - 1.0) * 10000 < 501.5
    one = np.array([[1.0, 2.0]])
    assert oo.onset_hits([[1.05005, 2.0]], one)[0, 0]
    assert not oo.onset_hits([[1.05015, 2.0]], one)[0, 0]
    assert oo.onset_hits([[1.05015, 2.0]], one, 0.0501)[0, 0]


def test_every_row_is_one_contiguous_run_in_sorted_estimate_order():
    n_rows = n_gaps = 0
    for ref, est, tol in CASES:
        ref, est = np.asarray(ref).reshape(-1, 2), np.asarray(est).reshape(-1, 2)
        for test, hits in ((0, oo.onset_hits(ref, est, tol["onset_tolerance"])),
                           (1, oo.offset_hits(ref, est, tol["offset_ratio"], tol["offset_min_tolerance"]))):
            order = np.argsort(est[:, test], kind="stable")
            for row in hits[:, order]:
                nz = np.flatnonzero(row)
                n_rows += 1
                if len(nz):
                    assert nz[-1] - nz[0] + 1 == len(nz), (ref, est, tol, test)
                    n_gaps += len(nz) < len(row)
    assert n_rows > 3000 and n_gaps > 500  # runs that are not the whole row are common


def test_kernel_model_equals_the_oracle():
    partial = 0
    for ref, est, tol in CASES:
        exp = oo.counts(ref, est, **tol)
        assert kernel_counts(ref, est, tol) == exp, (ref, est, tol)
        partial += 0 < min(exp[2:]) and max(exp[2:]) < min(exp[:2])
    assert partial > 50


def test_greedy_by_run_end_beats_input_order():
    """Offsets: a long reference listed first covers both estimates, a short one only the first.  Taking references in
    input order loses a pair; the kernel's order by run end does not."""
    ref = np.array([[0.0, 1.15], [0.9, 1.0]])  # limits 0.23 and 0.05
    est = np.array([[0.5, 1.0], [0.6, 1.3]])
    hits = oo.offset_hits(ref, est)
    assert hits.tolist() == [[True, True], [True, False]]
    taken, n_input_order = set(), 0
    for r in range(2):  # input order, smallest free estimate of the run
        free = [j for j in np.flatnonzero(hits[r]) if j not in taken]
        if free:
            taken.add(free[0])
            n_input_order += 1
    assert n_input_order == 1
    assert kernel_counts(ref, est)[3] == 2 == oo.counts(ref, est)[3]


def test_onset_offset_scores_hand_values():
    from basic_pitch_b200.evaluate import ONSET_OFFSET_FIELDS, onset_offset_scores

    assert ONSET_OFFSET_FIELDS == ("n_ref", "n_est", "onset_matched", "offset_matched")
    c = np.array([[10, 8, 4, 2], [0, 5, 0, 0], [3, 0, 0, 0], [4, 4, 0, 0], [4, 4, 4, 4]])
    s = onset_offset_scores(c)
    assert list(s) == ["onset_precision", "onset_recall", "onset_f_measure", "offset_precision", "offset_recall",
                       "offset_f_measure", "mean"]
    assert s["onset_precision"].tolist() == [0.5, 0.0, 0.0, 0.0, 1.0]
    assert s["onset_recall"].tolist() == [0.4, 0.0, 0.0, 0.0, 1.0]
    assert s["onset_f_measure"].tolist() == [2 * 0.5 * 0.4 / 0.9, 0.0, 0.0, 0.0, 1.0]
    assert s["offset_precision"].tolist() == [0.25, 0.0, 0.0, 0.0, 1.0]
    assert s["offset_recall"].tolist() == [0.2, 0.0, 0.0, 0.0, 1.0]
    assert s["offset_f_measure"].tolist() == [2 * 0.25 * 0.2 / 0.45, 0.0, 0.0, 0.0, 1.0]
    assert s["mean"]["onset_recall"] == np.mean([0.4, 0.0, 0.0, 0.0, 1.0])
    g = onset_offset_scores(c[:4].reshape(2, 2, 4))
    assert g["offset_precision"].shape == (2, 2) and g["mean"]["onset_precision"].tolist() == [0.25, 0.0]
    assert onset_offset_scores(np.zeros((3, 0, 4), np.int64))["mean"]["onset_f_measure"].tolist() == [0.0] * 3
    with pytest.raises(ValueError):
        onset_offset_scores(np.zeros((2, 6)))


def test_onset_offset_scores_equal_the_oracle_bit_for_bit():
    from basic_pitch_b200.evaluate import onset_offset_scores

    for ref, est, tol in CASES[::7]:
        s = onset_offset_scores(oo.counts(ref, est, **tol))
        on = oo.onset_precision_recall_f1(ref, est, tol["onset_tolerance"])
        off = oo.offset_precision_recall_f1(ref, est, tol["offset_ratio"], tol["offset_min_tolerance"])
        assert (s["onset_precision"], s["onset_recall"], s["onset_f_measure"]) == on
        assert (s["offset_precision"], s["offset_recall"], s["offset_f_measure"]) == off


def test_transcription_keys_are_mir_evals_in_order():
    from basic_pitch_b200.evaluate import TRANSCRIPTION_KEYS

    names = ["Precision", "Recall", "F-measure", "Average_Overlap_Ratio", "Precision_no_offset", "Recall_no_offset",
             "F-measure_no_offset", "Average_Overlap_Ratio_no_offset", "Onset_Precision", "Onset_Recall",
             "Onset_F-measure", "Offset_Precision", "Offset_Recall", "Offset_F-measure"]
    assert list(TRANSCRIPTION_KEYS) == names
    assert list(TRANSCRIPTION_KEYS.values()) == [n.lower().replace("-", "_") for n in names]
    ref, est = np.array([[0.0, 1.0], [1.0, 2.0]]), np.array([[0.01, 0.9]])
    assert list(oo.evaluate(ref, [440.0, 440.0], est, [440.0])) == names
