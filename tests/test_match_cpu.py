"""CPU: mir_eval 0.7's note matching restated in oracle/note_matching_ref.py (the reference for bp_match_*), and
evaluate.matching_scores, on graphs and note sets whose expected pairs and scores are derived by hand."""
import numpy as np
import pytest
import scipy.sparse
from scipy.sparse.csgraph import maximum_bipartite_matching

from oracle import note_matching_ref as nm
from oracle import transcription_ref as tr


def _check_matching(hits, matching):
    used = set()
    for v, u in matching.items():
        assert hits[v, u], (v, u)
        assert u not in used
        used.add(u)


def _scipy_size(hits):
    if not hits.any():
        return 0
    return int((maximum_bipartite_matching(scipy.sparse.csr_matrix(hits), perm_type="column") >= 0).sum())


def test_matching_is_maximum_on_random_graphs():
    """>= 1000 graphs: sparse, dense, with empty rows and columns, one side much larger than the other."""
    rng = np.random.default_rng(0)
    shapes = [(n, m) for n in (1, 2, 3, 5, 8, 13) for m in (1, 2, 3, 5, 8, 13)] + [(1, 40), (40, 1), (3, 60), (60, 3),
                                                                                  (50, 50), (100, 7), (7, 100)]
    n_graphs = 0
    for density in (0.02, 0.1, 0.3, 0.6, 0.95):
        for n_ref, n_est in shapes:
            for _ in range(5):
                hits = rng.random((n_ref, n_est)) < density
                if rng.random() < 0.3:
                    hits[rng.integers(0, n_ref)] = False  # an empty row
                    hits[:, rng.integers(0, n_est)] = False  # an empty column
                matching = nm.bipartite_match(nm.match_graph(hits))
                _check_matching(hits, matching)
                assert len(matching) == _scipy_size(hits), (density, n_ref, n_est)
                n_graphs += 1
    assert n_graphs >= 1000


def _hits(n_ref, n_est, edges):
    h = np.zeros((n_ref, n_est), bool)
    for r, e in edges:
        h[r, e] = True
    return h


def test_two_maximum_matchings_the_augmenting_path_decides():
    """G = {0: [0, 1], 1: [0]}: the greedy pass gives reference 0 to estimate 0 and leaves estimate 1 free; the one
    augmenting path 1 - r0 - 0 - r1 moves estimate 0 to reference 1."""
    assert nm.bipartite_match({0: [0, 1], 1: [0]}) == {0: 1, 1: 0}
    G = nm.match_graph(_hits(2, 2, [(0, 0), (0, 1), (1, 0)]))
    assert list(G.items()) == [(0, [0, 1]), (1, [0])]
    assert nm.bipartite_match(G) == {0: 1, 1: 0}


def test_key_order_is_set_by_the_first_hitting_reference():
    """Reference 0 hits estimates 1 and 2, reference 1 hits estimates 0 and 2.  Keys come in the order 1, 2, 0 (first
    reference 0, 0, 1): greedy gives r0 to 1 and r1 to 2, estimate 0 is left without an augmenting path, so the result
    is {0: 1, 1: 2}.  Keys in estimate order would give {0: 1, 1: 0}."""
    G = nm.match_graph(_hits(2, 3, [(0, 1), (0, 2), (1, 0), (1, 2)]))
    assert list(G) == [1, 2, 0] and G == {1: [0], 2: [0, 1], 0: [1]}
    assert nm.bipartite_match(G) == {0: 1, 1: 2}
    assert nm.bipartite_match({0: [1], 1: [0], 2: [0, 1]}) == {0: 1, 1: 0}


def _chains(lengths):
    """Components with augmenting paths of 2k + 1 edges: references r_0 .. r_k, estimates x_1 (index e), y (e + 1) and
    x_i (e + i) for i >= 2; x_i hits r_i-1 and r_i, y hits r_0.  Greedy: x_1 takes r_0, x_i takes r_i-1, y stays free.
    The only maximum matching gives r_0 to y and r_i to x_i."""
    edges, expect = [], {}
    rb = eb = 0
    for k in lengths:
        x = {1: eb, **{i: eb + i for i in range(2, k + 1)}}
        y = eb + 1
        edges.append((rb, y))
        for i in range(1, k + 1):
            edges += [(rb + i - 1, x[i]), (rb + i, x[i])]
            expect[rb + i] = x[i]
        expect[rb] = y
        rb += k + 1
        eb += k + 1
    return _hits(rb, eb, edges), expect


def test_components_that_need_three_phases():
    """Paths of 3, 5 and 7 edges: each phase augments along the shortest paths only, so the three components take three
    phases."""
    hits, expect = _chains([1, 2, 3])
    stats = {}
    assert nm.bipartite_match(nm.match_graph(hits), stats) == expect
    assert stats["phases"] == 3


def test_a_recursion_falls_back_after_a_dead_branch():
    """References z=0, c=1, a=2, b=3, y=4, v=5; estimates mD=0 {z}, mA=1 {z, a, v}, mC=2 {c, y}, f1=3 {c, a}, mB=4 {b, v},
    f2=5 {b}.  Keys mD, mA, mC, f1, mB, f2; greedy: z-mD, a-mA, c-mC, b-mB; f1 and f2 free.  Layers: {f1, f2}, then
    c, a, b, then mC, mA, mB, then y [mC], z [mA], v [mA, mB] with y and v unmatched.  recurse(y) takes mC, c and f1;
    recurse(v) tries mA first: a's only predecessor f1 is gone, a dead branch; mB, b and f2 then succeed."""
    hits = _hits(6, 6, [(0, 0), (0, 1), (1, 2), (1, 3), (2, 1), (2, 3), (3, 4), (3, 5), (4, 2), (5, 1), (5, 4)])
    G = nm.match_graph(hits)
    assert G == {0: [0], 1: [0, 2, 5], 2: [1, 4], 3: [1, 2], 4: [3, 5], 5: [3]} and list(G) == [0, 1, 2, 3, 4, 5]
    stats = {}
    assert nm.bipartite_match(G, stats) == {0: 0, 1: 3, 2: 1, 3: 5, 4: 2, 5: 4}
    assert stats["phases"] == 1 and stats["dead"] == 1


# ------------------------------------------------------------------------------------------------ matching_scores
def test_scores_of_a_single_matched_pair():
    """References v = (20, 100) -> (0, 1); reference 1 matched to estimate 0 (v = 50).  lstsq's minimum-norm solution of
    50 s + i = 1 is (50, 1) / 2501, which maps 50 to 1: the pair is kept.  P = 1, R = 1/2, F = 2/3; the overlap ratio
    of [1, 2] and [1.2, 2.5] is 0.8 / 1.5."""
    from basic_pitch_b200.evaluate import matching_scores

    s = matching_scores([[0.0, 0.5], [1.0, 2.0]], [20, 100], [[1.2, 2.5]], [50], np.array([[-1, 0], [-1, 0]]))
    for suffix in ("", "_no_offset"):
        assert s["velocity_precision" + suffix] == 1.0 and s["velocity_recall" + suffix] == 0.5
        assert s["velocity_f_measure" + suffix] == 2 * 1.0 * 0.5 / 1.5
        assert s["average_overlap_ratio" + suffix] == (2.0 - 1.2) / (2.5 - 1.0)
        assert s["velocity_average_overlap_ratio" + suffix] == (2.0 - 1.2) / (2.5 - 1.0)
    slope, intercept = np.linalg.lstsq(np.array([[50.0, 1.0]]), np.array([1.0]))[0]
    assert slope == pytest.approx(50 / 2501, rel=1e-12) and intercept == pytest.approx(1 / 2501, rel=1e-12)


def _four():
    iv = np.array([[0.0, 1.0], [1.0, 2.0], [2.0, 3.0], [3.0, 4.0]])
    return iv, np.array([0, 50, 100, 60]), iv + 0.01, np.full(4, 70), np.array([[0, 1, 2, 3], [0, 1, 2, 3]])


def test_scores_with_equal_estimate_velocities():
    """Every estimate velocity 70: the system is rank-deficient and the minimum-norm fit is the mean of the normalised
    reference velocities (0, 0.5, 1, 0.6), 0.525.  Differences 0.525, 0.025, 0.475, 0.075: pairs 1 and 3 are kept."""
    from basic_pitch_b200.evaluate import matching_scores

    ref_iv, rv, est_iv, ev, m = _four()
    s = matching_scores(ref_iv, rv, est_iv, ev, m)
    assert s["velocity_precision"] == 0.5 and s["velocity_recall"] == 0.5 and s["velocity_f_measure"] == 0.5
    ratio = (1.0 - 0.01) / (1.01 - 0.0)
    assert s["average_overlap_ratio"] == pytest.approx(ratio, rel=1e-12)
    assert s["velocity_average_overlap_ratio"] == pytest.approx(ratio, rel=1e-12)


def test_a_difference_exactly_at_the_tolerance_is_dropped():
    """The strict < of mir_eval: with the tolerance set to pair 3's difference itself, pair 3 goes; one ulp above, it
    stays."""
    from basic_pitch_b200.evaluate import matching_scores

    ref_iv, rv, est_iv, ev, m = _four()
    rn = (rv - rv.min()) / float(max(1, rv.max() - rv.min()))
    slope, intercept = np.linalg.lstsq(np.vstack([ev, np.ones(4)]).T, rn)[0]
    tol = float(np.abs(slope * ev + intercept - rn)[3])
    assert tol == pytest.approx(0.075, abs=1e-12)
    assert matching_scores(ref_iv, rv, est_iv, ev, m, velocity_tolerance=tol)["velocity_precision"] == 0.25
    assert matching_scores(ref_iv, rv, est_iv, ev, m, velocity_tolerance=np.nextafter(tol, 1.0))["velocity_precision"] == 0.5


def test_equal_reference_velocities_use_a_range_of_one():
    """All references 64: max(1, 0) = 1 normalises them to 0; the fit to zeros is exactly zero, every pair is kept."""
    from basic_pitch_b200.evaluate import matching_scores

    ref_iv, _, est_iv, _, m = _four()
    s = matching_scores(ref_iv, [64] * 4, est_iv, [10, 30, 90, 127], m)
    assert s["velocity_f_measure"] == 1.0 and s["velocity_f_measure_no_offset"] == 1.0


def test_empty_sides_and_unmatched():
    from basic_pitch_b200.evaluate import MATCH_FIELDS, matching_scores

    one = np.array([[0.0, 1.0]])
    for args in ((np.zeros((0, 2)), [], one, [3], np.zeros((2, 0), int)), (one, [3], np.zeros((0, 2)), [], [[-1], [-1]]),
                 (one, [3], one, [3], [[-1], [-1]])):
        s = matching_scores(*args)
        assert all(s[k] == 0.0 and s[k + "_no_offset"] == 0.0 for k in MATCH_FIELDS)
    with pytest.raises(ValueError, match="references note 1"):
        matching_scores([[0, 1], [1, 2]], [3, np.nan], one, [3], [[-1, 0], [-1, 0]])
    with pytest.raises(ValueError, match="estimates note 0"):
        matching_scores(one, [3], one, [-1], [[0], [0]])


def test_the_matching_shows_in_the_velocity_scores():
    """References r0, r1 = [1, 2] and r2 = [3, 4] at 440 Hz, velocities (10, 100, 40) -> (0, 1, 1/3); estimates e0, e1 at
    [1.01, 2] and e2 at [3, 4], velocities (20, 90, 45).  r0 and r1 both hit e0 and e1: mir_eval's greedy pass gives
    r0-e0, r1-e1, on the line v / 70 - 2 / 7 up to 1/42 at e2, so every pair is kept (F = 1).  The other maximum
    matching, r0-e1, r1-e0, fits badly and keeps one pair (F = 1/3)."""
    from basic_pitch_b200.evaluate import matching_scores

    ref_iv = np.array([[1.0, 2.0], [1.0, 2.0], [3.0, 4.0]])
    est_iv = np.array([[1.01, 2.0], [1.01, 2.0], [3.0, 4.0]])
    l2 = np.full(3, np.log2(440.0))
    rv, ev = np.array([10, 100, 40]), np.array([20, 90, 45])
    for with_offsets in (False, True):
        assert nm.match_notes(ref_iv, l2, est_iv, l2, with_offsets) == [(0, 0), (1, 1), (2, 2)]
    got = matching_scores(ref_iv, rv, est_iv, ev, np.array([[0, 1, 2], [0, 1, 2]]))
    other = matching_scores(ref_iv, rv, est_iv, ev, np.array([[1, 0, 2], [1, 0, 2]]))
    assert got["velocity_f_measure"] == 1.0 and other["velocity_f_measure"] == pytest.approx(1 / 3)
    p, r, f, aor = nm.velocity_scores(ref_iv, rv, est_iv, ev, [(0, 0), (1, 1), (2, 2)])
    assert (got["velocity_precision"], got["velocity_recall"], got["velocity_f_measure"],
            got["velocity_average_overlap_ratio"]) == (p, r, f, aor)


def test_matching_scores_equal_the_restatement_on_random_files():
    """matching_scores (vectorised) against the plain restatement of mir_eval, bit for bit, on random note sets."""
    from basic_pitch_b200.evaluate import matching_scores

    rng = np.random.default_rng(5)
    for _ in range(200):
        n_ref, n_est = rng.integers(0, 25, 2)

        def notes(n):
            on = np.round(rng.uniform(0, 3, n), 2)
            return np.stack([on, on + np.round(rng.uniform(0.05, 1.0, n), 2)], 1), np.log2(440.0) + rng.integers(-2, 3, n) / 12
        ref_iv, ref_l2 = notes(n_ref)
        est_iv, est_l2 = notes(n_est)
        rv = rng.integers(0, 128, n_ref) if rng.random() < 0.8 else np.full(n_ref, 50)
        ev = rng.integers(0, 128, n_est)
        pairs = [nm.match_notes(ref_iv, ref_l2, est_iv, est_l2, w) for w in (False, True)]
        m = np.stack([nm.match_array(p, n_ref) for p in pairs])
        got = matching_scores(ref_iv, rv, est_iv, ev, m)
        for suffix, p in (("_no_offset", pairs[0]), ("", pairs[1])):
            aor = 0.0 if n_ref == 0 or n_est == 0 else nm.average_overlap_ratio(ref_iv, est_iv, p)
            assert got["average_overlap_ratio" + suffix] == aor
            exp = nm.velocity_scores(ref_iv, rv, est_iv, ev, p)
            assert tuple(got[k + suffix] for k in ("velocity_precision", "velocity_recall", "velocity_f_measure",
                                                   "velocity_average_overlap_ratio")) == exp
        assert (m[1] >= 0).sum() == tr.counts(ref_iv, 2.0**ref_l2, est_iv, 2.0**est_l2)[3] if n_ref and n_est else True
