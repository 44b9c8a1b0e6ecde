"""CPU: the adversarial melody sets of tests/melodysets.py reach the edges they are built for (liveness), and the
comparison they feed has teeth: each mutant below restates one rule of include/bp_b200.h (bp_score_melody_grid_*,
bp_score_note_melody_grid_*, rules 1 to 4) with one slip a kernel could make, and its counts differ from the
oracle's on the sets.

The restatement `score` (rules 1 to 4 on cents and voicing, with scipy.interpolate.interp1d as oracle/melody_ref.py)
and `bins` (the arg-max of a bin range) can record what they saw and can be mutated; unmutated they equal
oracle/melody_ref.counts_cents applied to the host definition (melodysets.estimate, which equals
evaluate.salience_to_melody on the model's tables)."""
import numpy as np
import pytest
import scipy.interpolate

from oracle import melody_ref as mr
from tests import melodysets as ms

MUTANTS = ("highest_bin", "lowest_lane", "nan_wins", "gt_threshold", "f32_threshold", "tol_le", "octave_half_down",
           "tile_reset", "appended_voiced", "no_identity", "hi_inclusive")
# At d = 1200 n + 600 exactly both octaves are 600 cents away, and d / 1200 + 0.5 is an integer only there: rounding
# the octave half down gives the same |d - octave| for every float64 d.  The mutant is kept to show that the tie is
# reached (liveness) and that no count can tell it apart, rather than silently dropped.
EQUIVALENT = ("octave_half_down",)


# ------------------------------------------------------------------------------------------------ restatement
def bins(g, lo, hi, mut=()):
    """b* of every row of a file under the range [lo, hi) (-1: none), rule of bp_score_melody_grid_* or a mutant."""
    W = g.shape[1]
    if "hi_inclusive" in mut:
        hi = min(hi + 1, W)
    out = np.full(g.shape[0], -1, np.int64)
    if hi <= lo or g.shape[0] == 0:
        return out
    sub = g[:, lo:hi]
    if "nan_wins" in mut:  # np.argmax: the first NaN, else the first maximum
        return lo + np.argmax(sub, axis=1)
    ok = ~np.isnan(sub).all(axis=1)
    with np.errstate(invalid="ignore"):
        best = np.where(ok, np.nanmax(np.where(ok[:, None], sub, 0), axis=1), 0)
    tie = (sub == best[:, None]) & ok[:, None]
    idx = np.arange(hi - lo)
    if "highest_bin" in mut:
        b = (hi - lo - 1) - np.argmax(tie[:, ::-1], axis=1)
    elif "lowest_lane" in mut:  # a shuffle reduction keeping the lowest lane of a tie, lane = (b - lo) % 32
        key = np.where(tie, (idx % 32) * 4096 + idx, 1 << 30)
        b = idx[np.argmin(key, axis=1)]
    else:
        b = np.argmax(tie, axis=1)
    out[ok] = lo + b[ok]
    return out


def estimate(g, tab, p, mut=(), b=None):
    thr, lo, hi, guess = p
    if b is None:
        b = bins(g, lo, hi, mut)
    ok = b >= 0
    v = np.zeros(len(b), bool)
    cell = g[np.flatnonzero(ok), b[ok]]
    if "gt_threshold" in mut:
        v[ok] = cell.astype(np.float64) > thr
    elif "f32_threshold" in mut:
        v[ok] = cell >= np.float32(thr)
    else:
        v[ok] = cell.astype(np.float64) >= thr
    c = np.where(ok & (v | bool(guess)), tab[np.maximum(b, 0)], 0.0)
    return c, v.astype(np.int32)


def _rule1(t, *vals):
    if len(t) and t[0] > 0:
        return (np.insert(t, 0, 0.0),) + tuple(np.insert(v, 0, v[0]) for v in vals)
    return (t,) + vals


def score(ref, est_t, est_c, est_v, tol, mut=(), trace=None):
    """The seven counts of rule 4 for one (setting, file): ref (times, cents, voiced), the estimate's frame times,
    cents and voicing.  trace (a dict) receives the reference frames as the estimate reads them."""
    rt, rc, rv = _rule1(*(np.asarray(a, np.float64) for a in ref))
    et, c, v = _rule1(*(np.asarray(a, np.float64) for a in (est_t, est_c, est_v)))
    K, n = len(rt), len(et)
    ec, ev = np.zeros(K), np.zeros(K)
    if n and K:
        ident = n == K and np.allclose(et, rt) and "no_identity" not in mut
        if ident:
            ec, ev = c.copy(), v.copy()
        else:
            e, x = np.round(et, 10), np.round(rt, 10)
            app = x.max() > e.max()
            if app:
                e = np.append(e, x.max())
                c = np.append(c, 0.0)
                v = np.append(v, v[-1] if "appended_voiced" in mut else 0.0)
            held = c.copy()
            for k in range(1, len(held)):
                if held[k] == 0 and not ("tile_reset" in mut and k % 32 == 0 and k < n):
                    held[k] = held[k - 1]
            zero = scipy.interpolate.interp1d(e, c, "zero")(x)
            ec = scipy.interpolate.interp1d(e, held, "linear")(x) * (zero != 0)
            ev = scipy.interpolate.interp1d(e, v, "zero")(x)
            if trace is not None:
                j = np.searchsorted(e, x, "right") - 1
                trace.setdefault("read", []).append(dict(x=x, raw_x=rt, e=e, raw_e=et, c=c, j=j, n=n, app=app))
        if trace is not None:
            trace.setdefault("ident", []).append(ident)
    rvb, evb = rv > 0, ev > 0
    nz = (ec != 0) & (rc != 0)
    d = np.abs(rc - ec)
    if "octave_half_down" in mut:
        octave = 1200.0 * np.ceil(d / 1200 - 0.5)
    else:
        octave = 1200.0 * np.floor(d / 1200 + 0.5)
    lt = (lambda a: a <= tol) if "tol_le" in mut else (lambda a: a < tol)
    pitch = nz & rvb & lt(d)
    chroma = nz & rvb & lt(np.abs(d - octave))
    if trace is not None:
        trace.setdefault("d", []).append(d[nz & rvb])
    return [K, int(rvb.sum()), int((rvb & evb).sum()), int((~rvb & evb).sum()), int(pitch.sum()), int(chroma.sum()),
            int((pitch & evb).sum())]


def set_counts(s, tol, mut=(), trace=None):
    """(settings, files, 7) counts of a grid set under the restatement, the arg-max once per (file, distinct range)."""
    out = np.zeros((len(s.params), len(s.grams), 7), np.int64)
    for i, g in enumerate(s.grams):
        ft = ms.frame_times(g.shape[0])
        cache = {}
        for k, p in enumerate(s.params):
            r = (p[1], p[2])
            if r not in cache:
                cache[r] = bins(g, *r, mut)
            c, v = estimate(g, s.cents, p, mut, cache[r])
            out[k, i] = score(s.refs[i], ft, c, v, tol, mut, trace)
    return out


def oracle_counts(s, tol):
    """oracle/melody_ref.counts_cents on the host definition of every (setting, file)."""
    out = np.zeros((len(s.params), len(s.grams), 7), np.int64)
    for i, g in enumerate(s.grams):
        ft = ms.frame_times(g.shape[0])
        t, rc, rv = s.refs[i]
        for k, p in enumerate(s.params):
            c, v = ms.estimate(g, s.cents, p)
            out[k, i] = mr.counts_cents(t, rc, rv, ft, c, v, tol)
    return out


_EXP = {}


def expected(name, tol):
    if (name, tol) not in _EXP:
        _EXP[name, tol] = oracle_counts(ms.get(name), tol)
    return _EXP[name, tol]


# ------------------------------------------------------------------------------------------------ oracle entry
def test_counts_cents_equals_counts_on_random_pairs():
    from basic_pitch_b200.evaluate import melody_values
    from tests.test_melody_cpu import _random_pair

    rng = np.random.default_rng(11)
    for case in range(200):
        ref_t, ref_hz, est_t, est_hz = _random_pair(rng, case)
        rc, rv = melody_values(ref_hz)
        ec, ev = melody_values(est_hz)
        for tol in (50.0, 1.0):
            assert mr.counts_cents(ref_t, rc, rv, est_t, ec, ev, tol) == mr.counts(ref_t, ref_hz, est_t, est_hz, tol)
    assert mr.counts_cents([0.1, 0.2], [2000.0, 0.0], [1, 0], [], [], []) == [3, 2, 0, 0, 0, 0, 0]


# ------------------------------------------------------------------------------------------------ the sets
@pytest.mark.parametrize("name", ms.NAMES)
def test_sets_are_valid_inputs(name):
    """What bp_score_melody_grid_* validate before any launch (include/bp_b200.h): the reference times through
    bp_melody_map (the library's own check, estimate = the file's model frame times), the rest restated."""
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    s = ms.get(name)
    W = len(s.cents)
    assert np.isfinite(s.cents).all() and (np.diff(s.cents) >= 0).all() and 1 <= W <= 1024
    for thr, lo, hi, g in s.params:
        assert np.isfinite(thr) and thr > 0 and 0 <= lo <= hi <= W and g in (0, 1)
    assert [g.shape[0] for g in s.grams] == list(ms.LENGTHS)
    for g, (t, c, v) in zip(s.grams, s.refs):
        assert g.dtype == np.float32 and g.shape[1] == W
        assert np.isfinite(c).all() and set(np.unique(v)) <= {0, 1} and not (v[c == 0] != 0).any()
        ft = ms.frame_times(g.shape[0])
        K = len(t) + int(len(t) > 0 and t[0] > 0)
        ot, oi = np.zeros((max(K, 1), 3)), np.zeros((max(K, 1), 3), np.int64)
        t = np.ascontiguousarray(t, np.float64)
        assert lib.bp_melody_map(ft.ctypes.data, len(ft), t.ctypes.data, len(t), ot.ctypes.data, oi.ctypes.data) == 0
    if s.kind:
        from basic_pitch_b200.evaluate import melody_values

        for (t, hz), (t2, c, v) in zip(s.ref_hz, s.refs):
            mc, mv = melody_values(hz)
            assert t is t2 and mc.tobytes() == c.tobytes() and (mv == v).all()


@pytest.mark.parametrize("name", ["contour", "note"])
def test_host_definitions_agree(name):
    """On the model's tables the set's estimate is evaluate.salience_to_melody's, through the Hz settings that
    Model.score_melody_grid takes (their bin ranges are the set's)."""
    from basic_pitch_b200.evaluate import melody_values, salience_bin_range, salience_to_melody

    s = ms.get(name)
    hs = ms.hz_settings(s)
    for p, h in zip(s.params, hs):
        lo, hi = salience_bin_range(name, h.get("minimum_frequency"), h.get("maximum_frequency"))
        assert (lo, hi) == (p[1], p[2]) or (hi == lo and p[1] == p[2]), (p, h)
    for g in s.grams:
        for p, h in zip(s.params[::3], hs[::3]):
            c, v = ms.estimate(g, s.cents, p)
            _, f = salience_to_melody(g, kind=name, **h)
            mc, mv = melody_values(f)
            assert mc.tobytes() == c.tobytes() and (mv == v).all()


@pytest.mark.parametrize("name", ms.NAMES)
def test_restatement_equals_the_oracle(name):
    s = ms.get(name)
    for p in s.params[:4]:
        for g in s.grams:
            assert ms.argmax_bins(g, p[1], p[2]).tobytes() == bins(g, p[1], p[2]).tobytes()
    for tol in ms.TOLS:
        np.testing.assert_array_equal(set_counts(s, tol), expected(name, tol), err_msg=f"{name} {tol}")


def _lane(b, lo):
    return (b - lo) % 32


def test_sets_reach_the_arg_max_edges():
    seen = set()
    for name in ms.NAMES:
        s = ms.get(name)
        W = len(s.cents)
        for g in s.grams:
            for lo, hi in {(p[1], p[2]) for p in s.params}:
                if hi <= lo:
                    continue
                b = ms.argmax_bins(g, lo, hi)
                for t in range(g.shape[0]):
                    sub = g[t, lo:hi]
                    if b[t] < 0:
                        seen.add("nan_row" if np.isnan(g[t]).all() else "nan_in_range_only")
                        continue
                    best = g[t, b[t]]
                    tied = lo + np.flatnonzero(sub == best)
                    if len(tied) > 1:
                        lanes = _lane(tied, lo)
                        if len(set(lanes)) > 1:
                            seen.add("cross_lane_lower_bin_higher_lane" if _lane(b[t], lo) > lanes.min() else
                                     "cross_lane_lower_bin_lower_lane")
                        if any((tied - tied[0]) % 32 == 0):
                            seen.add("same_lane")
                        if tied[0] == lo and tied[-1] == hi - 1:
                            seen.add("tie_on_both_ends")
                        if len(tied) == hi - lo and hi - lo > 32:
                            seen.add("plateau")
                        if best == 0 and len(set(np.signbit(g[t, tied]))) == 2:
                            seen.add("signed_zero_tie")
                        if best == -np.inf:
                            seen.add("neg_inf_tie")
                    if (hi < W and g[t, hi] > best) or (lo > 0 and g[t, lo - 1] > best):
                        seen.add("larger_just_outside")
                    if np.isnan(sub).any():
                        seen.add("nan_beside_a_maximum")
                        if np.isnan(sub).sum() >= hi - lo - (hi - lo + 31) // 32 and hi - lo > 32:
                            seen.add("nan_in_all_lanes_but_one")
                        if any(np.isnan(g[t, c]) for c in range(lo, b[t])):
                            seen.add("nan_below_the_winner")
            for thr in ms.THRESHOLDS:
                if (g.astype(np.float64) == thr).any():
                    seen.add("cell_equals_threshold")
                if thr != float(np.float32(thr)) and (g == np.float32(thr)).any():
                    seen.add("threshold_rounds_to_a_cell")
    need = {"nan_row", "nan_in_range_only", "cross_lane_lower_bin_higher_lane", "cross_lane_lower_bin_lower_lane",
            "same_lane", "tie_on_both_ends", "plateau", "signed_zero_tie", "neg_inf_tie", "larger_just_outside",
            "nan_beside_a_maximum", "nan_in_all_lanes_but_one", "nan_below_the_winner", "cell_equals_threshold",
            "threshold_rounds_to_a_cell"}
    assert need <= seen, need - seen


def test_sets_reach_the_map_and_count_edges():
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    seen = set()
    counts = set()
    for name in ms.NAMES:
        s = ms.get(name)
        K = 0
        for i, (g, ref) in enumerate(zip(s.grams, s.refs)):
            t = ref[0]
            K += len(t) + int(len(t) > 0 and t[0] > 0)
            counts.add(len(t))
            if len(t) and t[0] > 0:
                seen.add("first_time_after_0")
            if len(t) and (np.diff(t) == 0).any():
                seen.add("duplicated_times")
            if len(t) and not ref[2].any():
                seen.add("wholly_unvoiced")
            T = g.shape[0]
            ft = ms.frame_times(T)
            if T and len(t):
                Km = len(t) + int(t[0] > 0)
                ot, oi = np.zeros((Km, 3)), np.zeros((Km, 3), np.int64)
                tt = np.ascontiguousarray(t, np.float64)
                lib.bp_melody_map(ft.ctypes.data, T, tt.ctypes.data, len(tt), ot.ctypes.data, oi.ctypes.data)
                base = ms.BASES[T]
                if base in ("identity", "near") and len(t) == T:
                    assert oi[:, 2].all(), (name, T)
                    seen.add(f"identity_{base}")
                if base in ("off", "far"):
                    assert not oi[:, 2].any(), (name, T)
                    seen.add(f"resampled_{base}")
            # the estimate under the first setting, read at the reference frames
            if T:
                tr = {}
                c, v = ms.estimate(g, s.cents, s.params[0])
                score(ref, ft, c, v, 50.0, trace=tr)
                for rd in tr.get("read", []):
                    x, e, cc, j, n = rd["x"], rd["e"], rd["c"], rd["j"], rd["n"]
                    if rd["app"]:
                        seen.add("appended_sample")
                        if (x == e[-1]).sum() >= 2:
                            seen.add("largest_reference_twice")
                    for k in range(len(x)):
                        jj = j[k]
                        knot = e[jj] == x[k]
                        if knot and rd["raw_x"][k] != rd["raw_e"][min(jj, n - 1)] and jj < n:
                            seen.add("knot_after_rounding")
                        elif knot:
                            seen.add("knot")
                        if not knot and jj + 1 < n and jj % 32 == 31 and cc[jj] != 0 and cc[jj + 1] == 0:
                            seen.add("between_lane_31_voiced_and_lane_0_zero")
                        if not knot and jj == 171 and jj + 1 < n:
                            seen.add("inside_the_window_step")
                        if not knot and jj == 343 and jj + 1 < n:
                            seen.add("inside_the_second_window_step")
        if (len(s.params) * K) % 32:
            seen.add("settings_times_frames_not_a_multiple_of_32")
        assert K % 32, (name, K)  # every s * K boundary falls inside a warp for some s
    # the distances of rule 4, with the tolerances of the GPU test
    for name in ("w31", "w32", "w64", "w65"):
        tr = {}
        set_counts(ms.get(name), 50.0, trace=tr)
        d = np.concatenate(tr["d"])
        for want, tag in ((50.0, "d_eq_50"), (600.0, "d_eq_600"), (1800.0, "d_eq_1800"), (1250.0, "d_eq_1200_plus_tol"),
                          (0.0, "d_eq_0")):
            if (d == want).any():
                seen.add(tag)
        if ((d < 50.0) & (d > 49.999)).any():
            seen.add("d_one_ulp_under_50")
    need = {"first_time_after_0", "duplicated_times", "wholly_unvoiced", "identity_identity", "identity_near",
            "resampled_off", "resampled_far", "appended_sample", "largest_reference_twice", "knot_after_rounding", "knot",
            "between_lane_31_voiced_and_lane_0_zero", "inside_the_window_step", "inside_the_second_window_step",
            "settings_times_frames_not_a_multiple_of_32", "d_eq_50", "d_eq_600", "d_eq_1800", "d_eq_1200_plus_tol",
            "d_eq_0", "d_one_ulp_under_50"}
    assert need <= seen, need - seen
    assert {0, 1, 31, 32, 33} <= counts


@pytest.mark.parametrize("mut", MUTANTS)
def test_mutants_are_caught(mut):
    """Each slip changes at least one count of one set, at one of the GPU test's tolerances."""
    for name in ms.NAMES:
        for tol in ms.TOLS:
            got = set_counts(ms.get(name), tol, (mut,))
            if not np.array_equal(got, expected(name, tol)):
                assert mut not in EQUIVALENT
                return
    assert mut in EQUIVALENT, f"no set tells {mut} apart"


# ------------------------------------------------------------------------------------------------ bent notes
def note_melody(start, end, pitch, bends, g, highest=False):
    """evaluate.note_frames_to_melody, frame by frame; `highest`: the highest pitch wins a tie (a mutant)."""
    from basic_pitch_b200.evaluate import BENT_HZ

    T = g.shape[0]
    f0 = np.zeros(T)
    for t in range(T):
        best = None
        for j in range(len(start)):
            if not (start[j] <= t < end[j]):
                continue
            p = int(pitch[j])
            key = 3 * (p - 21) + (int(bends[j][t - start[j]]) if bends[j] is not None and len(bends[j]) else 0)
            v = np.float32(g[t, p - 21])
            if best is None:
                best = (v, p, key)
                continue
            bv, bp = best[0], best[1]
            if p == bp:
                continue
            wins = (v > bv) or (np.isnan(bv) and not np.isnan(v)) or (
                v == bv and (p > bp if highest else p < bp)) or (np.isnan(v) and np.isnan(bv) and (
                    p > bp if highest else p < bp))
            if wins:
                best = (v, p, key)
        if best is not None:
            f0[t] = BENT_HZ[best[2]]
    return f0


def _bent_cases():
    from tests.test_postsets import oracle

    files, grid, refs = ms.bent()
    for i, (note, onset, contour) in enumerate(files):
        for p in grid:
            notes = oracle(note, onset, contour, p)
            start, end, pitch = (np.array([n[k] for n in notes], np.int64) for k in range(3))
            for bends_on in (True, False):
                bends = [n[4] if bends_on else None for n in notes]
                yield i, note, start, end, pitch, bends, refs[i]


def test_bent_set_reaches_its_edges_and_the_tie_mutant_is_caught():
    from basic_pitch_b200.evaluate import BENT_HZ, note_frames_to_melody

    from basic_pitch_b200.evaluate import melody_values

    for t, hz in ms.bent()[2]:  # valid reference tracks: times non-decreasing from >= 0, voiced only where cents != 0
        c, v = melody_values(hz)
        assert len(t) and t[0] >= 0 and (np.diff(t) >= 0).all() and not v[c == 0].any()
    seen = set()
    differs = False
    for i, note, start, end, pitch, bends, ref in _bent_cases():
        T = note.shape[0]
        t_est, f0 = note_frames_to_melody(start, end, pitch, bends, note)
        assert note_melody(start, end, pitch, bends, note).tobytes() == f0.tobytes()
        mutated = note_melody(start, end, pitch, bends, note, highest=True)
        if mr.counts(ref[0], ref[1], t_est, mutated) != mr.counts(ref[0], ref[1], t_est, f0):
            differs = True
        for t in range(T):
            sounding = [j for j in range(len(start)) if start[j] <= t < end[j]]
            ps = sorted({int(pitch[j]) for j in sounding})
            if not ps:
                if t % 32 == 0 and t > 0 and f0[t - 1] != 0:
                    seen.add("silence_starts_a_tile")
                if t % 32 == 0 and t > 0 and f0[t - 1] == 0 and (f0[:t] != 0).any():
                    seen.add("silence_across_a_tile")
                continue
            vals = note[t, np.array(ps) - 21]
            fin = vals[~np.isnan(vals)]
            if len(fin) and (fin == fin.max()).sum() >= 2:
                seen.add("tie")
            if np.isnan(vals).any() and len(fin):
                seen.add("nan_under_a_sounding_note")
            if len(fin) and vals[-1] == fin.max() and (fin == fin.max()).sum() == 1 and len(ps) > 1:
                seen.add("higher_pitch_wins")
            if f0[t] == BENT_HZ[0]:
                seen.add("key_0")
            if f0[t] == BENT_HZ[263]:
                seen.add("key_263")
            if len(ps) >= 3 and len(fin) and (fin == fin.max()).sum() >= 3:
                seen.add("three_way_tie")
    assert differs, "no bent case tells the highest-pitch tie mutant apart"
    need = {"tie", "three_way_tie", "nan_under_a_sounding_note", "higher_pitch_wins", "key_0", "key_263",
            "silence_across_a_tile", "silence_starts_a_tile"}
    assert need <= seen, need - seen
