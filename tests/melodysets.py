"""Adversarial inputs for the melody scorers (CPU only: plain NumPy, deterministic, seeded).

The shipped model's posteriorgrams are smooth sigmoid outputs and the reference tracks of the other tests are sampled
on ordinary grids, which leaves most edges of bp_score_melody_grid_* and bp_score_note_melody_grid_* (csrc/score_melody.cu,
the melody section of csrc/api.cu, rules 1 to 4 of include/bp_b200.h) unobserved.  A grid set is a `MelSet`: files
(posteriorgram, reference track), the bin cents table and the settings `(threshold, bin_lo, bin_hi, guess_unvoiced)` it
is meant for.

  contour / note   widths 264 and 88 with the model's tables (evaluate.melody_bins); references are Hz tracks, so the
                   sets also go through Model.score_melody_grid
  w1 .. w65        raw widths 1, 31, 32, 33, 64 and 65 with custom tables: equal neighbouring entries, an entry of
                   exactly 0 cents (10 Hz), negative cents, values on a 1/8-cent grid so that a reference at est +- tol
                   or est + 600 is exactly that far away; references are given as cents and voicing

Every grid set has files of 0, 1, 31, 32, 33, 64, 65, 171, 172, 173 and 349 model frames.  Their rows hold arg-max ties
within a lane and across lanes (both orders of lane and bin), on a range's ends, against a larger value just outside
the range, whole-row plateaus, +0.0 against -0.0, -inf cells and rows, NaN in every lane but one, NaN where the finite
maximum would be, rows NaN only inside a range, and cells equal to a threshold.  Frames 31 and 63 of a file are voiced
and frames 32 and 64 all-NaN, so that the held cents cross a 32-frame tile; a file ending voiced is followed by one
starting with NaN rows.  The references take identity bases (exact, within np.allclose, just outside it), a base of the
same length that is not close, a first time > 0, times past the last estimate time, knots and times that reach a knot
only after np.round(x, 10), duplicated times, times between frames 31 / 32 and 63 / 64 and across the 172-frame window
step of the model frame times; counts of 1, 31, 32, 33 and 0 frames per file, and a wholly unvoiced track.  Reference
cents sit at est +- tol, est +- (tol - 1 ulp), est +- 1200 +- tol, est + 600 and est + 1800 of the estimate that the
first setting reads there.

`bent()` is the bent-note set: note / onset / contour posteriorgrams whose decode sounds two or three pitches with equal
note values at once, a higher pitch that wins on some frames only, NaN note cells under a sounding note, winners at
bent keys 0 and 263 and a silent stretch across a 32-frame tile; decode settings follow tests/postsets.py.

Liveness (that each set reaches the edges it is built for) and mutants of the rules are in
tests/test_melody_edges_cpu.py; the device comparison is tests/test_gpu_melody_edges.py.
"""
from __future__ import annotations

import functools
from typing import List, NamedTuple, Optional, Tuple

import numpy as np

from tests import postsets

LENGTHS = (0, 1, 31, 32, 33, 64, 65, 171, 172, 173, 2 * 172 + 5)
WIDTHS = (264, 88, 1, 31, 32, 33, 64, 65)
NAMES = ("contour", "note") + tuple(f"w{w}" for w in WIDTHS[2:])
TOLS = (50.0, 600.0)

T3 = float(np.float32(0.3))
# thresholds: a float32 value, its float64 neighbours both ways, 0.1 (not a float32 value) and 0.5
THRESHOLDS = (T3, float(np.nextafter(T3, 1.0)), float(np.nextafter(T3, 0.0)), 0.1, 0.5)
# cells that equal or straddle them, and one that is voiced under every threshold
CELLS = (np.float32(T3), np.float32(0.1), np.float32(0.5), np.float32(0.75))
LOUD = np.float32(0.75)


class MelSet(NamedTuple):
    name: str
    kind: Optional[str]  # "contour" / "note": the model's table, Hz references; None: custom table
    cents: np.ndarray  # [width] float64
    grams: List[np.ndarray]  # per file (T, width) float32
    refs: List[Tuple[np.ndarray, np.ndarray, np.ndarray]]  # per file (times, cents, voiced int32)
    ref_hz: Optional[List[Tuple[np.ndarray, np.ndarray]]]  # per file (times, Hz) when kind is set
    params: List[Tuple[float, int, int, int]]  # (threshold, bin_lo, bin_hi, guess_unvoiced)


def frame_times(n: int) -> np.ndarray:
    from basic_pitch_b200.evaluate import model_frames_to_time

    return np.asarray(model_frames_to_time(n), np.float64)


def _q(x, step=64):
    return (np.round(np.asarray(x, np.float64) * step) / step).astype(np.float32)


# ------------------------------------------------------------------------------------------------------------ tables
def table(width: int) -> np.ndarray:
    """Cents of a custom table: Hz built first and read with evaluate.melody_values (as a caller would), on a 1/8-cent
    grid where that round trip is exact; non-decreasing, with equal neighbours, one entry of 0 cents (10 Hz) and
    negative entries (below 10 Hz) where the width allows."""
    from basic_pitch_b200.evaluate import melody_values

    if width == 1:
        want = np.array([4800.0])
    else:
        rng = np.random.default_rng(900 + width)
        steps = rng.choice([0.0, 12.5, 33.25, 100.0, 1200.0], width - 1, p=[0.15, 0.3, 0.25, 0.25, 0.05])
        want = 3000.0 + np.concatenate([[0.0], np.cumsum(steps)])
        if width >= 4:
            want[:3] = [-1200.0, -187.5, 0.0]  # below 10 Hz, below 10 Hz, exactly 10 Hz
            want[3:] = np.maximum(want[3:], 150.0)
            want = np.maximum.accumulate(want)
    hz = np.where(want == 0, 10.0, 10.0 * 2.0 ** (want / 1200.0))
    cents = melody_values(hz)[0]
    return np.ascontiguousarray(np.maximum.accumulate(cents))


def ranges(width: int) -> List[Tuple[int, int]]:
    """The whole width, empty ranges at 0 and at the width and inside, one bin, lo at 0, hi at the width, a cut inside."""
    W = width
    out = [(0, W), (0, 0), (W, W), (min(7, W - 1), min(7, W - 1) + 1), (0, max(1, W - 2)), (min(W - 1, 5), W)]
    if W > 40:
        out += [(3, W - 4), (W // 2, W // 2)]
    elif W > 2:
        out += [(1, W - 1)]
    seen, uniq = set(), []
    for r in out:
        if r not in seen:
            seen.add(r)
            uniq.append(r)
    return uniq


def settings(width: int) -> List[Tuple[float, int, int, int]]:
    """Every threshold x both guesses x every range, interleaved: consecutive settings use different ranges, so a
    setting's range index (first-seen order of distinct ranges) differs from its position."""
    rs = ranges(width)
    out = []
    k = 0
    for thr in THRESHOLDS:
        for g in (1, 0):
            for j in range(len(rs)):
                lo, hi = rs[(j + k) % len(rs)]
                out.append((thr, lo, hi, g))
            k += 1
    out.append((float(LOUD), 0, width, 1))  # an odd number of settings: s * K falls inside a warp
    return out


# -------------------------------------------------------------------------------------------------------------- rows
N_PATTERNS = 16


def _row(rng, W, pattern, rs):
    """One posteriorgram row of `pattern` against a target range drawn from rs (non-empty ones)."""
    row = _q(rng.integers(0, 6, W) / 64.0)  # background < 0.1
    live = [r for r in rs if r[1] > r[0]]
    lo, hi = live[int(rng.integers(0, len(live)))]
    n = hi - lo
    v = CELLS[int(rng.integers(0, len(CELLS)))]
    if pattern == 0 and n > 32:  # tie within one lane: bins b and b + 32
        b = lo + int(rng.integers(0, n - 32))
        row[b] = row[b + 32] = v
    elif pattern in (1, 2) and n > 32:  # tie across lanes; 1: the lower bin in the higher lane, 2: the other order
        a = int(rng.integers(1, 32))
        c = int(rng.integers(0, a))
        k = int(rng.integers(1, (n - c - 1) // 32 + 1)) if n - c - 1 >= 32 else 0
        b1, b2 = (lo + a, lo + 32 * k + c) if pattern == 1 else (lo + c, lo + 32 * k + a)
        if b2 < hi and b1 < b2:
            row[b1] = row[b2] = v
        else:
            row[lo] = row[hi - 1] = v
    elif pattern == 3:  # tie on the range's ends
        row[lo] = row[hi - 1] = v
    elif pattern == 4:  # the ends tie, a larger value just outside the range
        row[lo] = row[hi - 1] = np.float32(T3)
        if hi < W:
            row[hi] = LOUD
        if lo > 0:
            row[lo - 1] = LOUD
    elif pattern == 5:  # plateau over the whole row
        row[:] = v
    elif pattern == 6:  # +0.0 against -0.0 under a negative row
        row[:] = np.float32(-0.25)
        b1 = lo + int(rng.integers(0, n))
        b2 = lo + int(rng.integers(0, n))
        row[min(b1, b2)], row[max(b1, b2)] = (np.float32(-0.0), np.float32(0.0)) if rng.random() < 0.5 else (
            np.float32(0.0), np.float32(-0.0))
    elif pattern == 7:  # -inf cells around a maximum
        row[rng.random(W) < 0.5] = -np.inf
        row[lo + int(rng.integers(0, n))] = v
    elif pattern == 8:  # an all -inf row
        row[:] = -np.inf
    elif pattern == 9:  # NaN in every lane of the range but one
        keep = int(rng.integers(0, 32))
        idx = np.arange(W)
        row[((idx - lo) % 32 != keep)] = np.nan
        cand = [b for b in range(lo, hi) if (b - lo) % 32 == keep]
        if cand:
            row[cand[int(rng.integers(0, len(cand)))]] = v
    elif pattern == 10:  # NaN where the largest value would be, a smaller finite maximum elsewhere
        b = lo + int(rng.integers(0, n))
        row[b] = np.nan
        row[lo + (b - lo + 1 + int(rng.integers(0, max(n - 1, 1)))) % n] = np.float32(T3) if b != lo else row[lo]
    elif pattern == 11:  # NaN inside the range, finite (and loud) outside
        row[lo:hi] = np.nan
        row[:lo] = LOUD
        row[hi:] = LOUD
    elif pattern == 12:  # an all-NaN row
        row[:] = np.nan
    elif pattern == 13:  # unquantised noise
        row = rng.random(W).astype(np.float32)
    else:  # one maximum
        row[lo + int(rng.integers(0, n))] = v
    return row


def gram(rng, T, W, rs, prev_voiced_end=False):
    g = np.zeros((T, W), np.float32)
    for t in range(T):
        g[t] = _row(rng, W, int(rng.integers(0, N_PATTERNS)), rs)
    for t in (31, 63):  # voiced at tile position 31 under the whole range ...
        if t < T:
            g[t] = _q(rng.integers(0, 6, W) / 64.0)
            g[t, int(rng.integers(0, W))] = LOUD
    for t in (32, 64):  # ... and nothing at position 32 of the next tile
        if t < T:
            g[t] = np.nan
    if prev_voiced_end:  # the previous file ended voiced: this one starts with nothing
        g[:3] = np.nan
    if T >= 2:  # end voiced (the appended sample follows a voiced frame)
        g[T - 1] = _q(rng.integers(0, 6, W) / 64.0)
        g[T - 1, int(rng.integers(0, W))] = LOUD
    return g


# -------------------------------------------------------------------------------------------------------------- times
def _round_twin(t):
    """A time != t with np.round(x, 10) == np.round(t, 10), or t itself when none is near."""
    for d in (3e-12, -3e-12, 1e-12, -1e-12, 2e-11, -2e-11):
        x = t + d
        if x >= 0 and x != t and np.round(x, 10) == np.round(t, 10):
            return x
    return t


def ref_times(T: int, base: str, rng) -> np.ndarray:
    ft = frame_times(T)
    if base == "identity":
        return ft
    if base in ("near", "off"):  # |dt| just under / just over 1e-8 + 1e-5 |t| (np.allclose), both signs, t[0] = 0
        tol = 1e-8 + 1e-5 * np.abs(ft)
        sign = np.where(np.arange(T) % 2 == 0, 1.0, -1.0)
        t = ft + sign * tol * (0.999 if base == "near" else 1.001)
        t[0] = 0.0
        return t
    if base == "far":  # same length, not close
        return ft * 1.002 + 0.0007 * (np.arange(T) > 0)
    if base == "empty":
        return np.zeros(0)
    if base == "one":
        return np.array([ft[-1] * 0.5 + 0.001]) if T else np.array([0.0])
    if base == "unvoiced":
        return np.arange(0.0, 0.06, 0.01)
    # "mixed": knots, round-twins of knots, duplicates, tile and window-step interiors, times past the end
    pts = [0.0]
    knots = sorted(set(int(j) for j in rng.integers(0, T, min(T, 12))))
    pts += [ft[j] for j in knots]
    pts += [_round_twin(ft[j]) for j in knots[::2]]
    pts += [ft[knots[0]], ft[knots[-1]]]  # duplicated knots
    for j in (30, 31, 62, 63, 170, 171, 172, 342, 343, 344):  # interiors at the tile and window boundaries
        if j + 1 < T:
            for f in (0.125, 0.5, 0.875):
                pts.append(ft[j] + f * (ft[j + 1] - ft[j]))
    mid = ft[T // 2] + 0.3 * (ft[min(T // 2 + 1, T - 1)] - ft[T // 2]) if T > 1 else 0.004
    pts += [mid, mid]  # a duplicated non-knot
    end = ft[-1] if T else 0.0
    pts += [end + 0.0031, end + 0.02, end + 0.02]  # past the last estimate time, the largest one twice
    t = np.sort(np.array(pts, np.float64))
    if base == "late":  # first time > 0: rule 1 inserts a reference frame at 0
        t = t[t > 0]
        t = np.unique(np.concatenate([t, np.arange(0.005, end + 0.03, 0.01)]))
    return t


# per file length: the reference base (counts 1, 31, 32, 33 and 0 among them)
BASES = {0: "unvoiced", 1: "identity", 31: "identity", 32: "near", 33: "off", 64: "mixed", 65: "late", 171: "far",
         172: "empty", 173: "mixed", 349: "mixed"}


# ------------------------------------------------------------------------------------------------------- estimates
def argmax_bins(g: np.ndarray, lo: int, hi: int) -> np.ndarray:
    """b* of every row (-1: empty range or all NaN in range): the largest float32 value, the lowest bin on a tie."""
    out = np.full(g.shape[0], -1, np.int64)
    if hi <= lo or g.shape[0] == 0:
        return out
    sub = g[:, lo:hi]
    ok = ~np.isnan(sub).all(axis=1)
    with np.errstate(invalid="ignore"):
        best = np.where(ok, np.nanmax(np.where(ok[:, None], sub, 0), axis=1), 0)
    b = np.argmax((sub == best[:, None]) & ok[:, None], axis=1)
    out[ok] = lo + b[ok]
    return out


def estimate(g: np.ndarray, cents: np.ndarray, p, bins=None) -> Tuple[np.ndarray, np.ndarray]:
    """(cents, voiced) of every frame under setting p by the rule of include/bp_b200.h (bp_score_melody_grid_*)."""
    thr, lo, hi, guess = p
    b = argmax_bins(g, lo, hi) if bins is None else bins
    ok = b >= 0
    v = np.zeros(len(b), bool)
    v[ok] = g[np.flatnonzero(ok), b[ok]].astype(np.float64) >= thr
    c = np.where(ok & (v | bool(guess)), cents[np.maximum(b, 0)], 0.0)
    return c, v.astype(np.int32)


# ----------------------------------------------------------------------------------------------------- references
def _resampled(ref_t, est_t, est_c):
    """The estimate cents interp1d reads at the reference times (rules 1 to 3), held cents and the zero-order mask."""
    from oracle import melody_ref as mr

    if len(est_t) == 0 or len(ref_t) == 0:
        return np.zeros(len(ref_t))
    rt = np.insert(ref_t, 0, 0.0) if ref_t[0] > 0 else ref_t
    c, _ = mr.resample_melody_series(est_t, est_c, (est_c != 0).astype(float), rt)
    return c[len(rt) - len(ref_t):]


def ref_cents(rng, est, tol_set, tab):
    """Reference cents at the listed distances from the estimate cents `est` (a random table value where est is 0)."""
    out = np.empty(len(est))
    for k, e in enumerate(est):
        tol = tol_set[int(rng.integers(0, len(tol_set)))]
        if e == 0.0:
            c = float(tab[int(rng.integers(0, len(tab)))]) + 25.0
        else:
            s = 1.0 if rng.random() < 0.5 else -1.0
            opts = (0.0, tol, -tol, np.nextafter(e + tol, e) - e, np.nextafter(e - tol, e) - e, 1200.0 + tol,
                    -1200.0 - tol, 2400.0 - tol, 600.0, 1800.0, -600.0, s * 17.0, 600.0 + 1e-9)
            c = e + opts[int(rng.integers(0, len(opts)))]
        out[k] = c if c != 0.0 else 5.0
    return out


def _build(name: str) -> MelSet:
    from basic_pitch_b200.evaluate import melody_bins, melody_values

    kind = name if name in ("contour", "note") else None
    W = {"contour": 264, "note": 88}.get(name) or int(name[1:])
    rng = np.random.default_rng(sum(map(ord, name)) * 7919)
    tab = melody_bins(kind)[1] if kind else table(W)
    rs = ranges(W)
    ps = settings(W)
    grams, refs, ref_hz = [], [], []
    order = list(LENGTHS)
    prev_end = False
    for T in order:
        g = gram(rng, T, W, rs, prev_voiced_end=prev_end)
        prev_end = T >= 2
        grams.append(g)
        t = ref_times(T, BASES[T], rng)
        ft = frame_times(T)
        c0, _ = estimate(g, tab, ps[0])
        est_at = _resampled(t, ft, c0) if T else np.zeros(len(t))
        c = ref_cents(rng, est_at, TOLS, tab)
        voiced = (rng.random(len(t)) < 0.8).astype(np.int32)
        if BASES[T] == "unvoiced":
            voiced[:] = 0
            c[::2] = 0.0
        if kind:
            hz = 10.0 * 2.0 ** (c / 1200.0) * np.where(voiced == 1, 1.0, -1.0)
            hz[c == 0.0] = 0.0
            c, voiced = melody_values(hz)
            ref_hz.append((t, hz))
        voiced = np.where(c == 0.0, 0, voiced).astype(np.int32)
        refs.append((t, c, voiced))
    return MelSet(name, kind, np.ascontiguousarray(tab, np.float64), grams, refs, ref_hz if kind else None, ps)


@functools.lru_cache(maxsize=None)
def get(name: str) -> MelSet:
    return _build(name)


def hz_settings(s: MelSet) -> List[dict]:
    """The settings of a contour / note set as Model.score_melody_grid takes them: the bin range as frequencies (a cut
    inside the bin gap on each side, a minimum above the maximum for an empty range)."""
    from basic_pitch_b200.evaluate import salience_bins

    hz = salience_bins(s.kind)[0]
    W = len(hz)
    out = []
    for thr, lo, hi, g in s.params:
        d = dict(threshold=thr, guess_unvoiced=bool(g))
        if lo > 0:
            d["minimum_frequency"] = float(np.sqrt(hz[lo - 1] * hz[lo])) if lo < W else float(hz[-1] * 1.01)
        if hi < W:
            d["maximum_frequency"] = float(np.sqrt(hz[hi - 1] * hz[hi])) if hi > 0 else float(hz[0] * 0.99)
        if hi == lo and 0 < lo < W:
            d["maximum_frequency"] = float(hz[lo - 1])  # below the minimum
        out.append(d)
    return out


# ------------------------------------------------------------------------------------------------------- bent notes
BENT_T = (140, 40, 0, 70)


def _bent_file(rng, T, first):
    note = np.zeros((T, 88), np.float32)
    onset = np.zeros((T, 88), np.float32)
    contour = _q(rng.random((T, 264)) * 0.5)
    if T == 0:
        return note, onset, contour
    if first:
        # 60, 64, 67: equal note values on [2, 32) (the lowest sounds through a NaN stretch), 72 louder on [10, 20)
        for p in (60, 64, 67):
            onset[2, p - 21] = 0.75
            note[2:32, p - 21] = 0.5
        note[12:16, 60 - 21] = np.nan
        note[24:27, 60 - 21] = np.nan
        note[24:27, 64 - 21] = np.nan  # every sounding cell but one NaN
        onset[10, 72 - 21] = 0.75
        note[10:20, 72 - 21] = 0.625
        note[20:32, 72 - 21] = 0.375
        # silence on [32, 70): across the tile boundary at 64; then pitches 21 and 108 at the contour's ends
        onset[70, 0] = onset[70, 87] = 0.75
        note[70:100, 0] = 0.5
        note[70:85, 87] = 0.375
        note[85:100, 87] = 0.625
        contour[70:100, 0] = 1.0
        contour[70:100, 263] = 1.0
        # 62 and 63 tie on [104, 131), one frame past a tile boundary at 128
        for p in (62, 63):
            onset[104, p - 21] = 0.75
            note[104:131, p - 21] = 0.4375
    else:
        for p in (48, 55):
            onset[1, p - 21] = 0.75
            note[1:T - 3, p - 21] = 0.5
        contour[:, :] = _q(rng.random((T, 264)))
    return note, onset, contour


@functools.lru_cache(maxsize=None)
def bent():
    """(files [(note, onset, contour)], decode settings (tests/postsets.py params), reference tracks [(times, Hz)])."""
    rng = np.random.default_rng(4242)
    files = [_bent_file(rng, T, j == 0) for j, T in enumerate(BENT_T)]
    grid = [
        postsets.params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=2, energy_tol=3, infer_onsets=False,
                        melodia_trick=False),
        postsets.params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=2, energy_tol=3, infer_onsets=False),
        postsets.params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=2, energy_tol=3, infer_onsets=False,
                        melodia_trick=False, lo_col=40),
    ]
    refs = []
    for j, (note, onset, contour) in enumerate(files):
        T = note.shape[0]
        t = ref_times(T, "mixed" if j != 3 else "off", rng) if T else np.array([0.0, 0.01])
        c = np.full(len(t), 4800.0)
        if T:
            f0 = bent_f0(note, onset, contour, grid[0])
            c = ref_cents(rng, _resampled(t, frame_times(T), melody_values_cents(f0)), (50.0,), [4800.0])
        hz = 10.0 * 2.0 ** (c / 1200.0)
        hz[rng.random(len(t)) < 0.15] = 0.0
        refs.append((t, hz))
    return files, grid, refs


def melody_values_cents(hz):
    from basic_pitch_b200.evaluate import melody_values

    return melody_values(hz)[0]


def bent_f0(note, onset, contour, p, include_pitch_bends=True):
    """evaluate.note_frames_to_melody of the CPU decode (tests/test_postsets.oracle) of one file under p."""
    from basic_pitch_b200.evaluate import note_frames_to_melody
    from tests.test_postsets import oracle

    notes = oracle(note, onset, contour, p)
    start, end, pitch = (np.array([n[k] for n in notes], np.int64) for k in range(3))
    bends = [n[4] if include_pitch_bends else None for n in notes]
    return note_frames_to_melody(start, end, pitch, bends, note)[1]
