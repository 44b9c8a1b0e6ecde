"""CPU: a float64 NumPy restatement of the GPU sonification (csrc/sonify.cu) on the adversarial sets of
tests/sonifysets.py, against the stand-in synthesiser and its per-sample bound (`standin` of tests/test_gpu_sonify.py).

`render` restates `plan_file` (spans, fades, instruments, the time-sorted bend table, each event's switch sample, the
segments with their phase prefixes s0, the tiles and each entry's starting segment) and the tile kernel's per-sample
formula, with np.sin.  Three kinds of test:

  restatement  on every set, rate and multiple_pitch_bends value the restatement stays within the bound; so the plan
               the kernel is given, and the formula it evaluates, are the stand-in's up to the rounding of the phase
  liveness     the sets reach the edges they are built for, counted per rate
  mutants      a restated slip in any placement or velocity rule leaves the bound on at least one set; the mutants
               the bound cannot see, and should not, are documented in EQUIVALENT, each with the case it changes
               shown to be reached
"""
from __future__ import annotations

import bisect
import functools
import math
from fractions import Fraction

import numpy as np
import pytest

from tests import sonifysets as ss
from tests.test_gpu_sonify import assert_within, standin

TWO_PI = 2.0 * np.pi
TILE = ss.TILE

# restated slips, each of which must leave the bound somewhere
MUTANTS = {
    "round_a": "a = round(fs * start) instead of the truncation",
    "round_b": "b = round(fs * end) instead of the truncation",
    "ceil_only": "a bend's switch sample ceil(fs * t) without the two correction loops",
    "collapse_first": "the first, not the last, of the events sharing a switch sample",
    "side_left": 'searchsorted side="left": a bend switches after k / fs == t, not at it',
    "cum_from_zero": "the closed-form cumulative sum without the sample itself: k - k_seg, not k - k_seg + 1",
    "fade_off_by_one": "fade = min(fade_max, (len + 1) // 2)",
    "tail_len_m": "the tail ramp (len - m) / fade instead of (len - 1 - m) / fade",
    "drop_last_tile": "a note left out of its last tile",
    "seg_at_tile_end": "an entry's segment taken at the tile's last sample of the note instead of its first",
    "vel_f64": "the velocity product 127 * amplitude in float64",
    "vel_half_away": "the velocity rounded half away from zero",
    "touching_overlap": "drop_overlapping_pitch_bends treating touching notes (start == previous end) as overlapping",
    "signed_peak": "the peak as max y instead of max |y|",
}

# mutants the bound cannot see: each changes only what the bound is there to absorb, or nothing at all
EQUIVALENT = {
    "note_order": "the notes summed in reverse order: a different rounding of the sum of n(k) notes, the 2 (n + 1) u "
                  "term of the bound",
    "fma_accumulate": "acc = fma(sin(phase) * env, vscale, acc), the product's rounding error carried into the sum "
                      "(Dekker's two-product): one rounding fewer per note, inside the same term",
    "instrument_sorted": "with multiple_pitch_bends the instruments summed in pitch order instead of first use: only "
                         "the order of the sum changes",
    "seg_at_tile": "an entry's segment taken at 256 t instead of max(a, 256 t): the two differ only in a note's first "
                   "tile, where 256 t < a and every later segment starts after a, so the kernel's walk, which only "
                   "moves forward, starts and stays at the note's first segment either way (bit-identical output)",
}


# --------------------------------------------------------------------------------------------------------- restatement
def velocity(amp, mut=frozenset()) -> float:
    """int(np.round(127 * np.float32(amp))) as a float (exact), and its mutants."""
    p = 127.0 * float(amp) if "vel_f64" in mut else float(np.float32(127) * np.float32(amp))
    if "vel_half_away" in mut:
        return math.copysign(math.floor(abs(p) + 0.5), p)
    return float(np.round(p))


def drop_overlapping(ev, mut=frozenset()):
    ev = sorted(ev)
    for i in range(len(ev) - 1):
        for j in range(i + 1, len(ev)):
            if (ev[j][0] > ev[i][1]) if "touching_overlap" in mut else (ev[j][0] >= ev[i][1]):
                break
            ev[i] = ev[i][:-1] + (None,)
            ev[j] = ev[j][:-1] + (None,)
    return ev


def first_sample_at(t: float, fs: int, mut=frozenset()) -> int:
    """The first sample k with k / fs >= t (> t under side_left)."""
    if "side_left" in mut:
        if t < 0.0:
            return 0
        k = max(0, math.ceil(t * fs))
        while k > 0 and (k - 1) / fs > t:
            k -= 1
        while k / fs <= t:
            k += 1
        return k
    if not t > 0.0:
        return 0
    k = math.ceil(t * fs)
    if "ceil_only" in mut:
        return k
    while k > 0 and (k - 1) / fs >= t:
        k -= 1
    while k / fs < t:
        k += 1
    return k


def fma(x: float, y: float, z: float) -> float:
    return float(Fraction(x) * Fraction(y) + Fraction(z))


def _two_product(x, y):
    """p = fl(x y) and its exact error e = x y - p (Dekker, Veltkamp splitting), elementwise."""
    p = x * y
    c = 134217729.0 * x
    xh = c - (c - x)
    xl = x - xh
    c = 134217729.0 * y
    yh = c - (c - y)
    yl = y - yh
    return p, ((xh * yh - p) + xh * yl + xl * yh) + xl * yl


def _fma_add(acc, x, y):
    p, e = _two_product(x, y)
    s = acc + p
    bb = s - acc
    return s + (((acc - (s - bb)) + (p - bb)) + e)


def plan(events, fs: int, multi: bool, mut=frozenset()):
    """sonify.cu's plan_file: n_samples and the sounding notes in accumulation order, each a dict of its span, fade,
    vscale, segments (k, f, s0) and per-tile entry segments; plus what the liveness test counts."""
    ev = list(events)
    live = {}
    if not ev:
        return 0, [], live
    if not multi:
        ev = drop_overlapping(ev, mut)
    keys = list(dict.fromkeys((e[2] if multi else 0) for e in ev))
    if "instrument_sorted" in mut:
        keys.sort()
    bend_times = [np.linspace(e[0], e[1], len(e[4])) if e[4] else [] for e in ev]
    end_time = max([e[1] for e in ev] + [float(t) for bt in bend_times for t in bt])
    n = int(fs * (end_time + 1))
    fm = int(0.01 * fs)
    cnt = lambda key, by=1: live.__setitem__(key, live.get(key, 0) + by)  # noqa: E731
    notes = []
    for key in keys:
        idx = [i for i, e in enumerate(ev) if (e[2] if multi else 0) == key]
        bt = []
        for i in idx:
            if ev[i][4]:
                ticks = np.clip(np.round(np.array(ev[i][4]) * 4096 / 3).astype(int), -8192, 8191)
                cnt("clipped_ticks", int(np.sum(np.abs(ticks) == 8192) + np.sum(ticks == 8191)))
                bt += [(float(t), float(tk) * (2.0 / 8192.0)) for t, tk in zip(bend_times[i], ticks)]
        bt.sort(key=lambda x: x[0])  # stable, like sorted(..., key=time)
        kb = [first_sample_at(t, fs, mut) for t, _ in bt]
        for (t, _), k in zip(bt, kb):
            if t > 0 and k / fs == t:
                cnt("bend_at_k_over_fs")
            if t > 0 and math.ceil(t * fs) != first_sample_at(t, fs):
                cnt("ceil_needs_correction")
        cnt("equal_bend_times", sum(1 for j in range(1, len(bt)) if bt[j][0] == bt[j - 1][0]))

        def freq(pitch, j):
            semis = float(pitch) + (bt[j][1] if j >= 0 else 0.0)
            return 440.0 * 2.0 ** ((semis - 69.0) / 12.0)

        for i in idx:
            e = ev[i]
            rnd = lambda x, which: int(round(fs * x)) if which in mut else int(fs * x)  # noqa: E731
            a, b = rnd(e[0], "round_a"), rnd(e[1], "round_b")
            if b <= a:
                continue
            L = b - a
            fade = min(fm, (L + 1) // 2 if "fade_off_by_one" in mut else L // 2)
            for what, pos in (("a", a), ("b", b)):
                if pos % TILE in (TILE - 1, 0, 1):
                    cnt(f"{what}_at_tile_edge")
            for what, x in (("a_round_differs", e[0]), ("b_round_differs", e[1])):
                if int(round(fs * x)) != int(fs * x):
                    cnt(what)
            if L in (1, 2, 3, 2 * fm - 1, 2 * fm, 2 * fm + 1) and fm > 0:
                cnt(f"fade_len_{'short' if L <= 3 else 'two_fades' if L < 2 * fm + 1 else 'two_fades_plus'}")
            v = velocity(e[3], mut)
            pv = float(np.float32(127) * np.float32(e[3]))
            if pv - math.floor(pv) == 0.5:
                cnt("velocity_tie")
            if velocity(e[3], {"vel_f64"}) != velocity(e[3]):
                cnt("velocity_f32_f64")
            j = bisect.bisect_right(kb, a) - 1
            seg_k, seg_f, seg_s0 = [a], [freq(e[2], j)], [0.0]
            j += 1
            while j < len(kb) and kb[j] < b:
                first = j
                while j + 1 < len(kb) and kb[j + 1] == kb[j]:
                    j += 1
                cnt("collapsed_events", j - first)
                if kb[j] % TILE in (TILE - 1, 0, 1):
                    cnt("switch_at_tile_edge")
                if kb[j] == b - 1:
                    cnt("switch_at_b_minus_1")
                seg_f.append(freq(e[2], first if "collapse_first" in mut else j))
                seg_s0.append(fma(float(kb[j] - seg_k[-1]), seg_f[-2], seg_s0[-1]))  # std::fma on the host
                seg_k.append(kb[j])
                j += 1
            if any(k == a for k in kb):
                cnt("switch_at_a")
            if any(k == b for k in kb):
                cnt("switch_at_b")
            if any(k < a for k in kb):
                cnt("bend_before_a")
            seg_k = np.array(seg_k, np.int64)
            per_tile = np.bincount(seg_k[1:] // TILE) if len(seg_k) > 1 else np.zeros(1, int)
            cnt("tiles_with_8_switches", int(np.sum(per_tile >= 8)))
            t0, t1 = a // TILE, (b - 1) // TILE
            entry = []
            for t in range(t0, t1 + 1):
                if "seg_at_tile" in mut:
                    k = t * TILE
                elif "seg_at_tile_end" in mut:
                    k = min(b - 1, t * TILE + TILE - 1)
                else:
                    k = max(a, t * TILE)
                # plan_file's walk from the note's first segment: forwards while the next one starts at or before k
                entry.append(max(0, int(np.searchsorted(seg_k, k, side="right")) - 1))
                if t * TILE < a and len(seg_k) > 1 and seg_k[1] < (t + 1) * TILE:
                    cnt("switch_in_first_tile_after_mid_tile_start")
            notes.append(dict(a=a, b=b, fade=fade, inv=1.0 / fade if fade > 0 else 0.0, vscale=v / 127.0,
                              k=seg_k, f=np.array(seg_f), s0=np.array(seg_s0), t0=t0, t1=t1, entry=np.array(entry)))
    cover = np.zeros(max(n, 1) // TILE + 2, np.int64)
    for nt in notes:
        cover[nt["t0"] : nt["t1"] + 1] += 1
    live["longest_csr_row"] = int(cover.max())
    return n, notes, live


def render(events, fs: int, multi: bool, mut=frozenset()):
    """-> (samples, liveness counts) of the restated plan and tile kernel."""
    n, notes, live = plan(events, fs, multi, mut)
    if not list(events):
        return np.array([]), live
    y = np.zeros(n)
    order = notes[::-1] if "note_order" in mut else notes
    for nt in order:
        a, b = nt["a"], nt["b"]
        k = np.arange(a, b, dtype=np.int64)
        tile = k // TILE
        if "drop_last_tile" in mut:
            k = k[tile < nt["t1"]]
            tile = tile[tile < nt["t1"]]
        # the kernel's walk from the entry's segment: forwards while the next segment starts at or before k
        s = np.maximum(nt["entry"][tile - nt["t0"]], np.searchsorted(nt["k"], k, side="right") - 1)
        step = (k - nt["k"][s]) if "cum_from_zero" in mut else (k - nt["k"][s] + 1)
        cum = step.astype(np.float64) * nt["f"][s] + nt["s0"][s]
        phase = TWO_PI * cum / fs
        m, L, fade = k - a, b - a, nt["fade"]
        tail = (L - m) if "tail_len_m" in mut else (L - 1 - m)
        env = np.where(m < fade, m * nt["inv"], np.where(m >= L - fade, tail * nt["inv"], 1.0))
        x = np.sin(phase) * env
        if "fma_accumulate" in mut:
            y[k] = _fma_add(y[k], x, np.full_like(x, nt["vscale"]))
        else:
            y[k] += x * nt["vscale"]
    peak = float(y.max()) if "signed_peak" in mut else float(np.abs(y).max())
    if n and y[np.argmax(np.abs(y))] < 0:
        live["negative_peak"] = 1
    return (y / peak if peak > 0 else y), live


# --------------------------------------------------------------------------------------------------------------- cases
def cases(rates=ss.RATES):
    for fs in rates:
        for s in ss.sets(fs):
            for multi in (False, True):
                yield fs, s, multi


@functools.lru_cache(maxsize=None)
def _standin(fs, name, i, multi):
    s = next(x for x in ss.sets(fs) if x.name == name)
    return standin(s.files[i], fs, multi)


def ratio(got, fs, name, i, multi) -> float:
    """max err / bound of one file (inf on a shape mismatch or an error where the bound is 0)."""
    ref, tol = _standin(fs, name, i, multi)
    if got.shape != ref.shape:
        return math.inf
    err = np.abs(got - ref)
    if not err.size:
        return 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / tol)
    return float(r.max())


@pytest.mark.parametrize("fs", ss.RATES)
def test_restatement_stays_within_the_bound(fs):
    worst = {}
    for _fs, s, multi in cases((fs,)):
        for i, ev in enumerate(s.files):
            got, _ = render(ev, fs, multi)
            assert_within(got, ev, fs, multi, (fs, s.name, i, multi))
            worst[s.name] = max(worst.get(s.name, 0.0), ratio(got, fs, s.name, i, multi))
    print(fs, {k: f"{v:.3f}" for k, v in worst.items()})


def liveness(fs):
    tot = {}
    for _fs, s, multi in cases((fs,)):
        for ev in s.files:
            _, live = render(ev, fs, multi)
            for k, v in live.items():
                if k == "longest_csr_row":
                    tot[k] = max(tot.get(k, 0), v)
                else:
                    tot[k] = tot.get(k, 0) + v
    return tot


# each edge every rate must reach (and how often at least)
EVERY_RATE = dict(a_at_tile_edge=20, b_at_tile_edge=20, a_round_differs=10, b_round_differs=10, switch_at_tile_edge=5,
                  switch_at_a=2, switch_at_b=1, switch_at_b_minus_1=1, bend_before_a=2, collapsed_events=5,
                  tiles_with_8_switches=2, bend_at_k_over_fs=10, equal_bend_times=5, clipped_ticks=10,
                  velocity_tie=128, velocity_f32_f64=8, negative_peak=1, longest_csr_row=300,
                  switch_in_first_tile_after_mid_tile_start=2)


@pytest.mark.parametrize("fs", ss.RATES)
def test_the_sets_reach_every_edge(fs):
    live = liveness(fs)
    print(fs, dict(sorted(live.items())))
    for k, least in EVERY_RATE.items():
        assert live.get(k, 0) >= least, (fs, k, live.get(k, 0), least)
    if ss.fade_max(fs) > 0:
        for k in ("fade_len_short", "fade_len_two_fades", "fade_len_two_fades_plus"):
            assert live.get(k, 0) >= 1, (fs, k)


def test_ceil_needs_its_correction_somewhere():
    """ceil(fs * t) is not the first sample at or after t for some bend time of the sets (one rounding of the product
    away from it), at more than one rate; the mutant test shows that the difference is audible."""
    hits = {fs: liveness(fs).get("ceil_needs_correction", 0) for fs in ss.RATES}
    print(hits)
    assert sum(1 for v in hits.values() if v) >= 3, hits


def _caught(mut):
    """The first (fs, set, file, multi) on which the mutant leaves the bound, or None."""
    for fs, s, multi in cases():
        for i, ev in enumerate(s.files):
            if not ev:
                continue
            with np.errstate(all="ignore"):
                got, _ = render(ev, fs, multi, frozenset({mut}))
            if ratio(got, fs, s.name, i, multi) > 1.0:
                return fs, s.name, i, multi
    return None


@pytest.mark.parametrize("mut", sorted(MUTANTS))
def test_every_mutant_leaves_the_bound(mut):
    where = _caught(mut)
    print(mut, "caught at", where)
    assert where is not None, (mut, MUTANTS[mut])


EQUIVALENT_RATES = (50, 7919, 44100, 192000)


@pytest.mark.parametrize("mut", sorted(EQUIVALENT))
def test_equivalent_mutants_stay_within_the_bound_where_they_change_the_case(mut):
    """Each documented equivalent mutant stays within the bound everywhere, while the case it changes is reached:
    its output differs from the restatement's in the bits of some sample (seg_at_tile: some note starts inside a tile
    and switches within it, so the mutant asks for the segment at another sample; the output stays bit-identical)."""
    changed = 0
    for fs, s, multi in cases(EQUIVALENT_RATES):
        for i, ev in enumerate(s.files):
            if not ev:
                continue
            base, live = render(ev, fs, multi)
            got, _ = render(ev, fs, multi, frozenset({mut}))
            assert ratio(got, fs, s.name, i, multi) <= 1.0, (mut, fs, s.name, i, multi)
            if mut == "seg_at_tile":
                changed += live.get("switch_in_first_tile_after_mid_tile_start", 0)
                assert np.array_equal(base.view(np.uint64), got.view(np.uint64)), (fs, s.name, i, multi)
            else:
                changed += int(np.sum(base.view(np.uint64) != got.view(np.uint64)))
    print(mut, "changed", changed)
    assert changed > 0, (mut, EQUIVALENT[mut])
