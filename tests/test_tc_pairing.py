"""CPU: the pairing of frequency tiles into groups (tc_group_tile, kernels.cuh) as the library's planner applies it
(bp_debug_tc_plan), and the range / edge bookkeeping of the fused second convolutions built on it.

  * the group table is the pair-distance map: group g = position i = g % d of run g // d, tiles
    {2 d run + i, 2 d run + d + i} (contour: d = 1, neighbouring tiles; onset / note: d = G0 = 12),
  * the contour's two slots then share almost every weight tile: the ring walks 339 steps per 64-row M-tile instead of
    the 483 of the {g, g + 9} pairing,
  * every tile sums its steps in the order of that reference pairing, so its fp32 sums do not depend on its partner,
  * the halo of the fused conv2 is carried inside a slot's run of consecutive tiles and goes through the edge buffer at
    every other boundary: under every work split each boundary is finished exactly once, by the carry or by
    edge_fix_kernel, and the result is the direct convolution."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_fused_epilogue_math import CASES, MT, T, _thread_partials, _time_sum_tile
from tests.test_tc_plan import SPECS, _plan

NOUSE = 0xFFFFFFFF
CONTOUR_STEPS = 339  # contour ring steps per M-tile with neighbour pairs (the {g, g + 9} pairing: 483)
G0 = {0: 9, 1: 12, 2: 12}
CONV2 = {0: "contour2", 1: "onset2", 2: "note2"}


def _n_ft(which):
    FLT, WOUT = SPECS[which][7], SPECS[which][8]
    return (WOUT + FLT - 1) // FLT


def _pair_map(n_groups, n_ft, d):
    """The group -> tile map of tc_group_tile, restated."""
    gft = np.full((n_groups, 2), -1, np.int32)
    for g in range(n_groups):
        run, i = divmod(g, d)
        for slot in range(2):
            ft = 2 * d * run + slot * d + i
            gft[g, slot] = ft if ft < n_ft else -1
    return gft


def _pair_distance(which, gft):
    return int(gft[0, 1]) if which == 0 else G0[which]


@pytest.mark.parametrize("which", [0, 1, 2])
def test_group_table_is_the_pair_map(weights_np, which):
    tiles, tile_seq, slot_words, gso, gft, n_uses = _plan(which, weights_np[SPECS[which][0]])
    n_ft = _n_ft(which)
    d = _pair_distance(which, gft)
    assert len(gft) == G0[which]
    np.testing.assert_array_equal(gft, _pair_map(G0[which], n_ft, d))
    placed = sorted(int(t) for t in gft.reshape(-1) if t >= 0)
    assert placed == list(range(n_ft)), "every tile in exactly one (group, slot)"
    if which == 0:
        assert d == 1
        assert len(tile_seq) == CONTOUR_STEPS
        assert n_uses == 549  # the pairing only merges steps, it adds none


@pytest.mark.parametrize("which", [0, 1, 2])
def test_every_tile_sums_its_steps_in_the_reference_order(weights_np, which):
    """A tile's steps come in the order of the reference pairing {t, t + G0}, whatever tile the kernels pair it with:
    sorted by (time tap, A chunk), the weight tiles it has in common with its reference partner t +- G0 last for the
    lower tile and first for the upper one.  So its fp32 sums are those of that pairing, bit for bit."""
    tiles, tile_seq, slot_words, gso, gft, n_uses = _plan(which, weights_np[SPECS[which][0]])
    lbo16 = 64 + SPECS[which][1] - 1
    n_ft = _n_ft(which)
    seq = {}  # tile -> [(weight tile, dt, chunk)] in the order the slot walks them
    for g in range(len(gft)):
        for slot in range(2):
            for s in range(gso[g], gso[g + 1]):
                w = int(slot_words[slot, s])
                if w != NOUSE:
                    c8, dt = divmod(w & 0x3FFF, lbo16)
                    seq.setdefault(int(gft[g, slot]), []).append((int(tile_seq[s]), dt, c8))
                    assert bool(w & 0x8000) == (len(seq[int(gft[g, slot])]) == 1)  # first use zeroes the accumulator
    assert sorted(seq) == list(range(n_ft))
    for t in range(n_ft):
        partner = t + G0[which] if t < G0[which] else t - G0[which]
        common = {u[0] for u in seq[t]} & ({u[0] for u in seq[partner]} if partner < n_ft else set())
        own = sorted((u for u in seq[t] if u[0] not in common), key=lambda u: u[1:])
        shared = sorted((u for u in seq[t] if u[0] in common), key=lambda u: u[1:])
        assert seq[t] == (own + shared if t < G0[which] else shared + own), t


def _tile(gft, g, slot):
    return int(gft[g, slot]) if 0 <= g < len(gft) else -1


def _starts_range(gft, g, slot, item_start):
    ft = _tile(gft, g, slot)
    return item_start or ft <= 0 or _tile(gft, g - 1, slot) != ft - 1


def _ends_range(gft, g, slot, item_end):
    return item_end or _tile(gft, g + 1, slot) != _tile(gft, g, slot) + 1


def _fused_layer(gft, x_rows, w2, bias, KH2, KW, FLT, HALO, W, rpw, n_windows, n_split, extra=None):
    """conv_tc_kernel's fused epilogue + edge_fix_kernel for all M-tiles under one work split, with the tiles of every
    group read from the library's group table; returns out [n_windows][T][W] and how each boundary was finished."""
    H = (KH2 - 1) // 2
    MS = MT - 2 * H
    KE = 2 * HALO
    n_rows = n_windows * rpw
    n_mtiles = (n_rows + MS - 1) // MS
    n_ft = (W + FLT - 1) // FLT
    n_groups = len(gft)
    P = _thread_partials(x_rows, w2, KH2, KW, FLT, HALO, W)
    pad = 128 + 8
    out = np.full((n_windows, T, W), np.nan)
    edge = np.full((n_ft - 1, 2, KE, n_mtiles * MS), np.nan)  # [boundary - 1][side]
    how = {}  # (M-tile, boundary) -> "carry" / "edge"

    def finish(b, t, f, val):
        v = val + bias
        if extra is not None:
            v += extra[b, t, f]
        assert np.isnan(out[b, t, f]), "bin finished twice"
        out[b, t, f] = 1.0 / (1.0 + np.exp(-v))

    item_starts = {q * n_groups // n_split for q in range(n_split)}
    for mt in range(n_mtiles):
        m0 = mt * MS - H
        for q in range(n_split):
            g0, g1 = q * n_groups // n_split, (q + 1) * n_groups // n_split
            for slot in range(2):
                carry, prev = np.zeros((KE, MT)), None
                for g in range(g0, g1):
                    ft = _tile(gft, g, slot)
                    if ft < 0:
                        continue
                    first = _starts_range(gft, g, slot, g == g0)
                    last = _ends_range(gft, g, slot, g == g1 - 1)
                    S = _time_sum_tile(P[ft][:, :, m0 + pad : m0 + pad + MT], H)
                    lower = ft > 0
                    rows_ok = []
                    for row in range(2 * H, MT):
                        m = m0 + row - H
                        b, t = divmod(m, rpw) if m >= 0 else (0, -1)
                        if m >= 0 and b < n_windows and t < T:
                            rows_ok.append((row, b, t, m))
                    if first:
                        if lower:
                            for row, b, t, R in rows_ok:
                                edge[ft - 1, 0, :, R] = S[:KE, row]
                    else:
                        assert prev == ft - 1, "a carry comes from the tile below"
                        assert (mt, ft) not in how
                        how[(mt, ft)] = "carry"
                        S[:KE] += carry
                    jlo = (KE if lower else HALO) if first else 0
                    jhi = FLT + (HALO if (FLT == 4 and ft == n_ft - 1) else 0)
                    for row, b, t, R in rows_ok:
                        for j in range(jlo, jhi):
                            f = FLT * ft - HALO + j
                            if 0 <= f < W:
                                finish(b, t, f, S[j, row])
                    carry, prev = S[FLT : FLT + KE].copy(), ft
                    if last and ft < n_ft - 1:
                        for row, b, t, R in rows_ok:
                            edge[ft, 1, :, R] = S[FLT : FLT + KE, row]
    # edge_fix_kernel: the boundaries where a range starts under this split
    for ft_b in range(1, n_ft):
        (g,), (slot,) = np.nonzero(gft == ft_b)
        if not _starts_range(gft, g, slot, g in item_starts):
            continue
        for mt in range(n_mtiles):
            assert (mt, ft_b) not in how
            how[(mt, ft_b)] = "edge"
        for R in range(n_rows):
            b, t = divmod(R, rpw)
            if b >= n_windows or t >= T:
                continue
            for k in range(KE):
                f = FLT * ft_b - HALO + k
                if 0 <= f < W:
                    assert not np.isnan(edge[ft_b - 1, :, k, R]).any(), ("edge side never written", ft_b)
                    finish(b, t, f, edge[ft_b - 1, 0, k, R] + edge[ft_b - 1, 1, k, R])
    return out, how, n_mtiles


@pytest.mark.parametrize("which", [0, 1, 2])
def test_every_boundary_is_finished_once_under_every_split(weights_np, which):
    name = CONV2[which]
    key, C, KH2, KW, FLT, HALO, W, rpw, _g0 = CASES[name]
    gft = _plan(which, weights_np[SPECS[which][0]])[4]
    n_ft = _n_ft(which)
    rng = np.random.default_rng(10 + which)
    n_windows = 2
    x = np.maximum(rng.standard_normal((n_windows, C, T, W)), 0.0)
    w_full = weights_np[key].astype(np.float64)
    bias = float(weights_np[key[:-2] + "_b"].reshape(-1)[0])
    if name == "onset2":
        note = rng.random((n_windows, T, W))
        w2, wx = w_full[0, 1:], w_full[0, 0]
        extra = F.conv2d(torch.from_numpy(note)[:, None], torch.from_numpy(wx)[None, None], padding=(1, 1))[:, 0].numpy()
        full_in = np.concatenate([note[:, None], x], axis=1)
    else:
        w2, extra, full_in = w_full[0], None, x
    pad = 128 + 8
    x_rows = np.zeros((C, n_windows * rpw + 2 * pad + 128, W))
    for b in range(n_windows):
        x_rows[:, pad + b * rpw : pad + b * rpw + T, :] = x[b]
    ref = torch.sigmoid(F.conv2d(torch.from_numpy(full_in), torch.from_numpy(w_full), torch.tensor([bias], dtype=torch.float64),
                                 padding=(KH2 // 2, HALO)))[:, 0].numpy()
    d = _pair_distance(which, gft)
    for n_split in range(1, len(gft) + 1):
        got, how, n_mtiles = _fused_layer(gft, x_rows, w2, bias, KH2, KW, FLT, HALO, W, rpw, n_windows, n_split, extra)
        assert set(how) == {(mt, b) for mt in range(n_mtiles) for b in range(1, n_ft)}, n_split
        n_edges = sum(v == "edge" for (mt, _b), v in how.items() if mt == 0)
        if which == 0 and d == 1:
            assert n_edges == n_ft - 1  # every contour tile is a range of its own
        assert not np.isnan(got).any(), (n_split, f"{int(np.isnan(got).sum())} cells never finished")
        assert np.abs(got - ref).max() < 1e-12, n_split
