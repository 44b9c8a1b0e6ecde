"""CPU: the items one launch of a tensor-core conv kernel runs (tc_schedule, csrc/tc_conv.cu), as the library exports them
(bp_debug_tc_schedule):

  * every (M-tile, frequency group) of the launch is in exactly one item, for every batch size of a chunk and every
    layer, on 132 and 114 SMs; the first n_full M-tiles run whole, as many per CTA, the rest in group ranges,
  * the fused epilogue + edge_fix_kernel restated under the schedule (whole and cut M-tiles, each with its own edge
    mask) finish every tile boundary of every M-tile exactly once, by the register carry or the edge buffer, and give
    the direct convolution,
  * at the bench's full and last chunk on 132 SMs the busiest CTA's estimated work is within 3 % of the mean, where the
    uniform cut of every M-tile into k equal group runs left it up to 26 % above."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_fused_epilogue_math import CASES, MT, T, _thread_partials, _time_sum_tile
from tests.test_tc_pairing import CONV2, _ends_range, _n_ft, _starts_range, _tile
from tests.test_tc_plan import SPECS, _plan

NOUSE = 0xFFFFFFFF
# (layer, fused): the contour runs fused on forward path 1 and unfused (activations stored) on path 2
LAUNCHES = [(0, 1), (0, 0), (1, 1), (2, 1)]
# cost model of tc_schedule: contour: MMA uses + 14 per tile, 20 per item; onset / note: tiles, 0.25 per item
EPI_USES, ITEM_USES, ITEM_TILES = 14.0, 20.0, 0.25


def _chunk(n_sms):
    """windows per chunk (bp_model_create): 2 * n_sms spans of 122 rows of the note layer"""
    return max(1, 2 * n_sms * (128 - 6) // 175)


def schedule(which, fused, n_windows, n_sms):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    sizes = np.zeros(8, np.int32)
    lib.bp_debug_tc_schedule(which, fused, n_windows, n_sms, sizes.ctypes.data, None, None)
    items = np.zeros((int(sizes[0]), 3), np.int32)
    edges = np.zeros(2, np.uint32)
    lib.bp_debug_tc_schedule(which, fused, n_windows, n_sms, sizes.ctypes.data, items.ctypes.data, edges.ctypes.data)
    keys = ("n_items", "grid", "n_mtiles", "n_full", "n_ranges", "ms", "tail_row0", "G0")
    return dict(zip(keys, (int(v) for v in sizes))), items, (int(edges[0]), int(edges[1]))


@pytest.mark.parametrize("n_sms", [132, 114])
@pytest.mark.parametrize("which,fused", LAUNCHES)
def test_every_group_of_every_mtile_runs_once(which, fused, n_sms):
    rpw = CASES[CONV2[which]][7]
    for n in range(1, _chunk(n_sms) + 1):
        s, items, _ = schedule(which, fused, n, n_sms)
        G0, ms = s["G0"], s["ms"]
        assert ms == (64 if (which, fused) == (0, 0) else MT - (CASES[CONV2[which]][2] - 1))
        assert s["n_mtiles"] == -(-n * rpw // ms)
        assert s["grid"] == min(n_sms, s["n_items"]) and s["n_full"] % n_sms == 0 and s["n_mtiles"] - s["n_full"] < n_sms
        count = np.zeros((s["n_mtiles"], G0), np.int32)
        for it, (mt, g0, g1) in enumerate(items):
            assert 0 <= g0 < g1 <= G0, (n, it)
            if it < s["n_full"]:
                assert (mt, g0, g1) == (it, 0, G0), (n, it)
            count[mt, g0:g1] += 1
        assert (count == 1).all(), (which, fused, n, n_sms)
        # the cut M-tiles share one set of group ranges
        tail = {(int(g0), int(g1)) for _mt, g0, g1 in items[s["n_full"]:]}
        assert len(tail) == (s["n_ranges"] if s["n_mtiles"] > s["n_full"] else 0), (n, tail)


def _group_costs(which, weights_np):
    gft = _plan(which, weights_np[SPECS[which][0]])[4]
    tiles = (gft >= 0).sum(axis=1).astype(np.float64)
    if which != 0:
        return tiles, ITEM_TILES
    _t, _seq, words, gso, _gft, _n = _plan(0, weights_np["contour1_w"])
    uses = np.array([(words[:, gso[g]:gso[g + 1]] != NOUSE).sum() for g in range(len(gso) - 1)], np.float64)
    return uses + EPI_USES * tiles, ITEM_USES


def _cta_costs(items, grid, n_sms, cost, item):
    busy = np.zeros(n_sms)
    for it, (_mt, g0, g1) in enumerate(items):
        busy[it % grid] += cost[g0:g1].sum() + item
    return busy


def _uniform_items(n_mtiles, G0, n_sms):
    """the uniform cut the kernels ran before: split k of the least (waves x (groups per run + 0.5)), item (it / k, it % k)"""
    best, k = 1e30, 1
    for s in range(1, G0 + 1):
        c = -(-n_mtiles * s // n_sms) * (-(-G0 // s) + 0.5)
        if c < best - 1e-9:
            best, k = c, s
    return np.array([(it // k, (it % k) * G0 // k, (it % k + 1) * G0 // k) for it in range(n_mtiles * k)], np.int32)


@pytest.mark.parametrize("n_windows", [184, 102])
@pytest.mark.parametrize("which,fused", LAUNCHES)
def test_busiest_cta_within_3_percent_of_the_mean(weights_np, which, fused, n_windows):
    n_sms = 132
    cost, item = _group_costs(which, weights_np)
    s, items, _ = schedule(which, fused, n_windows, n_sms)
    busy = _cta_costs(items, s["grid"], n_sms, cost, item)
    old = _uniform_items(s["n_mtiles"], s["G0"], n_sms)
    busy_old = _cta_costs(old, min(len(old), n_sms), n_sms, cost, item)
    print(f"layer {which} fused {fused}, {n_windows} windows: busiest CTA / mean {busy.max() / busy.mean():.4f} "
          f"(uniform cut: {busy_old.max() / busy_old.mean():.4f}); {s['n_full']} whole M-tiles, "
          f"{s['n_mtiles'] - s['n_full']} in {s['n_ranges']} ranges")
    assert busy.max() <= 1.03 * busy.mean()
    assert busy.max() <= busy_old.max()


def _fused_layer(gft, x_rows, w2, bias, KH2, KW, FLT, HALO, W, rpw, n_windows, items, edges, tail_row0, extra=None):
    """conv_tc_kernel's fused epilogue over the items of a schedule + edge_fix_kernel with the edge mask of the M-tile
    that finishes each row; returns out [n_windows][T][W] and how each (M-tile, boundary) was finished."""
    H = (KH2 - 1) // 2
    MS = MT - 2 * H
    KE = 2 * HALO
    n_rows = n_windows * rpw
    n_mtiles = (n_rows + MS - 1) // MS
    n_ft = (W + FLT - 1) // FLT
    P = _thread_partials(x_rows, w2, KH2, KW, FLT, HALO, W)
    pad = 128 + 8
    out = np.full((n_windows, T, W), np.nan)
    edge = np.full((n_ft - 1, 2, KE, n_mtiles * MS), np.nan)
    how = {}

    def finish(b, t, f, val):
        v = val + bias
        if extra is not None:
            v += extra[b, t, f]
        assert np.isnan(out[b, t, f]), "bin finished twice"
        out[b, t, f] = 1.0 / (1.0 + np.exp(-v))

    for mt, g0, g1 in items:
        m0 = mt * MS - H
        rows_ok = []
        for row in range(2 * H, MT):
            m = m0 + row - H
            b, t = divmod(m, rpw) if m >= 0 else (0, -1)
            if m >= 0 and b < n_windows and t < T:
                rows_ok.append((row, b, t, m))
        for slot in range(2):
            carry, prev = None, None
            for g in range(g0, g1):
                ft = _tile(gft, g, slot)
                if ft < 0:
                    continue
                first = _starts_range(gft, g, slot, g == g0)
                last = _ends_range(gft, g, slot, g == g1 - 1)
                S = _time_sum_tile(P[ft][:, :, m0 + pad : m0 + pad + MT], H)
                lower = ft > 0
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
    # edge_fix_kernel: row R takes the mask of the M-tile R // MS that finishes it
    for mt in range(n_mtiles):
        mask = edges[0] if mt * MS < tail_row0 else edges[1]
        for ft_b in range(1, n_ft):
            if mask >> ft_b & 1:
                assert (mt, ft_b) not in how, ("boundary finished by the carry and the edge fix", mt, ft_b)
                how[(mt, ft_b)] = "edge"
    for R in range(n_rows):
        b, t = divmod(R, rpw)
        if b >= n_windows or t >= T:
            continue
        mask = edges[0] if R < tail_row0 else edges[1]
        for ft_b in range(1, n_ft):
            if not mask >> ft_b & 1:
                continue
            for k in range(KE):
                f = FLT * ft_b - HALO + k
                if 0 <= f < W:
                    assert not np.isnan(edge[ft_b - 1, :, k, R]).any(), ("edge side never written", ft_b, R)
                    finish(b, t, f, edge[ft_b - 1, 0, k, R] + edge[ft_b - 1, 1, k, R])
    return out, how, n_mtiles


@pytest.mark.parametrize("which", [0, 1, 2])
def test_every_boundary_is_finished_once_under_the_schedule(weights_np, which):
    """Two windows on 1 .. 6 SMs and on 132: every mix of whole and cut M-tiles and every number of ranges the
    planner picks for them"""
    name = CONV2[which]
    key, C, KH2, KW, FLT, HALO, W, rpw, _g0 = CASES[name]
    gft = _plan(which, weights_np[SPECS[which][0]])[4]
    n_ft = _n_ft(which)
    rng = np.random.default_rng(20 + which)
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
    seen = set()
    for n_sms in (1, 2, 3, 4, 5, 6, 132):
        s, items, edges = schedule(which, 1, n_windows, n_sms)
        seen.add((s["n_full"] > 0, s["n_mtiles"] > s["n_full"], s["n_ranges"]))
        got, how, n_mtiles = _fused_layer(gft, x_rows, w2, bias, KH2, KW, FLT, HALO, W, rpw, n_windows, items, edges,
                                          s["tail_row0"], extra)
        assert set(how) == {(mt, b) for mt in range(n_mtiles) for b in range(1, n_ft)}, n_sms
        if which == 0:
            assert edges == (0x1FFFE, 0x1FFFE)  # every contour tile is a range of its own
        else:
            assert edges[0] == 1 << 12  # whole M-tiles: the slot boundary only
        assert not np.isnan(got).any(), (n_sms, f"{int(np.isnan(got).sum())} cells never finished")
        assert np.abs(got - ref).max() < 1e-12, n_sms
    # whole and cut M-tiles in one launch, and cut M-tiles in several ranges, were both reached
    assert any(f and t for f, t, _r in seen) and any(t and r > 1 for _f, t, r in seen), seen
