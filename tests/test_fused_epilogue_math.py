"""CPU: the index arithmetic of the fused second convolutions in the epilogues of the tensor-core kernels
(csrc/tc_conv.cu: the conv2 MMAs with their weight matrix, the time taps from the staged sums, finish_pitch_tile,
finish_contour_tile, edge_fix_kernel),
restated in NumPy with the SAME structure and compared with the direct convolution of the oracle:

  * per frequency tile of FLT bins the thread of a frame reduces relu(conv1) over channels and frequency taps into
    P[dt][j], j = 0 .. FLT + 2*HALO - 1 (output bin FLT*ft - HALO + j),
  * time taps: the thread of tile row r finishes output row r - H, which takes P[dt] of row r - (2H - dt): always a row
    at or below its own, read from the staged sums of the tile; M-tiles advance by 64 - 2H rows, rows 2H .. 63 of a
    tile finish an output row,
  * frequency halo: a slot walks its tile range in ascending order carrying the top 2*HALO sums; where two ranges meet
    (slot 0 | slot 1, group splits) both sides go to the edge buffer and the fix-up adds them.

This pins the halo bookkeeping, tile ranges and zero padding; the GPU tests then only have to prove the kernels."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

CASES = {  # name: (weights key, C_in, KH2, KW, FLT, HALO, W, rows_per_window, G0)
    "contour2": ("contour2_w", 8, 5, 5, 16, 2, 264, 174, 9),
    "note2": ("note2_w", 32, 7, 3, 4, 1, 88, 175, 12),
    "onset2": ("onset2_w", 32, 3, 3, 4, 1, 88, 174, 12),  # channels 1..32 of the 33-channel conv; channel 0 is the note input
}
T = 172
MT = 64  # rows of an M-tile


def _thread_partials(x, w2, KH2, KW, FLT, HALO, W):
    """x: relu(conv1) [C][rows][W] (zero for rows that are not live) -> P[ft][dt][j][row] as the epilogue thread of a row
    accumulates it: input bin fl of the tile feeds output offset j = fl - df + 2*HALO."""
    C, R, _ = x.shape
    n_ft = (W + FLT - 1) // FLT
    J = FLT + 2 * HALO
    P = np.zeros((n_ft, KH2, J, R))
    for ft in range(n_ft):
        for fl in range(FLT):
            g = FLT * ft + fl
            if g >= W:  # bins past the image are zeroed in the epilogue's first pass
                continue
            for df in range(KW):
                j = fl - df + 2 * HALO
                for dt in range(KH2):
                    P[ft, dt, j, :] += np.einsum("cr,c->r", x[:, :, g], w2[:, dt, df])
    return P


def _time_sum_tile(Ptile, H):
    """Ptile [KH2][J][MT] (conv1 rows of one M-tile) -> S [J][MT] like the kernel: the thread of tile row r finishes
    output row r - H and adds tap dt from `a = 2H - dt` rows below it, a = 0 .. 2H in this order."""
    KH2, J, _ = Ptile.shape
    S = np.zeros((J, MT))
    for row in range(MT):
        for a in range(min(2 * H, row) + 1):
            S[:, row] += Ptile[2 * H - a, :, row - a]
    return S


def _fused_layer(x_rows, w2, bias, KH2, KW, FLT, HALO, W, rpw, G0, n_windows, n_split, extra=None):
    """Emulates conv_tc_kernel's fused epilogue + edge_fix_kernel for all M-tiles; returns out [n_windows][T][W]."""
    H = (KH2 - 1) // 2
    MS = MT - 2 * H
    KE = 2 * HALO
    n_rows = n_windows * rpw
    n_mtiles = (n_rows + MS - 1) // MS
    n_ft = (W + FLT - 1) // FLT
    n_groups = G0
    P = _thread_partials(x_rows, w2, KH2, KW, FLT, HALO, W)  # rows indexed by m + pad
    pad = 128 + 8
    out = np.full((n_windows, T, W), np.nan)
    edge = np.full((2 * n_split, 2, KE, n_mtiles * MS), np.nan)

    def finish(b, t, f, val):
        v = val + bias
        if extra is not None:
            v += extra[b, t, f]
        assert np.isnan(out[b, t, f]), "bin finished twice"
        out[b, t, f] = 1.0 / (1.0 + np.exp(-v))

    for mt in range(n_mtiles):
        m0 = mt * MS - H  # row (window, frame) index of tile row 0
        for q in range(n_split):
            g0, g1 = q * n_groups // n_split, (q + 1) * n_groups // n_split
            for slot in range(2):
                e_lo = slot * n_split + q
                e_hi = slot * n_split + q + 1 if q + 1 < n_split else (n_split if slot == 0 else -1)
                carry = np.zeros((KE, MT))
                for g in range(g0, g1):
                    ft = g + slot * G0
                    if ft >= n_ft:
                        continue
                    first, last = g == g0, (g == g1 - 1) or (ft == n_ft - 1)
                    S = _time_sum_tile(P[ft][:, :, m0 + pad : m0 + pad + MT], H)
                    lower = ft > 0
                    rows_ok = []
                    for row in range(2 * H, MT):
                        m = m0 + row - H  # output row of this thread
                        b, t = divmod(m, rpw) if m >= 0 else (0, -1)
                        if m >= 0 and b < n_windows and t < T:
                            rows_ok.append((row, b, t, m))
                    if first:
                        if lower:
                            for row, b, t, R in rows_ok:
                                edge[e_lo, 0, :, R] = S[:KE, row]
                    else:
                        S[:KE] += carry
                    jlo = (KE if lower else HALO) if first else 0
                    jhi = FLT + (HALO if (FLT == 4 and ft == n_ft - 1) else 0)  # pitch layers: the last tile finishes its top bin
                    for row, b, t, R in rows_ok:
                        for j in range(jlo, jhi):
                            f = FLT * ft - HALO + j
                            if 0 <= f < W:
                                finish(b, t, f, S[j, row])
                    carry = S[FLT : FLT + KE].copy()
                    if last and ft < n_ft - 1 and e_hi >= 0:
                        for row, b, t, R in rows_ok:
                            edge[e_hi, 1, :, R] = S[FLT : FLT + KE, row]
    # edge_fix_kernel
    for e in range(2 * n_split):
        es, eq = divmod(e, n_split)
        ft_b = eq * n_groups // n_split + es * G0
        if ft_b <= 0 or ft_b >= n_ft:
            continue
        for R in range(n_rows):
            b, t = divmod(R, rpw)
            if b >= n_windows or t >= T:
                continue
            for k in range(KE):
                f = FLT * ft_b - HALO + k
                if 0 <= f < W:
                    finish(b, t, f, edge[e, 0, k, R] + edge[e, 1, k, R])
    return out


@pytest.mark.parametrize("name,n_split", [("contour2", 1), ("contour2", 4), ("note2", 1), ("note2", 5), ("onset2", 1), ("onset2", 12)])
def test_fused_second_conv_structure(weights_np, name, n_split):
    key, C, KH2, KW, FLT, HALO, W, rpw, G0 = CASES[name]
    assert KW == 2 * HALO + 1
    rng = np.random.default_rng(len(name) + n_split)
    n_windows = 2
    x = np.maximum(rng.standard_normal((n_windows, C, T, W)), 0.0)  # relu(conv1) per window
    w_full = weights_np[key].astype(np.float64)  # [1][C(+1)][KH][KW]
    bias = float(weights_np[key[:-2] + "_b"].reshape(-1)[0])
    PT = KH2 // 2
    if name == "onset2":
        note = rng.random((n_windows, T, W))
        w2, wx = w_full[0, 1:], w_full[0, 0]
        extra = F.conv2d(torch.from_numpy(note)[:, None], torch.from_numpy(wx)[None, None], padding=(1, 1))[:, 0].numpy()
        full_in = np.concatenate([note[:, None], x], axis=1)
    else:
        w2, extra, full_in = w_full[0], None, x
    # rows of the (window, frame) space, generously padded; rows that are not live frames hold zeros (the kernel zeroes
    # relu(conv1) of separator rows: they are the zero padding of the next conv in time)
    pad = 128 + 8
    n_rows = n_windows * rpw
    x_rows = np.zeros((C, n_rows + 2 * pad + 128, W))
    for b in range(n_windows):
        x_rows[:, pad + b * rpw : pad + b * rpw + T, :] = x[b]
    got = _fused_layer(x_rows, w2, bias, KH2, KW, FLT, HALO, W, rpw, G0, n_windows, n_split, extra)
    ref = torch.sigmoid(F.conv2d(torch.from_numpy(full_in), torch.from_numpy(w_full), torch.tensor([bias], dtype=torch.float64),
                                 padding=(PT, HALO)))[:, 0].numpy()
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} cells never finished"
    assert got.shape == ref.shape == (n_windows, T, W)
    assert np.abs(got - ref).max() < 1e-12


def _b2_tiles(which, w2):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    sizes = np.zeros(5, np.int32)
    wc = np.ascontiguousarray(w2, np.float32)
    lib.bp_debug_tc_b2(which, wc.ctypes.data, sizes.ctypes.data, None)
    n_tiles, n2, kh2, width, js = (int(v) for v in sizes)
    tiles = np.zeros((n_tiles, 2, 2, n2, 8), np.uint16)
    lib.bp_debug_tc_b2(which, wc.ctypes.data, sizes.ctypes.data, tiles.ctypes.data)
    f = (tiles.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    full = (f[:, 0] + f[:, 1]).transpose(0, 1, 3, 2).reshape(n_tiles, 16, n2)  # [tile][k][n], hi + lo
    return full, n2, kh2, width, js


@pytest.mark.parametrize("name,which", [("contour2", 0), ("onset2", 1), ("note2", 2)])
def test_conv2_mma_windows_reproduce_thread_partials(weights_np, name, which):
    """The fused conv2 as a second tensor-core contraction (tc_conv.cu, TcB2 / tc_build_b2): the A operand is the row of
    relu(conv1) in accumulator order k = fl * COUT + c; K step ks multiplies elements 16 ks .. 16 ks + 15 by ONE small
    weight tile and accumulates into a window of conv2-accumulator columns (column j * JS + dt) that starts at
    10 ks (contour) / JS * (ks // 2) (onset, note; JS = 4 / 8).  Emulated here with the tiles the library builds (hi + lo planes
    summed) and compared with the per-thread partial sums P[dt][j] the epilogue needs (_thread_partials)."""
    key, C, KH2, KW, FLT, HALO, W, rpw, G0 = CASES[name]
    w2_full = weights_np[key].astype(np.float64)  # [1][C (+1)][KH2][KW]
    w2 = w2_full[0, 1:] if name == "onset2" else w2_full[0]
    tiles, n2, kh2, width, js = _b2_tiles(which, weights_np[key])
    assert kh2 == KH2
    rng = np.random.default_rng(which)
    R = 7
    x = np.abs(rng.standard_normal((C, R, W)))
    P = _thread_partials(x, w2, KH2, KW, FLT, HALO, W)  # [ft][dt][j][row]
    n_ft = (W + FLT - 1) // FLT
    J = FLT + 2 * HALO
    # the library rounds the weights to bf16 hi + lo (~2^-17 relative): compare against partial sums of the same weights
    worst = 0.0
    for ft in range(n_ft):
        a2 = np.zeros((R, 128))
        for fl in range(FLT):
            g = FLT * ft + fl
            if g < W:
                a2[:, fl * C : (fl + 1) * C] = x[:, :, g].T
        d2 = np.zeros((R, width + 32))
        for ks in range(8):
            if which == 0:
                col, tile = 10 * ks, 0
            else:
                col, tile = js * (ks // 2), ks % 2
            assert col % 2 == 0  # the D start column of an MMA must be even
            d2[:, col : col + n2] += a2[:, 16 * ks : 16 * ks + 16] @ tiles[tile]
        assert np.all(d2[:, width:] == 0), "a window writes past the accumulator"
        got = d2[:, : J * js].reshape(R, J, js)
        assert np.all(got[:, :, KH2:] == 0)
        got = got[:, :, :KH2]
        ref = P[ft].transpose(2, 1, 0)  # [row][j][dt]
        worst = max(worst, float(np.abs(got - ref).max()))
    assert worst < 2e-4 * float(np.abs(P).max()), worst  # bf16 hi + lo weights: relative 2^-16
