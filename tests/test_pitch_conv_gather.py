"""CPU: emulate the gathered conv1 of the onset and note layers (csrc/tc_conv.cu, TcGather: an implicit GEMM whose A
operand is gathered from the data tile into registers, against two resident B matrices for even and odd output bins) in
NumPy, with the B matrices, window starts and valid-bin ranges the library builds, and compare it with the direct
convolution of the oracle.  This pins the window placement, the parity variants and the zero gating (outside the input
row, outside the stacked harmonic image); the GPU tests then only have to prove the MMA mechanics."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref
from tests import weightsets

SPECS = {  # which: (weights key, KH, KW, SF, PT, PL, input bins, bins of the data tile)
    1: ("onset1_w", 5, 5, 3, 2, 1, 309, 312),
    2: ("note1_w", 7, 7, 3, 3, 2, 264, 264),  # single input channel: the contour posteriorgram
}
WOUT, COUT = 88, 32


def _gather_plan(which, w):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    wc = np.ascontiguousarray(w, np.float32)
    sizes = np.zeros(4, np.int32)
    lib.bp_debug_tc_gather(which, wc.ctypes.data, sizes.ctypes.data, None, None, None)
    K, n_ci, KH, wout = (int(v) for v in sizes)
    b1 = np.zeros((2, 2, K // 8, COUT, 8), np.uint16)
    starts = np.zeros((wout, n_ci), np.int32)
    ranges = np.zeros((n_ci, 2), np.int32)
    lib.bp_debug_tc_gather(which, wc.ctypes.data, sizes.ctypes.data, b1.ctypes.data, starts.ctypes.data,
                           ranges.ctypes.data)
    f = (b1.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    b = (f[:, 0] + f[:, 1]).transpose(0, 1, 3, 2).reshape(2, K, COUT)  # [parity][k][co], hi + lo
    return b, starts, ranges, K, n_ci, KH, wout


def _emulate(which, w, y):
    """conv1 as the kernel computes it: per output bin f, A[m][8 (dt * n_ci + ci) + j] = x[m + dt][starts[f, ci] + j]
    where ranges[ci] holds the bin, zero elsewhere; D_f = A @ B[f & 1]."""
    key, KH, KW, SF, PT, PL, bins, tile_bins = SPECS[which]
    b, starts, ranges, K, n_ci, kh, wout = _gather_plan(which, w)
    assert (kh, wout, n_ci) == (KH, WOUT, w.shape[1]) and K % 16 == 0 and K >= 8 * KH * n_ci
    assert (starts % 2 == 0).all()  # every A register is one aligned pair of bins
    n_t = y.shape[0]
    # what the data tile holds past the last input bin is not the gather's business: fill it with noise
    rng = np.random.default_rng(7)
    xt = rng.standard_normal((n_t + KH - 1, 512))
    xt[PT : PT + n_t, :bins] = y
    xt[:PT] = 0.0
    xt[PT + n_t :] = 0.0
    out = np.zeros((n_t, WOUT, COUT))
    for f in range(WOUT):
        a = np.zeros((n_t, K))
        for dt in range(KH):
            for ci in range(n_ci):
                lo, hi = ranges[ci]
                for j in range(8):
                    u = starts[f, ci] + j
                    if lo <= u < hi:
                        assert 0 <= u < tile_bins  # a live element never leaves the data tile
                        a[:, 8 * (dt * n_ci + ci) + j] = xt[dt : dt + n_t, u]
        out[:, f] = a @ b[f & 1]
    return out


def _check(which, w):
    key, KH, KW, SF, PT, PL, bins, tile_bins = SPECS[which]
    rng = np.random.default_rng(which)
    n_t = 12
    y = rng.standard_normal((n_t, bins))
    got = _emulate(which, w, y)
    h = model_ref.harmonic_stack(torch.from_numpy(y)[None]) if which == 1 else torch.from_numpy(y)[None, None]
    ref = F.conv2d(F.pad(h, (PL, PL, PT, PT)), torch.from_numpy(w.astype(np.float64)), stride=(1, SF))[0].numpy()
    ref = ref.transpose(1, 2, 0)  # [t][f][co]
    assert ref.shape == got.shape
    tol = 1e-4 * max(1.0, np.abs(ref).max())  # the weights are split to hi + lo bf16 (~2^-16 relative)
    err = np.abs(got - ref).max(axis=(0, 2))
    assert err.max() < tol, (int(err.argmax()), float(err.max()))
    # the bins where the gating matters: the image edges f = 0 / 87, and the upper harmonics that run past bin 309
    for f in (0, 1, 2, 85, 86, 87):
        assert err[f] < tol, (f, err[f])
    if which == 1:
        # shift 101 reaches past bin 309 from f = 70 on (3 f - 1 + 101 + 4 >= 309)
        assert np.abs(ref[:, 70:]).max() > 0.1 and err[70:].max() < tol


@pytest.mark.parametrize("wset", weightsets.NAMES)
@pytest.mark.parametrize("which", [1, 2])
def test_gathered_conv1_reproduces_convolution(which, wset):
    _check(which, weightsets.get(wset)[SPECS[which][0]])


@pytest.mark.parametrize("which", [1, 2])
def test_gather_windows_hold_every_tap(which):
    """Every tap of output bin f lies in its 8-bin window, at offset 0 or 1 (the parity of the first tap): the B matrix
    of f & 1 is the same for every f of that parity."""
    key, KH, KW, SF, PT, PL, bins, tile_bins = SPECS[which]
    w = weightsets.get("trained")[key]
    _, starts, ranges, *_ = _gather_plan(which, w)
    shifts = model_ref.HARMONIC_SHIFTS if which == 1 else [0]
    for f in range(WOUT):
        for ci, s in enumerate(shifts):
            u0 = SF * f - PL + s
            assert starts[f, ci] == u0 - (u0 % 2) and starts[f, ci] + 8 >= u0 + KW
