"""CPU: the K order the onset and note conv1 kernels run (csrc/tc_conv.cu, TcGather, bp_debug_tc_gather_packed): the onset
packs each (time tap, channel) window to 6 bins and orders the bin pairs by a slot map.  Emulate the exact per-lane
register contraction in NumPy against the oracle's direct convolution, and check that every tap has exactly one row and
that the shared-memory loads take the fewest wavefronts any K order allows."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref
from tests import weightsets
from tests.test_pitch_conv_gather import COUT, SPECS, WOUT, _gather_plan


def _packed(which, w):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    wc = np.ascontiguousarray(w, np.float32)
    sizes = np.zeros(1, np.int32)
    lib.bp_debug_tc_gather_packed(which, wc.ctypes.data, sizes.ctypes.data, None, None)
    K = int(sizes[0])
    b1 = np.zeros((2, 2, K // 8, COUT, 8), np.uint16)
    kmap = np.zeros((K, 3), np.int32)
    lib.bp_debug_tc_gather_packed(which, wc.ctypes.data, sizes.ctypes.data, b1.ctypes.data, kmap.ctypes.data)
    f = (b1.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return (f[:, 0] + f[:, 1]).transpose(0, 1, 3, 2).reshape(2, K, COUT), kmap


def _lane_rows(K):
    """k of the bf16 pair of register x[2 h + rr] (K-step ks, lane qd): the wgmma A fragment, k = 16 ks + 8 h + 2 qd."""
    return [(ks, h, qd, 16 * ks + 8 * h + 2 * qd) for ks in range(K // 16) for h in range(2) for qd in range(4)]


@pytest.mark.parametrize("which", [1, 2])
def test_every_tap_has_one_row(which):
    key, KH, KW, SF, PT, PL, bins, tile_bins = SPECS[which]
    _, kmap = _packed(which, weightsets.get("trained")[key])
    K = kmap.shape[0]
    assert K == (240 if which == 1 else 64) and K % 16 == 0
    live = [tuple(r) for r in kmap if r[0] >= 0]
    W = 6 if which == 1 else 8
    n_ci = 8 if which == 1 else 1
    assert sorted(live) == [(dt, ci, j) for dt in range(KH) for ci in range(n_ci) for j in range(W)]
    # a register is one aligned pair: rows 2 i and 2 i + 1 are bins j and j + 1 of one window, j even
    for i in range(0, K, 2):
        a, b = kmap[i], kmap[i + 1]
        assert (a[0] < 0 and b[0] < 0) or (a[:2].tolist() == b[:2].tolist() and a[2] % 2 == 0 and b[2] == a[2] + 1)


def _emulate(which, w, y):
    key, KH, KW, SF, PT, PL, bins, tile_bins = SPECS[which]
    b, kmap = _packed(which, w)
    _, starts, ranges, *_ = _gather_plan(which, w)
    K = kmap.shape[0]
    n_t = y.shape[0]
    rng = np.random.default_rng(7)
    xt = rng.standard_normal((n_t + KH - 1, 512))  # past the input bins the tile holds anything: noise
    xt[PT : PT + n_t, :bins] = y
    xt[:PT] = 0.0
    xt[PT + n_t :] = 0.0
    out = np.zeros((n_t, WOUT, COUT))
    for f in range(WOUT):
        a = np.zeros((n_t, K))
        for ks, h, qd, k in _lane_rows(K):  # what lane qd loads into its register: one pair, masked per bin
            dt, ci, j = kmap[k]
            if dt < 0:
                continue
            lo, hi = ranges[ci]
            for e in range(2):
                u = starts[f, ci] + j + e
                if lo <= u < hi:
                    assert 0 <= u < tile_bins
                    a[:, k + e] = xt[dt : dt + n_t, u]
        out[:, f] = a @ b[f & 1]
    return out


@pytest.mark.parametrize("wset", weightsets.NAMES)
@pytest.mark.parametrize("which", [1, 2])
def test_packed_conv1_reproduces_convolution(which, wset):
    key, KH, KW, SF, PT, PL, bins, tile_bins = SPECS[which]
    w = weightsets.get(wset)[key]
    rng = np.random.default_rng(which)
    n_t = 12
    y = rng.standard_normal((n_t, bins))
    got = _emulate(which, w, y)
    h = model_ref.harmonic_stack(torch.from_numpy(y)[None]) if which == 1 else torch.from_numpy(y)[None, None]
    ref = F.conv2d(F.pad(h, (PL, PL, PT, PT)), torch.from_numpy(w.astype(np.float64)), stride=(1, SF))[0].numpy()
    ref = ref.transpose(1, 2, 0)
    tol = 1e-4 * max(1.0, np.abs(ref).max())
    err = np.abs(got - ref).max(axis=(0, 2))
    assert err.max() < tol, (int(err.argmax()), float(err.max()))
    for f in (0, 1, 85, 86, 87):
        assert err[f] < tol, (f, err[f])
    if which == 1:  # harmonic 101 runs past bin 309 from f = 70 on
        assert np.abs(ref[:, 70:]).max() > 0.1 and err[70:].max() < tol


@pytest.mark.parametrize("which", [1, 2])
def test_gather_loads_take_fewest_wavefronts(which):
    """A lane's loads over the eight quads (eight consecutive 16-byte rows) fill the eight banks of its bin pair's index
    mod 4, so an instruction takes as many wavefronts as the most lanes of its quad share a class.  The note (8-bin
    windows) is conflict-free; the onset's 6-bin windows cannot be (per time tap the 24 pairs fall unevenly into the
    four classes), and its slot map must reach that lower bound at every output bin."""
    key, KH, KW, SF, PT, PL, bins, tile_bins = SPECS[which]
    w = weightsets.get("trained")[key]
    _, kmap = _packed(which, w)
    _, starts, *_ = _gather_plan(which, w)
    K = kmap.shape[0]
    rows = _lane_rows(K)
    for f in range(WOUT):
        total, per_tap = 0, {}
        for ks in range(K // 16):
            for h in range(2):
                cls = []
                for _, _, qd, k in [r for r in rows if r[0] == ks and r[1] == h]:
                    dt, ci, j = kmap[k]
                    if dt >= 0:
                        cls.append(((starts[f, ci] + j) // 2) % 4)
                        per_tap.setdefault(dt, []).append(cls[-1])
                total += max(np.bincount(cls, minlength=4)) if cls else 0
        if which == 2:
            assert total == 2 * (K // 16) - 1  # every instruction one wavefront (the last half is K padding)
        else:
            # per time tap the classes fall 5 / 6 / 6 / 7 (even f) or 5 / 8 / 3 / 8 (odd f): 7 and 9 wavefronts for
            # 6 instructions are the least any grouping of the 24 pairs into quads can take
            counts = sorted(np.bincount(per_tap[0], minlength=4).tolist())
            assert counts == ([5, 6, 6, 7] if f % 2 == 0 else [3, 5, 8, 8]), (f, counts)
            assert total == 5 * (7 if f % 2 == 0 else 9), (f, total)
