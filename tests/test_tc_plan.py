"""CPU: emulate the tensor-core programs of the contour and onset convolutions (csrc/tc_conv.cu, built by the host
code inside libbp_b200.so) in NumPy and compare with the direct convolution of the oracle.  This pins the
Toeplitz / aligned-chunk decomposition, the harmonic-stack folding and the edge gating; the GPU tests then only have
to prove the MMA mechanics."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model_ref
from tests import weightsets

SPECS = {  # which: (weights key, KH, KW, SF, PT, PL, COUT, FLT, WOUT)
    0: ("contour1_w", 3, 39, 1, 1, 19, 8, 16, 264),
    1: ("onset1_w", 5, 5, 3, 2, 1, 32, 4, 88),
    2: ("note1_w", 7, 7, 3, 3, 2, 32, 4, 88),  # single input channel: the contour posteriorgram (264 bins)
}


def _bf16_to_f32(u16):
    return (u16.astype(np.uint32) << 16).view(np.float32)


def _plan(which, w):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    sizes = np.zeros(4, np.int32)
    wc = np.ascontiguousarray(w, np.float32)
    lib.bp_debug_tc_plan(which, wc.ctypes.data, sizes.ctypes.data, None, None, None, None, None)
    n_tiles, n_steps, n_uses, n_groups = (int(x) for x in sizes)
    tiles = np.zeros((n_tiles, 2, 2, 128, 8), np.uint16)
    tile_seq = np.zeros(n_steps, np.int32)
    slot_words = np.zeros((2, n_steps), np.uint32)
    gso = np.zeros(n_groups + 1, np.int32)
    gft = np.zeros((n_groups, 2), np.int32)
    lib.bp_debug_tc_plan(which, wc.ctypes.data, sizes.ctypes.data, tiles.ctypes.data, tile_seq.ctypes.data,
                         slot_words.ctypes.data, gso.ctypes.data, gft.ctypes.data)
    return tiles, tile_seq, slot_words, gso, gft, n_uses


@pytest.mark.parametrize("which", [0, 1, 2])
def test_tc_program_reproduces_convolution(weights_np, which):
    _check_program_reproduces_convolution(which, weights_np[SPECS[which][0]])


@pytest.mark.parametrize("wset", [n for n in weightsets.NAMES if n != "trained"])
@pytest.mark.parametrize("which", [0, 1, 2])
def test_tc_program_reproduces_convolution_synthetic_weights(which, wset):
    """The same emulation under the synthetic weight sets: every tap non-zero (dense), only the outermost taps
    (edge_taps), one centre tap per channel pair (sparse, whose tiles used to de-duplicate into a different program)."""
    _check_program_reproduces_convolution(which, weightsets.get(wset)[SPECS[which][0]])


def _check_program_reproduces_convolution(which, w):
    key, KH, KW, SF, PT, PL, COUT, FLT, WOUT = SPECS[which]
    tiles, tile_seq, slot_words, gso, gft, n_uses = _plan(which, w)
    n_groups = len(gft)
    assert gso[0] == 0 and gso[-1] == len(tile_seq) < 1023 and n_groups <= 15  # constant-memory program area
    tf = _bf16_to_f32(tiles).astype(np.float64)
    t_full = (tf[:, 0] + tf[:, 1]).transpose(0, 1, 3, 2).reshape(len(tiles), 16, 128)  # [tile][k][n]
    rng = np.random.default_rng(which)
    n_t = 40
    bins = 309 if which < 2 else 264
    y = rng.standard_normal((n_t, bins))
    # the kernel's tile row (i + dt) holds input frame i + dt - PT
    ypad = np.zeros((n_t + KH - 1, 320))
    ypad[PT : PT + n_t, :bins] = y
    n_ft = (WOUT + FLT - 1) // FLT
    out = np.zeros((n_t, n_ft * 128))
    lbo16 = 64 + KH - 1  # the program is built for 64-row M-tiles
    seen_ft = set()
    used = 0
    for g in range(n_groups):
        first_seen = set()
        for step in range(gso[g], gso[g + 1]):
            for slot in (0, 1):
                wd = int(slot_words[slot, step])
                if wd == 0xFFFFFFFF:
                    continue
                used += 1
                aoff16, first_acc = wd & 0x3FFF, (wd >> 15) & 1
                assert wd >> 16 == 0
                c8, dt = divmod(aoff16, lbo16)  # 8-bin chunk index of the step's first k-chunk, time tap
                assert dt < KH and 8 * c8 + 16 <= 320
                ft = int(gft[g, slot])
                assert ft >= 0
                assert bool(first_acc) == (slot not in first_seen)
                first_seen.add(slot)
                a = ypad[dt : dt + n_t, 8 * c8 : 8 * c8 + 16]
                out[:, 128 * ft : 128 * ft + 128] += a @ t_full[tile_seq[step]]
        for slot in (0, 1):
            if gft[g, slot] >= 0:
                assert gft[g, slot] not in seen_ft and slot in first_seen
                seen_ft.add(int(gft[g, slot]))
    assert seen_ft == set(range(n_ft)) and used == n_uses
    got = out.reshape(n_t, n_ft * FLT, COUT)[:, :WOUT]  # n = fl * COUT + co
    h = model_ref.harmonic_stack(torch.from_numpy(y)[None]) if which < 2 else torch.from_numpy(y)[None, None]
    ref = F.conv2d(F.pad(h, (PL, PL, PT, PT)), torch.from_numpy(w.astype(np.float64)), stride=(1, SF))[0].numpy()
    assert ref.shape == (COUT, n_t, WOUT)
    err = np.abs(got - ref.transpose(1, 2, 0)).max()
    assert err < 1e-3 * max(1.0, np.abs(ref).max() / 10), err  # limited by the 16-bit (hi+lo) weights


def test_tc_program_statistics(weights_np):
    for which in (0, 1, 2):
        key = SPECS[which][0]
        tiles, tile_seq, slot_words, gso, gft, n_uses = _plan(which, weights_np[key])
        assert (tile_seq >= 0).all() and (tile_seq < len(tiles)).all()
        print(which, "tiles", len(tiles), "steps", len(tile_seq), "uses", n_uses)
        assert len(tiles) < 700 and n_uses < 2200


def test_tc_program_is_independent_of_the_weights():
    """The MMA programs live in process-wide __constant__ memory that every model shares, so they must be a function of
    the layer geometry alone: tile ids, tile count, step sequence, slot words, group offsets and group tiles are the same
    under every weight set.  (`sparse` gives all (co, ci) pairs the same weight pattern: de-duplicating tiles by value
    used to merge many of them and produce a different, smaller program.)"""
    for which in (0, 1, 2):
        key = SPECS[which][0]
        ref = None
        for wset in weightsets.NAMES:
            tiles, tile_seq, slot_words, gso, gft, n_uses = _plan(which, weightsets.get(wset)[key])
            prog = (len(tiles), tile_seq, slot_words, gso, gft, n_uses)
            if ref is None:
                ref = prog
                continue
            assert prog[0] == ref[0], (which, wset, "n_tiles", prog[0], ref[0])
            assert prog[5] == ref[5], (which, wset, "n_uses")
            for name, a, b in zip(("tile_seq", "slot_words", "group_step_off", "group_ft"), prog[1:5], ref[1:5]):
                np.testing.assert_array_equal(a, b, err_msg=f"layer {which}, {wset}: {name}")
