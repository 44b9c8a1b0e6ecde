"""CPU: the rule of a live PCM stream (bp_stream_group_open_pcm, include/bp_b200.h, DESIGN.md §4.6) through
bp_debug_pcm_stream_plan, the host function every PCM push calls, against the rule restated in NumPy; and the Python
validation of PCM blocks, which raises before any call into the library."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_ingest import RATES, design


def geometry(sr):
    """(up, down, half, T) of the resampler from sr to 22 050 Hz; the identity at 22 050 Hz."""
    if sr == 22050:
        return 1, 1, 0, 1
    up, down, _h, T, half = design(sr)
    return up, down, half, T


def final(n, up, down, half):
    """F(n) = max(0, ceil((n up - half) / down)): the outputs whose inputs have all arrived after n frames."""
    return max(0, -((half - n * up) // down))


def plan(sr, frames, ending=True, fmt=1, channels=2):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    fr = np.ascontiguousarray(frames, np.int64)
    m = len(fr) + (1 if ending else 0)
    out = [np.full(m, -7, np.int64) for _ in range(4)]
    lib.bp_debug_pcm_stream_plan(fmt, channels, sr, len(fr), fr.ctypes.data if len(fr) else None, int(ending),
                                 *[o.ctypes.data for o in out])
    return out


def schedules(sr, rng):
    """Block schedules: 0- and 1-frame blocks, blocks shorter than T, a second's worth, a recording shorter than
    half / up frames, one of one frame, an empty one, and random mixes."""
    up, down, half, T = geometry(sr)
    short = max(0, half // up - 1)
    out = [[], [0], [1], [0, 0, 1, 0], [short], [1] * 7 + [0, 2], [max(1, T - 1), 1, T, T + 1], [sr, 0, sr // 3 + 1]]
    for _ in range(4):
        k = int(rng.integers(1, 12))
        out.append([int(rng.choice([0, 1, 2, max(1, T // 2), T - 1 if T > 1 else 1, T + 3, 1000, 9_973]))
                    for _ in range(k)])
    return out


@pytest.mark.parametrize("sr", RATES)
def test_plan_follows_the_rule(sr):
    """Per push of every schedule: the outputs made final are [F(n_before), F(n_after)), the end adds the rest, the
    ranges partition [0, bp_resampled_length(n)), every input an output reads is held, new or zero fill, and the
    history is [i_max(F(n)) - T + 1, n) clipped at 0, never more than T - 1 floats."""
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    up, down, half, T = geometry(sr)
    rng = np.random.default_rng(sr)
    for frames in schedules(sr, rng):
        out_lo, out_hi, hist_lo, hist_hi = plan(sr, frames)
        n, prev_lo, k_next = 0, 0, 0
        for p in range(len(frames) + 1):
            ending = p == len(frames)
            n_after = n + (0 if ending else frames[p])
            F = final(n_after, up, down, half)
            exp_hi = -(-(n_after * up) // down) if ending else F
            assert out_lo[p] == k_next == final(n, up, down, half), (sr, frames, p)
            assert out_hi[p] == exp_hi, (sr, frames, p)
            k = np.arange(out_lo[p], out_hi[p], dtype=np.int64)
            if len(k):
                i_max = (k * down + half) // up
                lo = i_max - T + 1
                # every input read: below 0 (zero), in the held history or the new block, or past the end once ended
                assert np.all((np.maximum(lo, 0) >= prev_lo) | (i_max < 0)), (sr, frames, p)
                if not ending:
                    assert np.all(i_max < n_after), (sr, frames, p)
            assert hist_hi[p] == n_after
            if ending:
                assert hist_lo[p] == hist_hi[p]
            else:
                exp_lo = min(n_after, max(0, (F * down + half) // up - T + 1))
                assert hist_lo[p] == exp_lo, (sr, frames, p)
                assert 0 <= hist_hi[p] - hist_lo[p] <= T - 1, (sr, frames, p)
            prev_lo, k_next, n = hist_lo[p], out_hi[p], n_after
        assert k_next == lib.bp_resampled_length(n, sr), (sr, frames)
        if not frames or sum(frames) == 0:
            assert k_next == 0


def test_plan_without_end_and_same_rate():
    """Without the end no entry for it; at 22 050 Hz every frame is final at once and nothing is held."""
    frames = [0, 5, 1, 300]
    out_lo, out_hi, hist_lo, hist_hi = plan(22050, frames, ending=False, fmt=3, channels=3)
    assert list(out_lo) == [0, 0, 5, 6] and list(out_hi) == [0, 5, 6, 306]
    assert list(hist_lo) == list(hist_hi) == [0, 5, 6, 306]


def test_plan_refuses_what_open_refuses():
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    o = [np.zeros(2, np.int64) for _ in range(4)]
    fr = np.array([3], np.int64)
    for fmt, ch, sr in ((4, 1, 48000), (-1, 1, 48000), (1, 0, 48000), (1, 1, 0), (1, 1, 2_822_400)):
        with pytest.raises(_lib.BpError) as e:
            lib.bp_debug_pcm_stream_plan(fmt, ch, sr, 1, fr.ctypes.data, 1, *[x.ctypes.data for x in o])
        assert e.value.code == _lib.BP_E_INVALID
    with pytest.raises(_lib.BpError):
        lib.bp_debug_pcm_stream_plan(1, 1, 48000, 1, np.array([-1], np.int64).ctypes.data, 1, *[x.ctypes.data for x in o])


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"{name} called for a block that should have been refused")


def _group_without_device(pcm):
    from basic_pitch_b200.inference import StreamGroup

    g = object.__new__(StreamGroup)
    g._lib, g._h, g._pcm, g._bends = _NoLib(), None, dict(pcm), True
    return g


def test_pcm_blocks_are_validated_before_the_library():
    """A block of the wrong dtype, channel count or shape raises ValueError in StreamGroup.push before any library
    call; (n,) is taken for a one-channel stream only."""
    from basic_pitch_b200.inference import _pcm_block, _pcm_format

    g = _group_without_device({0: (np.dtype(np.int16), 2), 1: (np.dtype(np.uint8), 1)})
    bad = [
        {0: np.zeros((10, 2), np.int32)},
        {0: np.zeros((10, 2), np.float32)},
        {0: np.zeros((10, 3), np.int16)},
        {0: np.zeros(10, np.int16)},
        {0: np.zeros((10, 2, 1), np.int16)},
        {1: np.zeros((4, 2), np.uint8)},
        {1: np.zeros(4, np.int8)},
        {1: np.zeros(4, np.uint8), 0: np.zeros((3, 1), np.int16)},
    ]
    for blocks in bad:
        with pytest.raises(ValueError):
            g.push(blocks)
    assert _pcm_block(np.zeros(4, np.uint8), np.dtype(np.uint8), 1).shape == (4, 1)
    b = _pcm_block(np.zeros((6, 2), np.int16)[::1], np.dtype(np.int16), 2)
    assert b.shape == (6, 2) and b.flags.c_contiguous
    assert [_pcm_format(d) for d in (np.float32, np.int16, np.int32, np.uint8)] == [0, 1, 2, 3]
    for d in (np.float64, np.int8, np.uint16, np.int64):
        with pytest.raises(ValueError):
            _pcm_format(d)
