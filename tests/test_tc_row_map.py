"""CPU: the row maps of the tensor-core convs (tc_row_map, csrc/tc_conv.cu, bp_debug_tc_row_map).

The unwrapping entry points keep frames [15, 15 + r) of every window (r = UnwrapDesc::rows).  Every conv has time
stride 1, so going back from the kept frames through the network (onset conv2 3 time taps, onset conv1 5, note conv2 7,
note conv1 7, contour conv2 5, contour conv1 3) each stage needs a band of frames around them.  A NumPy restatement
checks, for random and edge r, that every frame of that dependency cone is a live row of its own window, that a live
row reads nothing outside its window or outside frames [0, 172), that the contour's live outputs are exactly the note
layer's input rows, and that the rows add up.  The uniform map (bp_forward_*) must be today's layout: 172 frames every
rows_per_window rows, nothing trimmed."""
import numpy as np
import pytest

KEEP0, FRAMES = 15, 172
RPW = {0: 174, 1: 174, 2: 175}  # tc_spec(layer).rows_per_window
KH = {0: 3, 1: 5, 2: 7}  # conv1 time taps
KH2 = {0: 5, 1: 3, 2: 7}  # fused conv2 time taps


def row_map(which, trimmed, kept):
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    kept = np.ascontiguousarray(kept, np.int32)
    out = np.zeros((max(len(kept), 1), 3), np.int32)
    info = np.zeros(3, np.int32)
    lib.bp_debug_tc_row_map(which, int(trimmed), kept.ctypes.data, len(kept), out.ctypes.data, info.ctypes.data)
    return out[: len(kept)], int(info[0]), int(info[1]), int(info[2])


def spans(m, lo):
    """per window: the frames [a, b) of its rows i with lo <= i < rows - lo"""
    return [(f + lo, f + r - lo) if r - 2 * lo > 0 else (0, 0) for _b, f, r in m]


def covers(span, need):
    return need[0] >= need[1] or (span[0] <= need[0] and need[1] <= span[1])


KEPT = [[142] * 7, [142, 142, 13], [1], [141], [142], [0], [-15, 142], [142, 0, 1, 141, -3, 13, 142]]


@pytest.mark.parametrize("kept", KEPT + [list(np.random.default_rng(s).integers(-15, 143, 40)) for s in range(4)])
def test_trimmed_map_covers_the_dependency_cone(kept):
    maps = {l: row_map(l, True, kept) for l in range(3)}
    for l, (m, total, lo1, lo2) in maps.items():
        rows = m[:, 2]
        # rows add up, windows back to back in order, none for a window that keeps nothing
        assert total == int(rows.sum()), (l, total)
        assert np.array_equal(m[:, 0], np.concatenate([[0], np.cumsum(rows)[:-1]])), l
        for (base, first, r), k in zip(m, kept):
            assert (r == 0) == (k <= 0), (l, k, r)
        h2, pt = (KH2[l] - 1) // 2, (KH[l] - 1) // 2
        assert lo2 == lo1 + h2 and lo1 >= pt, (l, lo1, lo2)
        for (base, first, r) in m:
            if r == 0:
                continue
            # a live conv1 row reads input rows i - pt .. i + pt of its own window, frames inside [0, 172)
            assert lo1 - pt >= 0 and first >= 0 and first + r <= FRAMES, (l, first, r)
    # what each stage needs, from the kept frames back (the frames of the stage's rows, per window)
    for b, k in enumerate(kept):
        r = max(0, min(int(k), 142))
        kept_span = (KEEP0, KEEP0 + r)
        grow = lambda s, n: (s[0] - n, s[1] + n) if s[1] > s[0] else s  # noqa: E731
        need = {}
        need[(1, "out")] = kept_span
        need[(1, "c1")] = grow(need[(1, "out")], 1)
        need[(1, "in")] = grow(need[(1, "c1")], 2)
        need[(2, "out")] = grow(need[(1, "out")], 1)  # the onset conv2 reads note frames t - 1 .. t + 1
        need[(2, "c1")] = grow(need[(2, "out")], 3)
        need[(2, "in")] = grow(need[(2, "c1")], 3)
        need[(0, "out")] = need[(2, "in")]
        need[(0, "c1")] = grow(need[(0, "out")], 2)
        need[(0, "in")] = grow(need[(0, "c1")], 1)
        for (l, what), s in need.items():
            m, _total, lo1, lo2 = maps[l]
            lo = {"in": 0, "c1": lo1, "out": lo2}[what]
            assert covers(spans(m, lo)[b], s), (l, what, b, k, spans(m, lo)[b], s)
            assert s[1] <= s[0] or (0 <= s[0] and s[1] <= FRAMES), (l, what, s)
        # the contour's live outputs are the note layer's input rows, one to one (TcOut::chl_map)
        mc, _, _, lo2c = maps[0]
        mn = maps[2][0]
        assert spans(mc, lo2c)[b] == spans(mn, 0)[b] or (mn[b, 2] == 0 and spans(mc, lo2c)[b] == (0, 0)), b
    # the onset shares the split of y with the contour
    assert np.array_equal(maps[0][0], maps[1][0]) and maps[0][1] == maps[1][1]


@pytest.mark.parametrize("n", [1, 7, 184])
def test_uniform_map_is_the_whole_window_layout(n):
    kept = np.full(n, 142, np.int32)
    for l in range(3):
        m, total, lo1, lo2 = row_map(l, False, kept)
        assert total == n * RPW[l] and lo1 == 0 and lo2 == 0, (l, total, lo1, lo2)
        assert np.array_equal(m[:, 0], np.arange(n) * RPW[l]) and (m[:, 1] == 0).all() and (m[:, 2] == FRAMES).all(), l
