"""CPU: posteriorgrams read as multi-f0 estimates (include/bp_b200.h, bp_score_salience_grid_*): the bin tables of
evaluate.salience_bins, the host definition evaluate.salience_to_multipitch against a per-cell loop on hand-made
posteriorgrams, the settings' conversion to bins, and the chunk size of bp_score_salience_chunk_params."""
import numpy as np
import pytest

from basic_pitch_b200 import constants, evaluate


def _per_cell(gram, threshold, peak, lo, hi, hz):
    """The rule of include/bp_b200.h cell by cell: range, float64 threshold, float32 strict peak on the whole row."""
    out = []
    for row in np.asarray(gram, np.float32):
        w, vals = len(row), []
        for b in range(w):
            v = row[b]
            if not lo <= b < hi:
                continue
            if not float(v) >= threshold:
                continue
            if peak and not (1 <= b <= w - 2 and v > row[b - 1] and v > row[b + 1]):
                continue
            vals.append(hz[b])
        out.append(np.array(vals, np.float64))
    return out


def _check(gram, threshold, peak=True, fmin=None, fmax=None, kind="contour"):
    hz = evaluate.salience_bins(kind)[0]
    lo, hi = evaluate.salience_bin_range(kind, fmin, fmax)
    t, got = evaluate.salience_to_multipitch(gram, threshold, peak, fmin, fmax, kind)
    exp = _per_cell(gram, threshold, peak, lo, hi, hz)
    assert len(got) == len(exp) == len(t)
    for a, b in zip(got, exp):
        np.testing.assert_array_equal(a, b)
        assert a.dtype == np.float64
    return got


@pytest.mark.parametrize("kind,table", [("contour", "FREQ_BINS_CONTOURS"), ("note", "FREQ_BINS_NOTES")])
def test_salience_bins_are_the_target_grids_bit_for_bit(kind, table):
    hz, midi, chroma = evaluate.salience_bins(kind)
    ref = getattr(constants, table)
    m, c = evaluate.multipitch_values(ref)
    assert hz.tobytes() == np.asarray(ref, np.float64).tobytes()
    assert midi.tobytes() == m.tobytes() and chroma.tobytes() == c.tobytes()
    assert (np.diff(midi) >= 0).all() and ((chroma >= 0) & (chroma < 12)).all()
    assert len(hz) == {"contour": 264, "note": 88}[kind]
    with pytest.raises(ValueError):
        evaluate.salience_bins("onset")


def _hand_made(width):
    g = np.zeros((9, width), np.float32)
    g[0, 10:12] = 0.8  # plateau of two: neither is a peak
    g[0, 20:24] = [0.5, 0.9, 0.9, 0.5]
    g[0, 30:33] = [0.2, 0.6, 0.2]  # a peak
    g[1, 0], g[1, 1] = 0.9, 0.1  # peaks on the first and last bins: never peaks
    g[1, -1], g[1, -2] = 0.9, 0.1
    g[2, 5:8] = [0.2, np.nan, 0.2]  # a NaN cell, and NaN neighbours of a high cell
    g[2, 40:43] = [np.nan, 0.7, 0.1]
    g[2, 50:53] = [0.1, 0.7, np.nan]
    g[3, 60:63] = [0.1, np.float32(0.3), 0.1]  # a peak exactly at the threshold 0.3 (as float32)
    g[4, 60:63] = [0.1, np.float32(0.3), 0.1]
    g[5, :] = 0.0  # an all-zero frame
    g[6, 1::2] = 0.4  # a comb: every odd bin a peak
    g[7, 2:5] = [0.5, 0.6, 0.5]  # a peak whose neighbours a frequency range may cut
    g[8, :] = np.nan
    return g


@pytest.mark.parametrize("kind", ["contour", "note"])
def test_salience_to_multipitch_equals_the_per_cell_rule_on_hand_made_posteriorgrams(kind):
    hz = evaluate.salience_bins(kind)[0]
    g = _hand_made(len(hz))
    c = float(np.float32(0.3))
    for peak in (True, False):
        for thr in (0.05, 0.1, 0.25, c, 0.5, 0.8, 0.9, 0.95):
            _check(g, thr, peak, kind=kind)
        # frequency ranges that cut the neighbours of the peak at bin 3 of frame 7 (the peak test reads the whole row)
        for fmin, fmax in ((hz[3], None), (None, hz[3]), (hz[3], hz[3]), (hz[2] * 1.001, hz[3] * 1.001), (hz[4], hz[2]),
                           (0.0, 1e9), (hz[10], hz[40]), (1e9, None)):
            _check(g, 0.1, peak, fmin, fmax, kind)
    # plateaus and edges are not peaks, the peak at the threshold is included, NaN is never an estimate
    got = evaluate.salience_to_multipitch(g, c, True, kind=kind)[1]
    assert hz[31] in got[0] and hz[10] not in got[0] and hz[11] not in got[0] and hz[21] not in got[0]
    assert len(got[1]) == 0 and len(got[2]) == 0 and len(got[5]) == 0 and len(got[8]) == 0
    assert got[3].tolist() == [hz[61]]
    assert evaluate.salience_to_multipitch(g, c, False, kind=kind)[1][8].size == 0
    # ranges: the peak at bin 3 stays a peak when its neighbours are outside the range
    assert evaluate.salience_to_multipitch(g, 0.1, True, hz[3], hz[3], kind)[1][7].tolist() == [hz[3]]
    assert evaluate.salience_to_multipitch(g, 0.1, True, hz[4], hz[2], kind)[1][7].size == 0  # empty range


def test_threshold_is_compared_in_float64():
    """A float64 threshold just above a float32 cell, which rounds back to that cell in float32, excludes the cell."""
    hz = evaluate.salience_bins("contour")[0]
    g = _hand_made(264)
    cell = np.float32(0.3)
    thr = float(np.nextafter(np.float64(cell), 1.0))
    assert np.float32(thr) == cell and float(cell) < thr
    got = _check(g, thr, True)
    assert got[3].size == 0 and hz[31] in got[0]
    assert _check(g, float(cell), True)[3].tolist() == [hz[61]]
    assert _check(g, float(cell), False)[4].tolist() == [hz[61]]


def test_random_posteriorgrams_with_ties_equal_the_per_cell_rule():
    rng = np.random.default_rng(3)
    for kind, width in (("contour", 264), ("note", 88)):
        hz = evaluate.salience_bins(kind)[0]
        g = rng.choice(np.array([0.0, 0.1, 0.25, 0.5, 0.5, 0.75, 1.0, np.nan], np.float32), size=(40, width))
        g[::7] = rng.random((len(g[::7]), width)).astype(np.float32)
        for thr in (0.1, 0.25, 0.5, 0.6, 1.0):
            for peak in (True, False):
                for fmin, fmax in ((None, None), (hz[width // 4], hz[width // 2]), (hz[1] * 0.999, hz[-2] * 1.0001)):
                    _check(g, thr, peak, fmin, fmax, kind)


def test_salience_to_multipitch_times_shapes_and_errors():
    from basic_pitch_b200.note_creation import model_frames_to_time

    g = np.zeros((5, 264), np.float32)
    t, f = evaluate.salience_to_multipitch(g, 0.5)
    assert t.tobytes() == model_frames_to_time(5).tobytes() and len(f) == 5
    t, f = evaluate.salience_to_multipitch(np.zeros((0, 88), np.float32), 0.5, kind="note")
    assert len(t) == 0 and f == []
    for bad in (0.0, -0.1, np.nan, np.inf):
        with pytest.raises(ValueError, match="threshold"):
            evaluate.salience_to_multipitch(g, bad)
    with pytest.raises(ValueError):
        evaluate.salience_to_multipitch(np.zeros((5, 88), np.float32), 0.5)  # a note posteriorgram as a contour
    with pytest.raises(ValueError):
        evaluate.salience_to_multipitch(g, 0.5, kind="onset")


def test_settings_become_bins_by_searchsorted():
    from basic_pitch_b200.inference import Model

    hz = evaluate.salience_bins("contour")[0]
    assert evaluate.salience_bin_range("contour", None, None) == (0, 264)
    assert evaluate.salience_bin_range("contour", hz[10], hz[20]) == (10, 21)
    assert evaluate.salience_bin_range("contour", np.nextafter(hz[10], np.inf), np.nextafter(hz[20], 0)) == (11, 20)
    assert evaluate.salience_bin_range("contour", 1e9, 0.0) == (264, 264)
    assert evaluate.salience_bin_range("note", hz[40], hz[5]) == (evaluate.salience_bin_range("note", hz[40], None)[0],) * 2
    ps = Model._salience_params([dict(threshold=0.3), dict(threshold=0.5, peak_picking=False, minimum_frequency=hz[10],
                                                           maximum_frequency=hz[20])], "contour")
    assert [(p.threshold, p.peak_pick, p.bin_lo, p.bin_hi) for p in ps] == [(0.3, 1, 0, 264), (0.5, 0, 10, 21)]
    with pytest.raises(TypeError, match="unknown"):
        Model._salience_params([dict(threshold=0.3, onset_thresh=0.5)], "contour")
    with pytest.raises(TypeError, match="threshold"):
        Model._salience_params([dict(peak_picking=True)], "contour")


def test_chunk_params_follow_their_formula():
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    for K, V in ((0, 0), (1, 0), (0, 1), (100, 400), (10**6, 3 * 10**6), (2 * 10**6, 16 * 10**6), (10**8, 10**9),
                 (-5, -7)):
        per = 16 * max(V, 0) + 8 * max(K, 0)
        assert lib.bp_score_salience_chunk_params(K, V) == max(1, 2**31 // max(1, per)), (K, V)
    assert lib.bp_score_salience_chunk_params(2 * 10**6, 16 * 10**6) == 7
