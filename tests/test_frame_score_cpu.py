"""CPU: the frame-level multi-pitch metric (include/bp_b200.h, bp_score_frames_grid_*): the oracle
(oracle/multipitch_ref.py) against brute force and hand-worked boundaries, the host-only time base bp_multipitch_map
against scipy's interp1d, and the Python helpers of basic_pitch_b200/evaluate.py."""
import functools
import itertools

import numpy as np
import pytest
import scipy.interpolate

from oracle import multipitch_ref as mr

W = 0.5


def _brute(hits) -> int:
    hits = np.asarray(hits, bool)
    n_ref, n_est = hits.shape

    @functools.lru_cache(maxsize=None)
    def best(i, used):
        if i == n_ref:
            return 0
        b = best(i + 1, used)
        for j in range(n_est):
            if hits[i, j] and not used >> j & 1:
                b = max(b, 1 + best(i + 1, used | 1 << j))
        return b

    return best(0, 0)


def _tp(rm, em, window=W):
    rm, em = np.asarray(rm, np.float64), np.asarray(em, np.float64)
    rc, ec = np.mod(np.mod(rm, 12), 12), np.mod(np.mod(em, 12), 12)
    if not len(rm) or not len(em):
        return 0, 0
    return mr.max_matching(mr.hit_matrix(rm, em, window, False)), mr.max_matching(mr.hit_matrix(rc, ec, window, True))


def test_oracle_matching_equals_brute_force_on_every_shape_up_to_7x7():
    rng = np.random.default_rng(5)
    for n_ref, n_est in itertools.product(range(8), range(8)):
        for _ in range(6):
            base = rng.uniform(30, 90)
            pool = base + np.array([-12, -0.5, 0, 0.25, 0.5, 0.75, 1, 11.5, 12, -11.75])
            rm, em = rng.choice(pool, n_ref), rng.choice(pool, n_est)  # repeats: multiplicities
            window = rng.choice([0.0, 0.25, 0.5, 1.0, 6.0])
            for chroma in (False, True):
                a, b = (np.mod(np.mod(rm, 12), 12), np.mod(np.mod(em, 12), 12)) if chroma else (rm, em)
                h = mr.hit_matrix(a, b, window, chroma)
                assert mr.max_matching(h) == _brute(h), (n_ref, n_est, chroma)


def test_hand_worked_boundaries():
    e = 60.3
    lo, hi = e - W, e + W
    assert _tp([lo], [e]) [0] == 1 and _tp([hi], [e])[0] == 1
    assert _tp([np.nextafter(lo, -np.inf)], [e])[0] == 0 and _tp([np.nextafter(hi, np.inf)], [e])[0] == 0
    # chroma wrap: 11.8 against 0.2 (midi 59.8 and 72.2): 12 - 11.6 = 0.4 <= 0.5
    assert _tp([59.8], [72.2]) == (0, 1)
    # a value just below 0 in midi: np.mod gives 12.0, the second np.mod 0.0 (from Hz, 69 + 12 log2(.) cannot get that
    # close to 0: its largest negative value is -2^-46, whose chroma stays just below 12)
    assert np.mod(-1e-17, 12) == 12.0 and np.mod(np.mod(-1e-17, 12), 12) == 0.0
    assert _tp([-1e-17], [11.9]) == (0, 1) and _tp([-1e-17], [0.6]) == (0, 0)
    from basic_pitch_b200.evaluate import multipitch_values

    hz = np.nextafter(np.nextafter(440.0 * 2 ** (-69 / 12), 0), 0)
    midi, chroma = multipitch_values([hz])
    assert midi[0] == -(2.0**-46) and chroma[0] == 12.0 - 2.0**-46 * 1.0 and chroma[0] < 12
    assert (midi[0], chroma[0]) == tuple(v[0] for v in mr.values([hz]))
    assert _tp(midi, [0.4]) == (1, 1) and _tp(midi, [0.6]) == (0, 0)
    # window 0: exact equality only; window >= 6: every chroma pair hits
    assert _tp([60.0, 61.0], [60.0, 61.0 + 1e-12], 0.0) == (1, 1)
    assert _tp([60.0, 61.0, 62.0], [66.0, 72.5], 6.0) == (1, 2)
    # duplicates and empty frames on either side
    assert _tp([60.0, 60.0, 60.0], [60.0, 60.0]) == (2, 2)
    assert _tp([], [60.0]) == (0, 0) and _tp([60.0], []) == (0, 0)
    t = np.array([0.0, 0.01, 0.02])
    c = mr.counts(t, [np.array([]), np.array([440.0, 440.0]), np.array([220.0])], t,
                  [np.array([440.0]), np.array([440.0]), np.array([])])
    assert c == [3, 2, 1, 1, 1, 2, 1]


# ------------------------------------------------------------------------------------------------ time base
def _map(est_t, ref_t):
    from basic_pitch_b200 import _lib

    est_t, ref_t = np.ascontiguousarray(est_t, np.float64), np.ascontiguousarray(ref_t, np.float64)
    out = np.full(len(ref_t), -7, np.int64)
    _lib.load().bp_multipitch_map(est_t.ctypes.data, len(est_t), ref_t.ctypes.data, len(ref_t), out.ctypes.data)
    return out


def _scipy_map(est_t, ref_t):
    n = len(est_t)
    if n == 0:
        return np.full(len(ref_t), -1)
    f = scipy.interpolate.interp1d(est_t, np.arange(n), kind="nearest", bounds_error=False, fill_value=n,
                                   assume_sorted=True)
    idx = f(np.asarray(ref_t, np.float64)).astype(np.int64)
    idx[idx == n] = -1
    return idx


def test_multipitch_map_equals_interp1d():
    from basic_pitch_b200.note_creation import model_frames_to_time

    est = model_frames_to_time(400)
    mids = est[:-1] / 2.0 + est[1:] / 2.0
    rng = np.random.default_rng(2)
    cases = [
        (est, mids),  # exactly at the midpoints
        (est, np.concatenate([[est[0] - 1e-9, -0.0, est[-1], np.nextafter(est[-1], np.inf), est[-1] + 1.0], est])),
        (est, np.arange(0, 5.0, 0.01)), (est, np.sort(rng.uniform(0, 5, 700))),
        (np.zeros(0), np.arange(0, 1, 0.1)), (np.array([0.5]), np.array([0.4, 0.5, 0.6])),
        (np.array([0.5, 0.7]), np.array([0.49, 0.5, 0.6, 0.6000000000000001, 0.7, 0.71])),
        (np.array([0.0, 0.2, 0.2, 0.2, 0.5]), np.arange(0, 0.6, 0.05)),  # duplicate est times
        (est, np.zeros(0)),
    ]
    for et, rt in cases:
        exp = _scipy_map(et, rt) if not (len(et) == len(rt) and len(et) and np.allclose(et, rt)) else np.arange(len(et))
        np.testing.assert_array_equal(_map(et, rt), exp)
        np.testing.assert_array_equal(mr.resample_index(et, rt), exp)
    # the allclose path: ref = est (1 + 1e-7) must not resample (although interp1d would move some frames) ...
    ref = est * (1 + 1e-7)
    np.testing.assert_array_equal(_map(est, ref), np.arange(len(est)))
    # ... while an equal size with a 1e-3 offset must
    ref = est + 1e-3
    got = _map(est, ref)
    np.testing.assert_array_equal(got, _scipy_map(est, ref))
    assert got[-1] == -1


def test_multipitch_map_rejects_bad_times():
    from basic_pitch_b200 import _lib

    with pytest.raises(_lib.BpError, match="estimate frame 2"):
        _map([0.0, 0.1, 0.05], [0.0])
    with pytest.raises(_lib.BpError, match="reference frame 1"):
        _map([0.0, 0.1], [0.0, np.nan])


# ------------------------------------------------------------------------------------------------ evaluate.py
def _random_series(rng, n, hop, p_empty=0.2):
    t = np.round(np.arange(n) * hop + (rng.uniform(0, hop / 3, n) if hop > 0.0105 else 0), 6)
    freqs = []
    for _ in range(n):
        k = 0 if rng.random() < p_empty else rng.integers(1, 5)
        freqs.append(440.0 * 2 ** ((rng.integers(-20, 20, k) + rng.choice([0, 0.3, -0.45, 12.0], k)) / 12.0))
    return t, freqs


def test_frame_scores_bit_identical_to_the_oracle_metrics():
    from basic_pitch_b200.evaluate import frame_scores

    rng = np.random.default_rng(8)
    e_t, e_f = _random_series(rng, 50, 0.0116)
    r_t, r_f = _random_series(rng, 60, 0.01)
    empty_t, empty_f = np.zeros(0), []
    silent_t, silent_f = r_t, [np.zeros(0)] * len(r_t)
    pairs = [(r_t, r_f, e_t, e_f), (r_t, r_f, empty_t, empty_f), (empty_t, empty_f, e_t, e_f),
             (silent_t, silent_f, e_t, e_f), (r_t, r_f, silent_t, silent_f), (silent_t, silent_f, silent_t, silent_f),
             (r_t, r_f, r_t, r_f)]
    for rt, rf, et, ef in pairs:
        c = mr.counts(rt, rf, et, ef)
        got = frame_scores(np.array(c))
        exp = mr.metrics(rt, rf, et, ef)
        for k, v in exp.items():
            assert got[k].tobytes() == np.float64(v).tobytes(), (k, got[k], v)
    assert frame_scores(np.zeros((2, 0, 7), np.int64))["mean"]["precision"].shape == (2,)


def test_notes_to_multipitch_is_the_piano_roll_of_decoded_notes(golden_dir):
    from basic_pitch_b200 import _lib
    from basic_pitch_b200.evaluate import notes_to_multipitch
    from basic_pitch_b200.note_creation import midi_to_hz

    z = np.load(golden_dir / "vocadito10.npz")
    T = z["gold_note"].shape[0]
    times = np.zeros(T + 1)
    _lib.load().bp_frame_times(T + 1, times.ctypes.data)
    for key in ("decode2", "decode3"):
        start, end, pitch = (np.asarray(z[f"{key}/{k}"], np.int64) for k in ("start", "end", "pitch"))
        roll = np.zeros((T, 128), np.int64)
        for a, b, p in zip(start, end, pitch):
            roll[a:b, p] += 1
        assert roll.max() >= 1
        series = notes_to_multipitch(np.stack([times[start], times[end]], 1), midi_to_hz(pitch.astype(np.float64)),
                                     times[:T])
        assert len(series) == T
        assert notes_to_multipitch(np.stack([times[start], times[end]], 1), midi_to_hz(pitch.astype(np.float64)), []) == []
        for t in range(T):
            exp = np.repeat(midi_to_hz(np.arange(128, dtype=np.float64)), roll[t])
            np.testing.assert_array_equal(np.sort(series[t]), np.sort(exp), err_msg=f"{key} frame {t}")
