"""CPU: the pieces of note-level scoring that need no GPU — the NumPy oracle of mir_eval's note matching
(oracle/transcription_ref.py) against brute force and hand-worked boundary cases, the frame-time table the library builds
(bp_frame_times), `evaluate.note_scores`, and the annotated synthetic clips (synth.*_events)."""
import hashlib
import itertools

import numpy as np
import pytest

from oracle import transcription_ref as tr


def _brute_max_matching(hits) -> int:
    """Largest number of disjoint (row, column) hits, by dynamic programming over the set of used columns."""
    n_r, n_c = hits.shape
    best = {0: 0}
    for i in range(n_r):
        nxt = dict(best)
        for used, m in best.items():
            for j in range(n_c):
                if hits[i, j] and not used >> j & 1:
                    k = used | 1 << j
                    nxt[k] = max(nxt.get(k, 0), m + 1)
        best = nxt
    return max(best.values())


def test_oracle_matching_equals_brute_force():
    rng = np.random.default_rng(5)
    n = 0
    for n_r, n_c in itertools.product(range(9), range(9)):
        for density in (0.1, 0.3, 0.6, 1.0):
            for _ in range(3):
                hits = rng.random((n_r, n_c)) < density
                assert tr.max_matching(hits) == _brute_max_matching(hits), hits
                n += 1
    assert n == 81 * 12


def _one(ref_on, ref_off, ref_l2, est_on, est_off, est_l2, **tol):
    a, b = tr.hit_matrices([[ref_on, ref_off]], [ref_l2], [[est_on, est_off]], [est_l2], **{**tr.TOLERANCES, **tol})
    return bool(a[0, 0]), bool(b[0, 0])


def test_onset_rounds_to_the_tolerance():
    # |1.0 - 1.05| = 0.050000000000000044 rounds to 0.05: a hit; 0.05004 rounds down to 0.05: a hit; 0.05006 does not
    assert abs(1.0 - 1.05) > 0.05
    assert _one(1.0, 2.0, 8.0, 1.05, 2.0, 8.0) == (True, True)
    assert _one(1.0, 2.0, 8.0, 1.05004, 2.0, 8.0) == (True, True)
    assert _one(1.0, 2.0, 8.0, 1.05006, 2.0, 8.0) == (False, False)


def test_onset_rounding_ties_go_to_even():
    found = {0: None, 1: None}
    for k in range(1, 2000):
        x = (k + 0.5) / 1e4
        if x * 1e4 == k + 0.5 and found[k % 2] is None:
            found[k % 2] = (k, x)
    assert None not in found.values(), found
    k, x = found[0]  # rint(k + 0.5) = k for even k: within a tolerance of k / 1e4
    assert _one(0.0, 5.0, 8.0, x, 5.0, 8.0, onset_tolerance=k / 1e4) == (True, True)
    k, x = found[1]  # odd k rounds up to k + 1
    assert _one(0.0, 5.0, 8.0, x, 5.0, 8.0, onset_tolerance=k / 1e4) == (False, False)
    assert _one(0.0, 5.0, 8.0, x, 5.0, 8.0, onset_tolerance=(k + 1) / 1e4) == (True, True)


def test_offset_tolerance_at_its_minimum_and_at_the_ratio():
    # reference of 0.1 s: 0.2 x 0.1 < 0.05, the minimum applies
    assert _one(0.0, 0.1, 8.0, 0.0, 0.15, 8.0) == (True, True)
    assert _one(0.0, 0.1, 8.0, 0.0, 0.1501, 8.0) == (True, False)
    # reference of 1 s: 0.2 s; |1.0 - 1.2| = 0.19999999999999996 rounds to 0.2
    assert _one(0.0, 1.0, 8.0, 0.0, 1.2, 8.0) == (True, True)
    assert _one(0.0, 1.0, 8.0, 0.0, 1.2001, 8.0) == (True, False)
    assert _one(0.0, 1.0, 8.0, 0.0, 0.8, 8.0) == (True, True)
    assert _one(0.0, 1.0, 8.0, 0.0, 1.2, 8.0, offset_ratio=0.0) == (True, False)


def fifty_cents(a: float = 0.0):
    """(a, b, b_next): log2 values with |1200 * (a - b)| == 50.0 exactly in float64 and |1200 * (a - b_next)| > 50."""
    b = a + 1.0 / 24.0
    for _ in range(256):
        d = abs(1200 * (a - b))
        if d == 50.0:
            break
        b = np.nextafter(b, np.inf) if d < 50.0 else np.nextafter(b, -np.inf)
    assert abs(1200 * (a - b)) == 50.0, a
    nb = b
    while abs(1200 * (a - nb)) == 50.0:
        nb = np.nextafter(nb, np.inf)
    return a, float(b), float(nb)


def test_pitch_distance_of_exactly_fifty_cents():
    a, b, nb = fifty_cents()
    assert _one(0.0, 1.0, a, 0.0, 1.0, b) == (True, True)
    assert _one(0.0, 1.0, a, 0.0, 1.0, nb) == (False, False)
    assert _one(0.0, 1.0, b, 0.0, 1.0, a) == (True, True)  # the distance is symmetric
    assert _one(0.0, 1.0, a, 0.0, 1.0, b, pitch_tolerance=np.nextafter(50.0, 0)) == (False, False)


def test_oracle_counts_of_empty_sides():
    iv = np.array([[0.0, 1.0]])
    assert tr.counts(iv, [440.0], np.zeros((0, 2)), []) == [1, 0, 0, 0]
    assert tr.counts(np.zeros((0, 2)), [], iv, [440.0]) == [0, 1, 0, 0]
    assert tr.counts(iv, [440.0], iv, [440.0]) == [1, 1, 1, 1]


def test_oracle_equals_mir_eval_when_available():
    transcription = pytest.importorskip("mir_eval.transcription")
    rng = np.random.default_rng(3)
    for _ in range(50):
        sets = []
        for n in rng.integers(1, 40, 2):
            on = np.round(rng.uniform(0, 5, n), 2)
            iv = np.stack([on, on + np.round(rng.uniform(0.05, 1.0, n), 2)], 1)
            sets.append((iv, 440.0 * 2.0 ** (rng.integers(-5, 6, n) / 12.0 + rng.choice([0, 0.04, 0.0417], n))))
        (ri, rp), (ei, ep) = sets
        got = tr.counts(ri, rp, ei, ep)
        m0 = transcription.match_notes(ri, rp, ei, ep, offset_ratio=None)
        m1 = transcription.match_notes(ri, rp, ei, ep)
        assert got == [len(rp), len(ep), len(m0), len(m1)]


def test_frame_times_equal_model_frames_to_time():
    import ctypes as C

    from basic_pitch_b200 import _lib
    from basic_pitch_b200.note_creation import model_frames_to_time

    lib = _lib.load()
    n = 1 << 20
    out = np.empty(n, np.float64)
    lib.bp_frame_times(n, out.ctypes.data)
    exp = model_frames_to_time(n)
    assert out.tobytes() == exp.tobytes(), np.flatnonzero(out != exp)[:10]
    with pytest.raises(_lib.BpError):
        lib.bp_frame_times(-1, out.ctypes.data)
    lib.bp_frame_times(0, C.c_void_p())


def _mir_eval_prf(m, n_ref, n_est):
    """precision_recall_f1_overlap's arithmetic (mir_eval 0.7, beta = 1) from a matched count."""
    if n_ref == 0 or n_est == 0:
        return 0.0, 0.0, 0.0
    p = float(m) / n_est
    r = float(m) / n_ref
    f = 0.0 if p == 0 and r == 0 else (1 + 1**2) * p * r / ((1**2) * p + r)
    return p, r, f


def test_note_scores_follow_the_mir_eval_formulas():
    from basic_pitch_b200.evaluate import note_scores

    rng = np.random.default_rng(11)
    c = np.zeros((3, 7, 4), np.int64)
    c[..., 0] = rng.integers(0, 30, (3, 7))
    c[..., 1] = rng.integers(0, 30, (3, 7))
    c[0, 0, :2] = (0, 0)
    c[0, 1, :2] = (0, 5)
    c[0, 2, :2] = (5, 0)
    m = np.minimum(c[..., 0], c[..., 1])
    c[..., 2] = (m * rng.random((3, 7))).astype(np.int64)
    c[..., 3] = (c[..., 2] * rng.random((3, 7))).astype(np.int64)
    c[1, 3, 2:] = 0
    s = note_scores(c)
    for k, i in itertools.product(range(3), range(7)):
        for suffix, col in (("", 3), ("_no_offset", 2)):
            p, r, f = _mir_eval_prf(int(c[k, i, col]), int(c[k, i, 0]), int(c[k, i, 1]))
            assert (s["precision" + suffix][k, i], s["recall" + suffix][k, i], s["f_measure" + suffix][k, i]) == (p, r, f)
    for key in ("precision", "recall", "f_measure", "f_measure_no_offset"):
        np.testing.assert_array_equal(s["mean"][key], s[key].mean(axis=1))
    one = note_scores(c[1])
    assert one["mean"]["f_measure"] == s["f_measure"][1].mean()
    assert note_scores(np.zeros((2, 0, 4), np.int64))["mean"]["precision"].tolist() == [0.0, 0.0]


# SHA-256 of random_notes_clip's float32 output, taken before the note draws moved into a helper the event function shares
RANDOM_NOTES_SHA = {
    (3.0, 0, 5.0): "cfbe631756445514c0aea2af5109df24cc99f687eb80f533a43a04cff4223f0a",
    (10.0, 7, 5.0): "8038c934db16d29f7067ba1c96f46a9a4d1239aa50f069523542b23f4615edac",
    (0.05, 3, 5.0): "28714958e1118b52cccfbf1c0b25e0daa5d9257ffae009ba685b40d41ec310d9",
    (7.3, 123, 12.0): "3e88306b9de590c8a17d51ffc175bbf3c71caf1c714e1b1cf2fe9f3dbe17c5af",
}


@pytest.mark.parametrize("key", sorted(RANDOM_NOTES_SHA))
def test_random_notes_clip_is_unchanged(key):
    from basic_pitch_b200 import synth

    x = synth.random_notes_clip(*key)
    assert hashlib.sha256(x.tobytes()).hexdigest() == RANDOM_NOTES_SHA[key]


def test_annotation_helpers_describe_the_rendered_notes():
    from basic_pitch_b200 import synth

    sr = synth.SR
    for seconds, seed, nps in RANDOM_NOTES_SHA:
        iv, hz = synth.random_notes_events(seconds, seed, nps)
        n = int(round(seconds * sr))
        assert iv.shape == (len(hz), 2) and (iv[:, 1] > iv[:, 0]).all() and (iv[:, 1] <= n / sr).all()
        midi = 69 + 12 * np.log2(hz / 440.0)
        np.testing.assert_allclose(midi, np.round(midi), atol=1e-9)
        assert ((midi > 35.5) & (midi < 89.5)).all()
        x = synth.random_notes_clip(seconds, seed, nps)
        for a, b in iv:  # every note's first sample sounds (the envelope starts at 0, so look one sample later)
            i = int(round(a * sr))
            assert abs(i - a * sr) < 1e-6
            if i + 1 < len(x):
                assert np.any(x[i : min(i + 64, len(x))] != 0)
    assert len(synth.random_notes_events(0.05, 3)[1]) == 1
    iv, hz = synth.dense_chords_events(1.2)
    assert iv.shape == (3 * 88, 2)
    np.testing.assert_array_equal(np.unique(iv[:, 0]), [0.0, 0.5, 1.0])
    assert iv[-1, 1] == int(round(1.2 * sr)) / sr
    np.testing.assert_array_equal(hz[:88], [440.0 * 2 ** ((m - 69) / 12) for m in range(21, 109)])
