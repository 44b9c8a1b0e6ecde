"""CPU: the bent-note estimates of basic_pitch_b200/evaluate.py (BENT_HZ, bent_bins, note_frames_to_multipitch,
note_frames_to_melody), the host definitions of bp_score_bent_frames_grid_* and bp_score_note_melody_grid_*, against
brute force; and the property that lets the device work from the count roll: a pitch's bend depends on (file, pitch,
frame) only, checked on every overlapping note-frame of the reference's decodes in tests/golden/decode_edges.npz."""
import numpy as np

from basic_pitch_b200 import evaluate as ev
from basic_pitch_b200.note_creation import model_frames_to_time
from tests import postsets
from tests.golden_util import edges_case

_EST_HZ = 440.0 * 2.0 ** ((np.arange(128, dtype=np.float64) - 69.0) / 12.0)  # the Hz behind EST_LOG2_HZ / EST_MIDI


def test_bent_tables():
    c = np.arange(88)
    hz, midi, chroma, cents = ev.bent_bins()
    assert hz.shape == midi.shape == chroma.shape == cents.shape == (264,)
    assert hz[3 * c].tobytes() == _EST_HZ[21 + c].tobytes()
    assert np.array_equal(np.log2(hz[3 * c]), ev.EST_LOG2_HZ[21 + c])
    assert midi[3 * c].tobytes() == ev.EST_MIDI[21 + c].tobytes()
    assert chroma[3 * c].tobytes() == ev.EST_CHROMA[21 + c].tobytes()
    for a in (hz, midi, cents):
        assert (np.diff(a) > 0).all()
    assert (cents > 0).all() and ((chroma >= 0) & (chroma < 12)).all()
    assert cents.tobytes() == ev.melody_values(hz)[0].tobytes()


def _random_notes(rng, T, n, lo=21, hi=109, bends=True):
    start = rng.integers(0, max(T, 1), n)
    end = np.minimum(start + rng.integers(1, 40, n), T)
    keep = end > start
    start, end = start[keep], end[keep]
    pitch = rng.integers(lo, hi, len(start))
    # same-pitch overlaps: copy some notes onto others' spans
    dup = rng.random(len(start)) < 0.2
    if dup.any() and len(start) > 1:
        src = rng.integers(0, len(start), dup.sum())
        pitch[dup] = pitch[src]
    bl = []
    for j in range(len(start)):
        if not bends:  # a setting without bends: None or empty for every note
            bl.append(None if rng.random() < 0.5 else [])
            continue
        c = 3 * (pitch[j] - 21)
        b = rng.integers(max(-25, -c), min(25, 263 - c) + 1, end[j] - start[j])
        bl.append(b)
    return start, end, pitch, bl


def _consistent(start, end, pitch, bl):
    """Bends that depend on (pitch, frame) only, as the decode's do: the first note's bend at a frame wins for all."""
    seen = {}
    out = []
    for j in range(len(start)):
        if bl[j] is None or len(bl[j]) == 0:
            out.append(bl[j])
            continue
        b = np.array(bl[j])
        for t in range(start[j], end[j]):
            b[t - start[j]] = seen.setdefault((pitch[j], t), b[t - start[j]])
        out.append(b)
    return out


def _brute_keys(start, end, pitch, bl, T):
    frames = [[] for _ in range(T)]  # (pitch, key) of every sounding note
    for j in range(len(start)):
        for t in range(start[j], end[j]):
            b = 0 if bl[j] is None or len(bl[j]) == 0 else int(bl[j][t - start[j]])
            frames[t].append((int(pitch[j]), 3 * (int(pitch[j]) - 21) + b))
    return frames


def test_multipitch_without_bends_is_the_piano_roll():
    rng = np.random.default_rng(1)
    for T in (0, 1, 7, 300):
        start, end, pitch, _ = _random_notes(rng, T, 60, bends=False)
        t, got = ev.note_frames_to_multipitch(start, end, pitch, None, T)
        times = model_frames_to_time(T + 1)
        assert t.tobytes() == times[:T].tobytes()
        exp = ev.notes_to_multipitch(np.stack([times[start], times[end]], 1), _EST_HZ[pitch], times[:T])
        assert len(got) == len(exp) == T
        for a, b in zip(got, exp):
            assert np.sort(b).tobytes() == a.tobytes()
        _, got0 = ev.note_frames_to_multipitch(start, end, pitch, [[]] * len(start), T)
        assert all(a.tobytes() == b.tobytes() for a, b in zip(got, got0))


def test_host_definitions_match_brute_force():
    rng = np.random.default_rng(2)
    n_keys_edge = set()
    for case in range(60):
        T = int(rng.choice([0, 1, 5, 64, 250]))
        lo, hi = [(21, 109), (21, 25), (104, 109), (60, 62)][case % 4]
        start, end, pitch, bl = _random_notes(rng, T, int(rng.integers(0, 80)), lo, hi, bends=case % 5 != 4)
        bl = _consistent(start, end, pitch, bl)
        # note posteriorgram on a coarse grid (ties) with NaN cells and whole NaN rows
        gram = (rng.integers(0, 4, (T, 88)) / 4).astype(np.float32)
        gram[rng.random((T, 88)) < 0.15] = np.nan
        if T:
            gram[rng.integers(0, T)] = np.nan
        t_mp, mp = ev.note_frames_to_multipitch(start, end, pitch, bl, T)
        t_mel, f0 = ev.note_frames_to_melody(start, end, pitch, bl, gram)
        assert t_mp.tobytes() == t_mel.tobytes() == model_frames_to_time(T).tobytes()
        frames = _brute_keys(start, end, pitch, bl, T)
        for t, fr in enumerate(frames):
            keys = sorted(k for _, k in fr)
            n_keys_edge |= {k for k in keys if k in (0, 263)}
            assert mp[t].tobytes() == ev.BENT_HZ[np.array(keys, np.int64)].tobytes(), (case, t)
            if not fr:
                assert f0[t] == 0.0
                continue
            best = None
            for p, k in sorted(set(fr)):
                v = gram[t, p - 21]
                if best is None or v > best[0] or (np.isnan(best[0]) and not np.isnan(v)):
                    best = (v, p, k)
            assert f0[t] == ev.BENT_HZ[best[2]], (case, t, best)
    assert n_keys_edge == {0, 263}


def test_melody_ties_and_nan_cells():
    gram = np.zeros((4, 88), np.float32)
    gram[0, [39, 43]] = 0.5            # tie: the lower pitch (60) wins
    gram[1, 39], gram[1, 43] = np.nan, 0.1  # NaN loses to a number
    gram[2, [39, 43]] = np.nan         # all NaN: the lowest sounding pitch
    gram[3, 39], gram[3, 43] = -np.inf, np.nan  # -inf is a number
    start, end, pitch = np.array([0, 0]), np.array([4, 4]), np.array([60, 64])
    bl = [np.array([1, 2, -3, 0]), None]
    _, f0 = ev.note_frames_to_melody(start, end, pitch, bl, gram)
    k60, k64 = 3 * 39, 3 * 43
    assert f0.tolist() == [ev.BENT_HZ[k60 + 1], ev.BENT_HZ[k64], ev.BENT_HZ[k60 - 3], ev.BENT_HZ[k60]]
    _, f0 = ev.note_frames_to_melody([], [], [], None, np.zeros((3, 88), np.float32))
    assert f0.tolist() == [0.0, 0.0, 0.0]
    t, mp = ev.note_frames_to_multipitch([], [], [], None, 0)
    assert len(t) == 0 and mp == []


def test_bend_depends_on_pitch_and_frame_only(golden_dir):
    z = np.load(golden_dir / "decode_edges.npz")
    shared = 0
    for name in postsets.NAMES:
        n_files = len(z[f"{name}/sha"])
        j = 0
        while f"{name}/p{j}/start" in z.files:
            c = edges_case(z, f"{name}/p{j}")
            j += 1
            if len(c["bends"]) == 0:
                continue
            for i in range(n_files):
                seen = {}
                for n in range(int(c["note_off"][i]), int(c["note_off"][i + 1])):
                    b = c["bends"][c["bend_off"][n] : c["bend_off"][n + 1]]
                    for t in range(int(c["start"][n]), int(c["end"][n])):
                        key = (int(c["pitch"][n]), t)
                        if key in seen:
                            shared += 1
                            assert seen[key] == b[t - c["start"][n]], (name, j - 1, i, key)
                        else:
                            seen[key] = b[t - c["start"][n]]
    assert shared > 1000, shared
