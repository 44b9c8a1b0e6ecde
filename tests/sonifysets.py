"""Adversarial note sets for the MIDI sonification (CPU only: plain NumPy, deterministic, seeded).

The decoded clips and the hand-made files of tests/test_gpu_sonify.py switch bends at most once per 256-sample tile and
never put a note or a switch on a tile edge on purpose, so most of the host planning of csrc/sonify.cu (the sample
positions, the collapse of bend events onto one switch sample, the per-tile CSR of notes and each entry's starting
segment) and the kernel's segment walk go unobserved.  `sets(fs)` returns, for one sample rate, a list of `SonSet`s: a
name and the event lists of a batch of files (`(start_s, end_s, pitch, np.float32 amplitude, bends or None)` per note),
meant for both values of multiple_pitch_bends.

Every position is built from a target sample index k, so that each edge is hit exactly: `t_at(k, fs)` is the smallest
time t with int(fs * t) == k (fs * t at or just above k) and `t_below(k, fs)` its predecessor (fs * t just below k, so
int gives k - 1 and round would give k).  Bend events are placed through zero-length "carrier" notes of the target's
pitch, whose one bend sits at their start: with multiple_pitch_bends they share the target's instrument and switch it
at the first sample whose time k / fs is >= the carrier's time; without it a carrier inside a note overlaps it, and both
lose their bends (drop_overlapping_pitch_bends), which is a case of its own.

  tile_edges   note spans with a and b in {256 j - 1, 256 j, 256 j + 1}, through both t_at and t_below, a note inside
               one tile, one exactly a tile long and one ending on a tile's last sample
  bends        switches at 256 j and 256 j +- 1, at a, b - 1 and b (no effect) and before a (active at a); events that
               collapse onto one sample (distinct times, equal times from different notes, one note's equal times);
               bend times k / fs and their nextafter neighbours; a single-bend note; ticks clipped at +-8192
  dense        more than 8 switches in one tile, by carriers and by a note's own bends (kept without
               multiple_pitch_bends too)
  fades        note lengths 1, 2, 3, 2 fade_max - 1, 2 fade_max and 2 fade_max + 1 samples
  crowd        320 notes covering one tile (a long CSR row), pitches out of order
  same_pitch   overlapping notes of one pitch; touching notes whose bends carry; equal bend times from two notes
  velocity_*   a reference note of amplitude 1.0 with: amplitudes 0, negative and above 1; for every k in 0..127 the
               float32 amplitude whose float32 product with 127 is k + 0.5; float32 amplitudes whose velocity differs
               when the product is taken in float64; 2e7, -3e9 and 1e30
  pitch        pitches 0, 127, -5 and 200
  peak         a file whose peak is a negative sample, and one whose peak is in a long note's last tile
  layout       empty files and files of zero-length notes only between others, n_samples = 0, 1 and 255 (mod 256)
  many         1 000 files in one call, most of them empty

Low rates have no fades (int(0.01 fs) = 0 below 100 Hz) and put every position a whole second or more apart.  The
float64 restatement of the renderer, the liveness counts and the mutants are in tests/test_sonify_edges_cpu.py; the
device comparison is tests/test_gpu_sonify_edges.py.
"""
from __future__ import annotations

import functools
from typing import List, NamedTuple

import numpy as np

RATES = (1, 50, 8000, 7919, 11025, 16000, 22050, 44100, 48000, 96000, 192000)
TILE = 256
f32 = np.float32


class SonSet(NamedTuple):
    name: str
    files: List[list]  # per file: [(start_s, end_s, pitch, np.float32 amplitude, bends or None)]


def fade_max(fs: int) -> int:
    return int(0.01 * fs)


def t_at(k: int, fs: int) -> float:
    """The smallest float t >= 0 with int(fs * t) == k."""
    if k <= 0:
        return 0.0
    t = k / fs
    while int(fs * t) < k:
        t = float(np.nextafter(t, np.inf))
    while int(fs * float(np.nextafter(t, -np.inf))) >= k:
        t = float(np.nextafter(t, -np.inf))
    return t


def t_below(k: int, fs: int) -> float:
    """The largest float t with int(fs * t) == k - 1: fs * t lies just below k."""
    return float(np.nextafter(t_at(k, fs), -np.inf))


def end_for(n_samples: int, fs: int) -> float:
    """An end time e with int(fs * (e + 1)) == n_samples (the stand-in's output length for a file ending at e)."""
    e = n_samples / fs - 1.0
    while int(fs * (e + 1.0)) < n_samples:
        e = float(np.nextafter(e, np.inf))
    while int(fs * (e + 1.0)) > n_samples:
        e = float(np.nextafter(e, -np.inf))
    assert e >= 0.0 and int(fs * (e + 1.0)) == n_samples, (n_samples, fs)
    return e


@functools.lru_cache(maxsize=None)
def tie_amplitudes() -> np.ndarray:
    """[128] float32: for every k the amplitude closest to (k + 0.5) / 127 whose float32 product with 127 is exactly
    k + 0.5, a tie that np.round breaks to the even neighbour."""
    out = np.zeros(128, np.float32)
    for k in range(128):
        want = f32(k + 0.5)
        lo = hi = f32((k + 0.5) / 127.0)
        for _ in range(64):  # outwards from the nearest float32, both ways
            hit = [c for c in (lo, hi) if f32(127) * c == want]
            if hit:
                out[k] = hit[0]
                break
            lo, hi = np.nextafter(lo, f32(-1)), np.nextafter(hi, f32(2))
        else:
            raise AssertionError(f"no float32 tie amplitude for k = {k}")
    return out


@functools.lru_cache(maxsize=None)
def f64_disagreements(n: int = 8) -> np.ndarray:
    """float32 amplitudes in [0, 1) (seeded random search) whose velocity np.round(f32(127) * amp) differs from the
    velocity of the float64 product 127.0 * float(amp)."""
    rng = np.random.default_rng(2024)
    amps = rng.random(4_000_000, dtype=np.float32)
    v32 = np.round(f32(127) * amps).astype(np.float64)
    v64 = np.round(127.0 * amps.astype(np.float64))
    hit = amps[v32 != v64]
    assert hit.size >= n, hit.size
    return hit[:n]


def _carrier(t: float, pitch: int, tick_bends) -> tuple:
    """A zero-length note at time t: it never sounds, and its bends all sit at t."""
    return (t, t, pitch, f32(0.25), list(tick_bends))


def _note(a: int, b: int, fs: int, pitch: int, amp: float, bends=None) -> tuple:
    return (t_at(a, fs), t_at(b, fs), pitch, f32(amp), bends)


def _ref(fs: int, a: int = 300, b: int = 900) -> tuple:
    """The reference note of a velocity file: amplitude 1.0, velocity 127."""
    return _note(a, b, fs, 69, 1.0)


def tile_edges(fs: int) -> List[SonSet]:
    E = [TILE * j + d for j in (1, 2, 3) for d in (-1, 0, 1)]
    pairs = [(a, b) for a in E for b in E if b > a]
    files = []
    for side in range(2):
        notes = []
        for i, (a, b) in enumerate(pairs):
            ts = t_at(a, fs) if side == 0 else t_below(a + 1, fs)
            te = t_at(b, fs) if (side + i) % 2 == 0 else t_below(b + 1, fs)
            notes.append((ts, te, 40 + (i * 7) % 48, f32(0.2 + 0.06 * ((i * 5) % 11)), None))
        files.append(notes)
    files.append([_note(300, 400, fs, 62, 0.5),  # inside one tile
                  _note(512, 768, fs, 65, 0.6),  # exactly one tile
                  _note(600, 768, fs, 67, 0.7),  # ends on a tile's last sample
                  _note(1024, 1100, fs, 71, 0.4, [2, -3]),  # starts on a tile's first sample
                  (t_below(1281, fs), t_below(1536, fs), 72, f32(0.8), None)])  # 1280 .. 1534 through t_below
    return [SonSet("tile_edges", files)]


TICKS = (-6, 6, 7, -7, 3, -2, 5, 1, -4, 2)  # bends of 1/3 semitone: +-6 and +-7 clip at -8192 / 8191


def bends(fs: int) -> List[SonSet]:
    P, a, b = 60, 300, 1100
    files = []
    # switches on tile edges, at a, at b - 1, at b and before a; times k / fs, nextafter(k / fs, +-inf), (k - 1/2) / fs
    switch = [200, a, 511, 512, 513, 767, 768, 769, 1023, 1024, 1025, b - 1, b]
    notes = [_note(a, b, fs, P, 0.7)]
    for i, k in enumerate(switch):
        exact = k / fs
        t = (exact, float(np.nextafter(exact, -np.inf)), (k - 0.5) / fs)[i % 3]
        notes.append(_carrier(t, P, [TICKS[i % len(TICKS)]]))
    notes.append(_carrier(float(np.nextafter(900 / fs, np.inf)), P, [4]))  # just after 900 / fs: switches at 901
    files.append(notes)
    # events collapsing onto one switch sample: distinct times, equal times from two notes, one note's equal times
    k = 640
    notes = [_note(a, b, fs, P, 0.6)]
    notes += [_carrier((k - 0.9) / fs, P, [3]), _carrier((k - 0.5) / fs, P, [-5]), _carrier(k / fs, P, [6])]
    notes += [_carrier(800 / fs, P, [2]), _carrier(800 / fs, P, [-2]), _carrier(800 / fs, P, [1])]
    notes += [_carrier(t_at(950, fs), P, [5, -1, 3])]
    notes += [_carrier(a / fs, P, [2]), _carrier(a / fs, P, [-3])]  # collapse at a: the last is active from a
    files.append(notes)
    # a single-bend note (its bend is at its start), alone, and a note whose bends are all before a
    files.append([_note(200, 700, fs, 64, 0.5, [5]), _note(800, 1000, fs, 66, 0.5)])
    files.append([_carrier(100 / fs, P, [4, -6]), _carrier(t_at(150, fs), P, [7]), _note(a, 700, fs, P, 0.5)])
    return [SonSet("bends", files)]


def dense(fs: int) -> List[SonSet]:
    P = 57
    carriers = [520, 524, 530, 533, 540, 551, 560, 571, 590, 600, 601, 602, 700, 766]  # 14 switches in tile 2
    notes = [_note(100, 1000, fs, P, 0.8)]
    notes += [_carrier(k / fs if i % 2 else t_below(k, fs), P, [TICKS[i % len(TICKS)]]) for i, k in enumerate(carriers)]
    rng = np.random.default_rng(fs)
    own = [_note(100, 700, fs, 52, 0.6, rng.integers(-7, 8, 120).tolist())]  # a switch every 5 samples
    return [SonSet("dense", [notes, own])]


def fades(fs: int) -> List[SonSet]:
    fm = fade_max(fs)
    lengths = sorted({n for n in (1, 2, 3, 2 * fm - 1, 2 * fm, 2 * fm + 1) if n >= 1})
    notes, pos = [], 300
    for i, n in enumerate(lengths):
        notes.append(_note(pos, pos + n, fs, 60 + 3 * i, 0.5 + 0.1 * i, [1, -2] if i % 2 else None))
        pos += n + 37
    return [SonSet("fades", [notes])]


def crowd(fs: int) -> List[SonSet]:
    notes = []
    for i in range(320):
        a, b = 300 + (i * 13) % 212, 768 + (i * 29) % 300  # all cover tile 2 (512 .. 767)
        bends_i = [(i % 5) - 2, (i % 3) - 1] if i % 7 == 0 else None
        notes.append(_note(a, b, fs, 21 + (i * 37) % 88, 0.1 + 0.8 * ((i * 11) % 17) / 16, bends_i))
    return [SonSet("crowd", [notes])]


def same_pitch(fs: int) -> List[SonSet]:
    overlap = [_note(300, 800, fs, 60, 0.6, [1, 2, 3, 4]), _note(500, 1000, fs, 60, 0.5, [-3, -1]),
               _note(700, 900, fs, 60, 0.4), _note(600, 650, fs, 64, 0.3, [2])]
    # touching notes: each starts where the last ended, so their bends survive drop_overlapping_pitch_bends; the last
    # bend of one (at its end) and the first of the next (at its start) are equal times from two notes
    touching = [_note(200, 400, fs, 55, 0.6, [1, 2, 3]), _note(400, 650, fs, 57, 0.5, [-2, 4]),
                _note(650, 900, fs, 55, 0.7, [3, -1, 5]), _note(900, 1000, fs, 55, 0.4)]
    return [SonSet("same_pitch", [overlap, touching])]


def velocity(fs: int) -> List[SonSet]:
    def around(amps, pitch0=40):
        return [_ref(fs)] + [(t_at(1000 + 120 * i, fs), t_at(1100 + 120 * i, fs), pitch0 + i % 40, f32(x), None)
                             for i, x in enumerate(amps)]

    return [SonSet("velocity_sign", [around([0.0, -0.5, 1.7, -1e-3, 2.0])]),
            SonSet("velocity_ties", [around(tie_amplitudes())]),
            SonSet("velocity_f64", [around(f64_disagreements())]),
            SonSet("velocity_big", [around([2e7]), around([-3e9]), around([1e30])])]


def pitch(fs: int) -> List[SonSet]:
    return [SonSet("pitch", [[_ref(fs), _note(950, 1200, fs, 0, 0.5, [3]), _note(1300, 1500, fs, 127, 0.6, [-2, 7]),
                              _note(1600, 1800, fs, -5, 0.7), _note(1900, 2100, fs, 200, 0.8, [1])]])]


def peak(fs: int) -> List[SonSet]:
    # a note of 3 samples: its loudest sample (the middle one when there is a fade) decides the sign of the peak
    fm = fade_max(fs)
    for p in range(0, 256):  # above 127 at high rates: the stand-in does not clamp pitches
        f = 440.0 * 2.0 ** ((p - 69.0) / 12.0)
        y = np.sin(2.0 * np.pi * f * np.arange(1, 4) / fs) * (np.array([0.0, 1.0, 0.0]) if fm else 1.0)
        if y[np.argmax(np.abs(y))] < -0.1:
            break
    else:
        raise AssertionError(f"no pitch gives a negative peak at {fs} Hz")
    negative = [_note(500, 503, fs, p, 0.9)]
    last_tile = [_note(100, 1000, fs, 48, 0.2), _note(900, 1000, fs, 50, 1.0)]
    return [SonSet("peak", [negative, last_tile])]


def layout(fs: int) -> List[SonSet]:
    files = []
    base = TILE * (fs // TILE + 2)  # n_samples >= fs: every file lasts its end time + 1 s
    for r in (0, 1, 255):
        n = base + r
        e = end_for(n, fs)
        files.append([_note(200, 400, fs, 60 + r % 12, 0.5, [1, -1]), (t_at(500, fs), e, 62, f32(0.6), None)])
        files.append([])
        files.append([(t_at(300, fs), t_at(300, fs), 64, f32(0.5), [2])])  # b == a only: zeros
        files.append([(t_at(300, fs), t_below(301, fs), 65, f32(0.5), None),
                      (t_at(700, fs), t_at(650, fs), 66, f32(0.5), None)])  # b == a and b < a: zeros
    return [SonSet("layout", files)]


def many(fs: int) -> List[SonSet]:
    files = []
    for i in range(1000):
        if i % 25:
            files.append([])
        else:
            bend = [i % 5 - 2] if i % 2 else None
            files.append([_note(100 + i % 256, 400 + (i * 7) % 300, fs, 40 + i % 50, 0.5, bend)])
    return [SonSet("many", files)]


BUILDERS = (tile_edges, bends, dense, fades, crowd, same_pitch, velocity, pitch, peak, layout, many)


@functools.lru_cache(maxsize=None)
def sets(fs: int) -> List[SonSet]:
    return [s for build in BUILDERS for s in build(fs)]
