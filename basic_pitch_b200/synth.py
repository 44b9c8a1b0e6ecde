"""Deterministic synthetic 22 050 Hz mono audio for tests and benchmarks (SURVEY.md §8(d) configs).

No datasets are reachable from the build/bench machines, so every workload is generated:
  tones_clip        config 1 — 2 s: three harmonic tones + noise at -40 dB
  random_notes_clip config 2/3/4 — random note events (MIDI 36..89), 5 partials, exponential decay
  dense_chords_clip config 5 — all 88 piano pitches re-struck every 0.5 s
"""
from __future__ import annotations

import numpy as np

SR = 22050


def _normalise(x: np.ndarray) -> np.ndarray:
    peak = float(np.max(np.abs(x))) if x.size else 0.0
    return (x / max(1.0, peak)).astype(np.float32)


def tones_clip(seconds: float = 2.0, seed: int = 0) -> np.ndarray:
    rng = np.random.default_rng(seed)
    n = int(round(seconds * SR))
    t = np.arange(n) / SR
    x = np.zeros(n)
    for midi in (57, 64, 72):
        f0 = 440.0 * 2 ** ((midi - 69) / 12)
        for h in range(1, 5):
            if f0 * h < SR / 2:
                x += (0.25 / h) * np.sin(2 * np.pi * f0 * h * t + rng.uniform(0, 2 * np.pi))
    x += 0.01 * rng.standard_normal(n)
    return _normalise(x)


def _random_notes(seconds: float, seed: int, notes_per_second: float):
    """The draws of `random_notes_clip`: (first sample, length in samples, MIDI pitch) per note, in drawing order."""
    rng = np.random.default_rng(seed)
    n_notes = max(1, int(round(notes_per_second * seconds)))
    starts = rng.uniform(0, max(seconds - 1.0, 0.1), n_notes)
    durs = rng.uniform(0.15, 1.5, n_notes)
    pitches = rng.integers(36, 90, n_notes)
    return [(int(s * SR), int(d * SR), int(p)) for s, d, p in zip(starts, durs, pitches)], durs


def _hz(midi: int) -> float:
    return 440.0 * 2 ** ((midi - 69) / 12)


def random_notes_clip(seconds: float, seed: int, notes_per_second: float = 5.0) -> np.ndarray:
    n = int(round(seconds * SR))
    x = np.zeros(n + SR * 2)
    notes, durs = _random_notes(seconds, seed, notes_per_second)
    for (i0, m, p), d in zip(notes, durs):
        f0 = _hz(p)
        tt = np.arange(m) / SR
        env = np.exp(-3.0 * tt / d) * np.minimum(1.0, tt / 0.01)
        sig = np.zeros(m)
        for h in range(1, 6):
            if f0 * h < SR / 2:
                sig += np.sin(2 * np.pi * f0 * h * tt) / h
        x[i0 : i0 + m] += 0.1 * env * sig
    return _normalise(x[:n])


def random_notes_events(seconds: float, seed: int, notes_per_second: float = 5.0):
    """The notes `random_notes_clip(seconds, seed, notes_per_second)` renders, as mir_eval takes them: (intervals
    (n, 2) in seconds, pitches (n,) in Hz), in drawing order.  A note sounds from its first rendered sample; its offset is
    clipped to the clip's length, and a note starting at or after the end of the clip is left out."""
    n = int(round(seconds * SR))
    notes, _ = _random_notes(seconds, seed, notes_per_second)
    kept = [(i0, min(i0 + m, n), p) for i0, m, p in notes if i0 < n and m > 0]
    intervals = np.array([(a / SR, b / SR) for a, b, _ in kept], np.float64).reshape(-1, 2)
    return intervals, np.array([_hz(p) for _, _, p in kept], np.float64)


def dense_chords_events(seconds: float = 10.0):
    """The notes of `dense_chords_clip(seconds)` (any seed): all 88 piano pitches struck every 0.5 s, each sounding
    until the next strike or the end of the clip, as (intervals (n, 2) in seconds, pitches (n,) in Hz)."""
    n = int(round(seconds * SR))
    seg = int(0.5 * SR)
    intervals, pitches = [], []
    for s in range(0, n, seg):
        for midi in range(21, 109):
            intervals.append((s / SR, min(s + seg, n) / SR))
            pitches.append(_hz(midi))
    return np.array(intervals, np.float64).reshape(-1, 2), np.array(pitches, np.float64)


def dense_chords_clip(seconds: float = 10.0, seed: int = 7) -> np.ndarray:
    rng = np.random.default_rng(seed)
    n = int(round(seconds * SR))
    x = np.zeros(n)
    seg = int(0.5 * SR)
    tt = np.arange(seg) / SR
    env = np.exp(-4.0 * tt) * np.minimum(1.0, tt / 0.005)
    for s in range(0, n, seg):
        chord = np.zeros(seg)
        for midi in range(21, 109):
            f0 = 440.0 * 2 ** ((midi - 69) / 12)
            for h in range(1, 5):
                if f0 * h < SR / 2:
                    chord += np.sin(2 * np.pi * f0 * h * tt + rng.uniform(0, 2 * np.pi)) / h
        m = min(seg, n - s)
        x[s : s + m] += (env * chord)[:m]
    return _normalise(x)


def window_batch(n_windows: int, seed: int = 2, n_samples: int = 43844) -> np.ndarray:
    """(n_windows, 43844) float32: one long random-notes signal chopped into model windows
    (a few distinct windows tiled when n_windows is large, so generation stays cheap)."""
    distinct = min(n_windows, 64)
    clip = random_notes_clip(distinct * n_samples / SR, seed)
    base = clip[: distinct * n_samples].reshape(distinct, n_samples)
    reps = -(-n_windows // distinct)
    return np.ascontiguousarray(np.tile(base, (reps, 1))[:n_windows])
