"""Adversarial posteriorgram sets for the note decode (CPU only: plain NumPy, deterministic).

The shipped model's posteriorgrams are smooth and the default parameters fixed, which leaves most index arithmetic of
the decode (csrc/decode.cu, the decode half of csrc/api.cu) unobserved.  Each set is a list of files `(note, onset,
contour)` and the parameter grid it is meant for:

  lengths      files of 0 .. 4097 frames in one batch, most T * 88 not multiples of 32: 32-frame tiles and 32-cell
               candidate words straddle files; used with onset_thresh <= 0, so every cell is a candidate
  ties         a 3109-frame file (13 blocks of 256 frames) of values on a 1/8 grid: equal maxima on both sides of
               block boundaries, at t = 0 and T - 1, in adjacent and distant columns of one frame; notes spanning blocks;
               and an 8709-frame file (35 blocks) with tied maxima 32 blocks apart in one column
  runs         quiet runs of energy_tol - 1, energy_tol and energy_tol + 1 frames, starting 0, 31, 32 and 33 frames
               after the start of the scan, for the onset loop and both melodia scans; notes ending at T - 2 / T - 1,
               candidates at t = 1 and T - 2
  crowded      a file whose decode yields more than 8 T + 64 notes (the first allowance of note slots) between two
               ordinary files
  long_notes   isolated notes of unquantised float32 values, 1 .. 4097 frames: every branch of NumPy's pairwise sum
  pitch_edges  notes at pitches 21, 22, 29, 30, 100, 107, 108 (the pitch-bend window clipped at contour bins 0 and
               263) whose contour rows have exactly tied weighted products, values below 0 and above 1
  nan_file     a time-constant file (max(frame_diff) == 0: inferred onsets all NaN) and a file whose onsets are all 0,
               between ordinary files, in one batch

Values that must tie are multiples of 1/64 (exact in float32 and float64).  Liveness of each set (that it reaches what
it is built for) is checked in tests/test_postsets.py; the reference decode's output on every set and grid is pinned in
tests/golden/decode_edges.npz (oracle/make_golden.py).
"""
from __future__ import annotations

import functools
from typing import Dict, List, Tuple

import numpy as np

NAMES = ("lengths", "ties", "runs", "crowded", "long_notes", "pitch_edges", "nan_file")
N_PITCH, N_BINS = 88, 264
BLOCK = 256  # frames per block of the melodia loop's block maxima (csrc/decode.cu: kDecBlk)

File = Tuple[np.ndarray, np.ndarray, np.ndarray]


def params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=11, infer_onsets=True, melodia_trick=True,
           lo_col=0, hi_col=N_PITCH) -> Dict:
    return dict(onset_thresh=float(onset_thresh), frame_thresh=float(frame_thresh), min_note_len=int(min_note_len),
                energy_tol=int(energy_tol), infer_onsets=bool(infer_onsets), melodia_trick=bool(melodia_trick),
                lo_col=int(lo_col), hi_col=int(hi_col))


def _q(x, step=64) -> np.ndarray:
    return (np.round(np.asarray(x, np.float64) * step) / step).astype(np.float32)


def _blobs(rng, n_t, n_f, density, max_len, lo=0.25, hi=1.0, step=64):
    """Sparse plateaus (random length, value on a 1/step grid) over a zero background."""
    x = np.zeros((n_t, n_f), np.float32)
    for _ in range(int(density * n_t * n_f / 100)):
        f, t0 = int(rng.integers(0, n_f)), int(rng.integers(0, max(n_t, 1)))
        ln = int(rng.integers(1, max_len + 1))
        x[t0 : t0 + ln, f] = rng.uniform(lo, hi)
    return _q(x, step)


def _contour(rng, n_t):
    """A sawtooth over the contour bins that moves with the frame (period 13, 17 or 19 bins, random phase and speed):
    every frame's pitch-bend arg-max differs from its neighbours', while the bends repeat and the fixture stays small."""
    period, speed, phase = int(rng.choice([13, 17, 19])), int(rng.integers(1, 6)), int(rng.integers(0, 19))
    t, b = np.arange(n_t)[:, None], np.arange(N_BINS)[None, :]
    return _q(((b + speed * t + phase) % period) / period)


def _ordinary(rng, n_t) -> File:
    return _blobs(rng, n_t, N_PITCH, 3.0, 40), _blobs(rng, n_t, N_PITCH, 1.0, 3), _contour(rng, n_t)


# ------------------------------------------------------------------------------------------------------------- lengths
LENGTHS = (0, 1, 2, 3, 4, 5, 31, 32, 33, 63, 255, 256, 257, 511, 512, 513, 1023, 4097)


def _lengths():
    rng = np.random.default_rng(101)
    order = rng.permutation(len(LENGTHS))
    files = []
    for i in order:
        n_t = LENGTHS[i]
        note = _blobs(rng, n_t, N_PITCH, 0.3, 30)
        onset = _blobs(rng, n_t, N_PITCH, 0.5, 2)
        if n_t >= 3:  # the first and last rows share their 32-cell candidate words with the neighbouring files; a
            # two-frame plateau at t = 0 is a note from the candidate at t = 0 (min_note_len 1, energy_tol 1)
            note[0:2, 1::3] = 0.75
            note[2, 1::3] = 0.0
            note[-2:, ::3] = 0.5
        files.append((note, onset, _contour(rng, n_t)))
    grid = [
        params(onset_thresh=0.0, frame_thresh=0.3, min_note_len=1, energy_tol=1),
        params(onset_thresh=-0.1, frame_thresh=0.05, min_note_len=1, energy_tol=2, infer_onsets=False, lo_col=1, hi_col=87),
        params(onset_thresh=0.0, frame_thresh=0.3, min_note_len=11, energy_tol=33, melodia_trick=False),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=128, energy_tol=300),
    ]
    return files, grid


# ---------------------------------------------------------------------------------------------------------------- ties
TIES_T = 12 * BLOCK + 37


def _ties():
    """Background plateaus on a 1/8 grid (many accidental ties) plus planted maxima:
      1.0   at (255, 10) and (256, 40): a tie on both sides of the first block boundary, lower frame first;
            at (0, 60) and (T - 1, 62), (T - 1, 70): ties at the first and the last frame;
            at (600, 20), (600, 21) [adjacent columns] and (600, 75) [distant]: same-frame ties;
            at (700, 30) and (1100, 30): one column, tied maxima in two blocks (the lower block wins);
            at (511, 50) and (512, 52): the second block boundary
      0.875 long notes in columns 5, 44, 83 spanning 3 - 5 blocks, and a column whose later maximum lies in a block the
            note before touched (1300 - 1560 in column 15, then 1545 in column 16)."""
    rng = np.random.default_rng(202)
    n_t = TIES_T
    note = _blobs(rng, n_t, N_PITCH, 2.5, 60, lo=0.3, hi=0.8, step=8)
    onset = np.zeros((n_t, N_PITCH), np.float32)
    onset[::97, ::5] = 0.875
    note[250:262, 10] = 0.5
    note[255, 10] = 1.0
    note[256:270, 40] = 0.5
    note[256, 40] = 1.0
    note[0:12, 60] = 0.625
    note[0, 60] = 1.0
    note[n_t - 14 :, 62] = 0.625
    note[n_t - 1, 62] = 1.0
    note[n_t - 9 :, 70] = 0.625
    note[n_t - 1, 70] = 1.0
    for f in (20, 21, 75):
        note[590:615, f] = 0.5
        note[600, f] = 1.0
    note[690:720, 30] = 0.5
    note[700, 30] = 1.0
    note[1090:1120, 30] = 0.5
    note[1100, 30] = 1.0
    note[505:512, 50] = 0.625
    note[511, 50] = 1.0
    note[512:530, 52] = 0.625
    note[512, 52] = 1.0
    note[300:1200, 5] = 0.875  # blocks 1 - 4
    note[1500:2800, 44] = 0.875  # blocks 5 - 10
    note[2000:2600, 83] = 0.875  # blocks 7 - 10
    note[1300:1560, 15] = 0.875  # blocks 5 - 6
    note[1545:1600, 16] = 0.75  # starts in block 6, inside the range the note in column 15 wipes
    contour = _contour(rng, n_t)
    # more than 32 blocks: a lane of the block reduction holds blocks b and b + 32; tied maxima in blocks 1 and 33 of
    # column 12, and one in column 50 between them in time
    n_long = 34 * BLOCK + 5
    long_note = np.zeros((n_long, N_PITCH), np.float32)
    for t, f in ((300, 12), (4000, 50), (33 * BLOCK + 52, 12)):
        long_note[t - 20 : t + 20, f] = 0.5
        long_note[t, f] = 1.0
    long_file = (long_note, np.zeros_like(long_note), _contour(rng, n_long))
    grid = [
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=11, infer_onsets=False),
        params(onset_thresh=0.95, frame_thresh=0.05, min_note_len=0, energy_tol=2, infer_onsets=False),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=1, energy_tol=64),
        params(onset_thresh=0.95, frame_thresh=0.3, min_note_len=128, energy_tol=300, infer_onsets=False),
        params(onset_thresh=0.95, frame_thresh=0.3, min_note_len=11, energy_tol=33, infer_onsets=False, lo_col=40,
               hi_col=41),
        params(onset_thresh=0.95, frame_thresh=0.3, min_note_len=11, energy_tol=2**31 - 1, infer_onsets=False),
    ]
    return [(note, onset, contour), long_file], grid


# ---------------------------------------------------------------------------------------------------------------- runs
RUN_TOLS = (11, 32, 33, 64)
RUN_OFFSETS = (0, 31, 32, 33)


def _runs_file(rng, tol):
    """Columns 2, 4, .. host one experiment each: (kind, offset, run length).  kind 0: onset-loop note from a candidate at
    t0; kind 1: melodia forward scan from a maximum at tm; kind 2: melodia backward scan from a maximum at tm.  The run
    of quiet frames (value 1/8 < 0.3) starts `offset` frames after the scan's first frame, then the note resumes."""
    exps = [(k, o, r) for k in range(3) for o in RUN_OFFSETS for r in (tol - 1, tol, tol + 1)]
    act = 40  # active frames after the run
    n_t = 2 + 34 + (tol + 1) + act + 4 + 40
    note = np.zeros((n_t, N_PITCH), np.float32)
    onset = np.zeros((n_t, N_PITCH), np.float32)
    for j, (kind, off, run) in enumerate(exps[:40]):
        f = 2 + 2 * j
        if kind < 2:  # scan runs forward from s = t + 1
            t = 2 + int(rng.integers(0, 3))
            s = t + 1
            note[t : s + off + run + act, f] = 0.5
            note[s + off : s + off + run, f] = 0.125
            if kind == 0:
                onset[t, f] = 0.75
            else:
                note[t, f] = 0.75
        else:  # backward from s = tm - 1
            tm = n_t - 3 - int(rng.integers(0, 3))
            s = tm - 1
            note[s - off - run - act + 1 : tm + 1, f] = 0.5
            note[s - off - run + 1 : s - off + 1, f] = 0.125
            note[tm, f] = 0.75
    # ends and starts at the edges of the file
    note[1:, 82] = 0.5
    onset[1, 82] = 0.75  # candidate at t = 1, note to T - 1
    note[1 : n_t - 2, 84] = 0.5
    onset[1, 84] = 0.625  # note to T - 2
    onset[n_t - 2, 86] = 0.75  # candidate at T - 2 (a one-frame note at most)
    note[n_t - 2 :, 86] = 0.5
    note[0:30, 87] = 0.5
    note[0, 87] = 0.625  # melodia maximum at t = 0 (the backward scan never runs)
    return note, onset, _contour(rng, n_t)


def _runs():
    rng = np.random.default_rng(303)
    files = [_runs_file(rng, tol) for tol in RUN_TOLS]
    grid = []
    for tol in (1, 11, 31, 32, 33, 64):
        grid.append(params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0 if tol % 2 else 1, energy_tol=tol,
                           infer_onsets=False))
    grid.append(params(onset_thresh=0.5, frame_thresh=0.0, min_note_len=0, energy_tol=32, infer_onsets=False))
    grid.append(params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=33, infer_onsets=True,
                       melodia_trick=False))
    return files, grid


# ------------------------------------------------------------------------------------------------------------- crowded
CROWDED_T = 200


def _crowded():
    """Onset peaks at every odd frame of every column: with min_note_len 0 every candidate is a note (the onset loop never
    looks at the energy of the candidate's own frame), 44 notes per frame against the first allowance of 8 per frame."""
    rng = np.random.default_rng(404)
    n_t = CROWDED_T
    note = _blobs(rng, n_t, N_PITCH, 4.0, 6, lo=0.2, hi=0.9)
    onset = np.zeros((n_t, N_PITCH), np.float32)
    onset[1::2] = 0.75
    files = [_ordinary(rng, 150), (note, onset, _contour(rng, n_t)), _ordinary(rng, 171)]
    grid = [
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, energy_tol=1, infer_onsets=False),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=1, energy_tol=2, infer_onsets=False),
        params(onset_thresh=0.5, frame_thresh=0.05, min_note_len=0, energy_tol=1, infer_onsets=True),
    ]
    return files, grid


# ---------------------------------------------------------------------------------------------------------- long_notes
LONG_LENGTHS = tuple(range(1, 18)) + (127, 128, 129, 135, 136, 137, 255, 256, 257, 1000, 4097)
LONG_T = 4160


def _long_notes():
    """One note per column (every third column), onset peak at t0, values uniform in [0.3, 1) as float32 (no rounding),
    then quiet values in [0, 0.25).  Onset loop: the note is [t0, t0 + L); melodia alone: [t0, t0 + L - 1)."""
    rng = np.random.default_rng(505)
    n_t = LONG_T
    note = (0.25 * rng.random((n_t, N_PITCH))).astype(np.float32)
    onset = np.zeros((n_t, N_PITCH), np.float32)
    for j, ln in enumerate(LONG_LENGTHS):
        f = 3 * j
        t0 = 2 + int(rng.integers(0, max(1, n_t - ln - 40)))
        note[t0 : t0 + ln, f] = (0.3 + 0.7 * rng.random(ln)).astype(np.float32)
        onset[t0, f] = 0.75
    contour = rng.random((n_t, N_BINS)).astype(np.float32)
    grid = [
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, energy_tol=11, infer_onsets=False),
        params(onset_thresh=1.5, frame_thresh=0.3, min_note_len=0, energy_tol=11, infer_onsets=False),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=128, energy_tol=2, infer_onsets=False,
               melodia_trick=False),
    ]
    return [(note, onset, contour)], grid


# --------------------------------------------------------------------------------------------------------- pitch_edges
EDGE_PITCHES = (21, 22, 29, 30, 100, 107, 108)
EDGE_T = 260


def edge_bend_row(rng, c, kind):
    """One contour row for a note at contour bin c.  kind 0: two bins at equal distance on both sides of c (or, where
    the window is clipped, all window bins) hold the row's largest value — a tie of the weighted products; 1: all
    zero; 2: the top / bottom bin of the window dominates with a value > 1; 3: negative values with ties;
    4: unquantised noise."""
    row = _q(rng.random(N_BINS) * 0.5, 64)
    lo, hi = max(c - 25, 0), min(N_BINS, c + 26)
    if kind == 0:
        d = int(rng.integers(1, 6))
        if c - d >= lo and c + d < hi:
            row[lo:hi] = np.minimum(row[lo:hi], 0.25)
            row[c - d] = row[c + d] = 0.75
        else:
            row[lo:hi] = 0.5
    elif kind == 1:
        row[:] = 0.0
    elif kind == 2:
        row[lo:hi] = 0.25
        row[hi - 1 if c > N_BINS // 2 else lo] = 1.5
    elif kind == 3:
        row[:] = -0.5
        d = int(rng.integers(1, 4))
        if c - d >= lo and c + d < hi:
            row[lo:hi] = -1.0
            row[c - d] = row[c + d] = -0.25
    else:
        row = (rng.random(N_BINS) * 1.5 - 0.25).astype(np.float32)
    return row


def edge_notes():
    """(start, end, pitch) of the notes of the pitch_edges file, also given to bp_pitch_bends_host directly."""
    out = []
    for j, p in enumerate(EDGE_PITCHES):
        t0 = 3 + 36 * j
        ln = (34, 9, 40, 12, 33, 70, 64)[j]
        out.append((t0, min(t0 + ln, EDGE_T - 1), p))
    return out


def _pitch_edges():
    rng = np.random.default_rng(606)
    n_t = EDGE_T
    note = np.zeros((n_t, N_PITCH), np.float32)
    onset = np.zeros((n_t, N_PITCH), np.float32)
    contour = _q(rng.random((n_t, N_BINS)) * 0.5, 64)
    for t0, t1, p in edge_notes():
        f = p - 21
        note[t0:t1, f] = 0.5
        onset[t0, f] = 0.75
        for t in range(t0, t1):
            contour[t] = edge_bend_row(rng, 3 * f, (t - t0) % 5)
    grid = [
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, energy_tol=11, infer_onsets=False),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=11, infer_onsets=False, lo_col=1, hi_col=87),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, energy_tol=11, infer_onsets=False, lo_col=87, hi_col=88),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=0, energy_tol=11, lo_col=0, hi_col=0),
        params(onset_thresh=-0.1, frame_thresh=0.3, min_note_len=11, energy_tol=11, lo_col=50, hi_col=20),
    ]
    return [(note, onset, contour)], grid


# ------------------------------------------------------------------------------------------------------------ nan_file
def _nan_file():
    rng = np.random.default_rng(707)
    const = (np.full((70, N_PITCH), 0.5, np.float32), np.full((70, N_PITCH), 0.25, np.float32), _contour(rng, 70))
    a = _ordinary(rng, 45)
    zero_onsets = _ordinary(rng, 50)
    zero_onsets = (zero_onsets[0], np.zeros_like(zero_onsets[1]), zero_onsets[2])
    files = [a, const, _ordinary(rng, 33), zero_onsets, _ordinary(rng, 90)]
    grid = [
        params(),
        params(onset_thresh=0.0, frame_thresh=0.05, min_note_len=1, energy_tol=2),
        params(onset_thresh=-0.1, frame_thresh=0.05, min_note_len=11, energy_tol=1, infer_onsets=False),
        params(onset_thresh=0.5, frame_thresh=0.0, min_note_len=0, energy_tol=31),
        params(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=11, melodia_trick=False),
    ]
    return files, grid


_BUILDERS = {
    "lengths": _lengths, "ties": _ties, "runs": _runs, "crowded": _crowded, "long_notes": _long_notes,
    "pitch_edges": _pitch_edges, "nan_file": _nan_file,
}  # fmt: skip


@functools.lru_cache(maxsize=None)
def _cached(name):
    return _BUILDERS[name]()


def file_sha(f: File) -> bytes:
    """SHA-256 of one (note, onset, contour) triple: identifies the inputs a fixture was made from."""
    import hashlib

    h = hashlib.sha256()
    for a in f:
        h.update(np.ascontiguousarray(a, np.float32).tobytes())
    return h.digest()


def get(name: str) -> Tuple[List[File], List[Dict]]:
    """(files, parameter grid) of a set; the arrays are fresh copies (the reference decode zeroes its inputs in place)."""
    files, grid = _cached(name)
    return [tuple(np.array(a, copy=True) for a in f) for f in files], [dict(p) for p in grid]
