"""ORACLE (test infrastructure, not product code): NumPy restatement of the reference note decode.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` legs may
import this module.  The product path never does.

Restates, function by function, reference: basic_pitch/note_creation.py
  * `constrain_frequency`          :314-343
  * `get_infered_onsets`           :289-311
  * `output_to_notes_polyphonic`   :360-511   (peak pick :398-404, onset loop :409-447, melodia :449-509)
  * `get_pitch_bends`              :182-219   (`midi_pitch_to_contour_bin` :168-179)
  * `model_frames_to_time`         :346-357
  * `model_output_to_notes`        :52-116    (minus the pretty_midi object)
  * `drop_overlapping_pitch_bends` :274-286
and the two `librosa` one-liners it calls (`hz_to_midi`, `midi_to_hz`, `frames_to_time`).

dtype discipline follows the reference exactly (SURVEY.md Appendix B): `frames` stay float32, the
onset matrix becomes float64 once onsets are inferred, thresholds are Python floats (float64
compares), amplitudes are float32 `np.mean` results.

Parity pin: checked against the reference's golden `tests/resources/vocadito_10/note_events.npz`
(reference: tests/test_inference.py:72-76) and against outputs of the reference module itself
imported through `oracle/ref_shims` (fixtures + generator in tests/golden/).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

SR = 22050
HOP = 256
N_FRAMES_WINDOW = 172
N_SAMPLES_WINDOW = 43844
MIDI_OFFSET = 21
TOP_PITCH_IDX = 87
N_CONTOUR_BINS = 264
ALIGN_OFFSET = 0.0018


def hz_to_midi(hz):
    return 12 * (np.log2(np.asanyarray(hz)) - np.log2(440.0)) + 69


def midi_to_hz(m):
    return 440.0 * (2.0 ** ((np.asanyarray(m) - 69.0) / 12.0))


def constrain_frequency(onsets, frames, max_freq: Optional[float], min_freq: Optional[float],
                        lo_col: Optional[int] = None, hi_col: Optional[int] = None):
    """Zero (IN PLACE, like the reference) pitch columns outside [min_freq, max_freq).  `lo_col` / `hi_col` give the
    column range directly (the library's min_pitch_idx / max_pitch_idx) and take precedence over the frequencies."""
    lo, hi = 0, onsets.shape[1]
    if min_freq is not None:
        lo = int(np.round(hz_to_midi(min_freq) - MIDI_OFFSET))
    if max_freq is not None:
        hi = int(np.round(hz_to_midi(max_freq) - MIDI_OFFSET))
    if lo_col is not None:
        lo = int(lo_col)
    if hi_col is not None:
        hi = int(hi_col)
    for m in (onsets, frames):
        m[:, :lo] = 0
        m[:, hi:] = 0
    return onsets, frames


def infer_onsets(onsets: np.ndarray, frames: np.ndarray, n_diff: int = 2) -> np.ndarray:
    """float64 (T,88): max(onsets, rescaled positive frame differences)."""
    n_t, n_f = frames.shape
    f64 = frames.astype(np.float64)
    diff = None
    for n in range(1, n_diff + 1):
        lagged = np.concatenate([np.zeros((n, n_f)), f64])[:n_t]
        d = f64 - lagged
        diff = d if diff is None else np.minimum(diff, d)
    diff[diff < 0] = 0
    diff[:n_diff, :] = 0
    with np.errstate(invalid="ignore", divide="ignore"):
        diff = np.max(onsets) * diff / np.max(diff)
    return np.maximum(onsets.astype(np.float64), diff)


def strict_time_peaks(m: np.ndarray) -> np.ndarray:
    """Boolean (T,F): strictly greater than both time neighbours; first/last frame never
    (== scipy.signal.argrelmax(m, axis=0, order=1, mode='clip'))."""
    pk = np.zeros(m.shape, dtype=bool)
    if m.shape[0] >= 3:
        with np.errstate(invalid="ignore"):
            pk[1:-1] = (m[1:-1] > m[:-2]) & (m[1:-1] > m[2:])
    return pk


def output_to_notes_polyphonic(
    frames: np.ndarray,
    onsets: np.ndarray,
    onset_thresh: float,
    frame_thresh: float,
    min_note_len: int,
    infer_onsets_flag: bool,
    max_freq: Optional[float],
    min_freq: Optional[float],
    melodia_trick: bool = True,
    energy_tol: int = 11,
    lo_col: Optional[int] = None,
    hi_col: Optional[int] = None,
) -> List[Tuple[int, int, int, np.float32]]:
    n_t = frames.shape[0]
    onsets, frames = constrain_frequency(onsets, frames, max_freq, min_freq, lo_col, hi_col)
    if infer_onsets_flag:
        onsets = infer_onsets(onsets, frames)

    pk = strict_time_peaks(onsets)
    peak_val = np.where(pk, onsets, 0.0).astype(np.float64)
    with np.errstate(invalid="ignore"):
        cand_t, cand_f = np.where(peak_val >= onset_thresh)
    cand_t, cand_f = cand_t[::-1], cand_f[::-1]  # latest first, highest pitch first within a frame

    energy = np.array(frames, dtype=np.float64)  # "remaining energy"
    notes: List[Tuple[int, int, int, np.float32]] = []

    def wipe(t0: int, t1: int, f: int) -> None:
        energy[t0:t1, f] = 0
        if f < TOP_PITCH_IDX:
            energy[t0:t1, f + 1] = 0
        if f > 0:
            energy[t0:t1, f - 1] = 0

    for t0, f in zip(cand_t, cand_f):
        t0, f = int(t0), int(f)
        if t0 >= n_t - 1:
            continue
        i, quiet = t0 + 1, 0
        while i < n_t - 1 and quiet < energy_tol:
            quiet = quiet + 1 if energy[i, f] < frame_thresh else 0
            i += 1
        i -= quiet
        if i - t0 <= min_note_len:
            continue
        wipe(t0, i, f)
        notes.append((t0, i, f + MIDI_OFFSET, np.mean(frames[t0:i, f])))

    if melodia_trick:
        while np.max(energy) > frame_thresh:
            tm, f = np.unravel_index(np.argmax(energy), energy.shape)
            tm, f = int(tm), int(f)
            energy[tm, f] = 0
            # forward
            i, quiet = tm + 1, 0
            while i < n_t - 1 and quiet < energy_tol:
                quiet = quiet + 1 if energy[i, f] < frame_thresh else 0
                wipe(i, i + 1, f)
                i += 1
            t_end = i - 1 - quiet
            # backward
            i, quiet = tm - 1, 0
            while i > 0 and quiet < energy_tol:
                quiet = quiet + 1 if energy[i, f] < frame_thresh else 0
                wipe(i, i + 1, f)
                i -= 1
            t_start = i + 1 + quiet
            if t_end - t_start <= min_note_len:
                continue
            notes.append((t_start, t_end, f + MIDI_OFFSET, np.mean(frames[t_start:t_end, f])))
    return notes


def gaussian_window(m: int = 51, std: float = 5.0) -> np.ndarray:
    """== scipy.signal.windows.gaussian(m, std) (symmetric)."""
    n = np.arange(0, m) - (m - 1.0) / 2.0
    return np.exp(-(n**2) / (2 * std * std))


def pitch_bends(contours: np.ndarray, notes, tol: int = 25):
    win = gaussian_window(2 * tol + 1, 5.0)
    out = []
    for t0, t1, pitch, amp in notes:
        c = int(np.round(12.0 * 3 * np.log2(midi_to_hz(pitch) / 27.5)))
        lo = max(c - tol, 0)
        hi = min(N_CONTOUR_BINS, c + tol + 1)
        w = win[max(0, tol - c) : 2 * tol + 1 - max(0, c - (N_CONTOUR_BINS - tol - 1))]
        sub = contours[t0:t1, lo:hi] * w
        shift = tol - max(0, tol - c)
        out.append((t0, t1, pitch, amp, list(np.argmax(sub, axis=1) - shift)))
    return out


def frames_to_time(n_frames: int) -> np.ndarray:
    idx = np.arange(n_frames)
    t = (idx * HOP).astype(int) / float(SR)
    win = np.floor(idx / N_FRAMES_WINDOW)
    off = (HOP / SR) * (N_FRAMES_WINDOW - (N_SAMPLES_WINDOW / HOP)) + ALIGN_OFFSET
    return t - off * win


def model_output_to_note_events(
    output: Dict[str, np.ndarray],
    onset_thresh: float,
    frame_thresh: float,
    infer_onsets_flag: bool = True,
    min_note_len: int = 11,
    min_freq: Optional[float] = None,
    max_freq: Optional[float] = None,
    include_pitch_bends: bool = True,
    melodia_trick: bool = True,
    energy_tol: int = 11,
    lo_col: Optional[int] = None,
    hi_col: Optional[int] = None,
):
    """Returns (frame-indexed notes with bends, second-indexed note events)."""
    frames, onsets, contours = output["note"], output["onset"], output["contour"]
    notes = output_to_notes_polyphonic(
        frames, onsets, onset_thresh, frame_thresh, min_note_len, infer_onsets_flag, max_freq, min_freq, melodia_trick,
        energy_tol, lo_col, hi_col,
    )
    if include_pitch_bends:
        with_bends = pitch_bends(contours, notes)
    else:
        with_bends = [(a, b, p, amp, None) for a, b, p, amp in notes]
    times = frames_to_time(contours.shape[0])
    events = [(times[a], times[b], p, amp, bends) for a, b, p, amp, bends in with_bends]
    return with_bends, events


def drop_overlapping_pitch_bends(events):
    ev = sorted(events)
    for i in range(len(ev) - 1):
        for j in range(i + 1, len(ev)):
            if ev[j][0] >= ev[i][1]:
                break
            ev[i] = ev[i][:-1] + (None,)
            ev[j] = ev[j][:-1] + (None,)
    return ev
