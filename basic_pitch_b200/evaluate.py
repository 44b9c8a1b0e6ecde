"""Note-level and frame-level transcription scores (addition; no reference counterpart).

The library counts, per (setting, file) or item, the reference notes, the estimated notes and the size of a maximum
matching with and without the offset test (`Model.score_grid`, `Model.score_notes`, `inference.evaluate_grid`;
include/bp_b200.h, bp_score_*).  This module turns the counts into the precision, recall and F-measure of
mir_eval.transcription.precision_recall_f1_overlap (0.7, beta = 1, strict=False), by its formulas.

Frame level: the library sums, per (setting, file) or item, the seven counts of `FRAME_FIELDS` over the reference
frames (`Model.score_frames_grid`, `Model.score_multipitch`, `inference.evaluate_frames_grid`; include/bp_b200.h,
bp_score_frames_grid_* / bp_score_multipitch_host).  `frame_scores` turns them into the 14 numbers of
mir_eval.multipitch.metrics (0.7), bit for bit.

Matched pairs: the library also returns which estimated note mir_eval's matching pairs with each reference note
(`Model.match_grid`, `Model.match_notes`; include/bp_b200.h, bp_match_*).  `matching_scores` turns one file's pairs into
the average overlap ratio and the note scores with velocity (mir_eval.transcription_velocity), with mir_eval's own
NumPy expressions; `inference.evaluate_velocity_grid` does this for a grid of settings.

Onsets and offsets alone: the library counts, per (setting, file) or item, the onsets and the offsets matched without
the pitch test (`Model.score_onset_offset_grid`, `Model.score_onsets_offsets`; include/bp_b200.h,
bp_score_onset_offset_*); `onset_offset_scores` turns them into mir_eval's onset-only and offset-only scores, and
`inference.evaluate_transcription_grid` returns every value of mir_eval.transcription.evaluate (`TRANSCRIPTION_KEYS`)
for a grid of settings.

Posteriorgrams as multi-f0 estimates: `salience_to_multipitch` reads a contour (or note) posteriorgram under a
threshold, peak picking and a frequency range as the series those metrics score (include/bp_b200.h,
bp_score_salience_grid_*); `Model.score_salience_grid` / `inference.evaluate_salience_grid` score a grid of such
settings on the device.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import numpy as np

from . import constants
from .note_creation import model_frames_to_time

# mir_eval.transcription's defaults: onset within 50 ms, pitch within 50 cents, offset within
# max(0.2 x reference duration, 50 ms)
TOLERANCES = dict(onset_tolerance=0.05, pitch_tolerance=50.0, offset_ratio=0.2, offset_min_tolerance=0.05)

# log2(Hz) of MIDI numbers 0..127, the pitch of an estimated note as mir_eval sees it: np.log2 of
# `note_creation.midi_to_hz`
EST_LOG2_HZ = np.ascontiguousarray(np.log2(440.0 * 2.0 ** ((np.arange(128, dtype=np.float64) - 69.0) / 12.0)))

FIELDS = ("n_ref", "n_est", "matched_no_offset", "matched")

# Frame level: the default window of mir_eval.multipitch.metrics, in semitones
WINDOW = 0.5
FRAME_FIELDS = ("n_ref", "n_est", "tp", "tp_chroma", "n_min", "miss", "false_alarm")
_METRICS = ("precision", "recall", "accuracy", "substitution_error", "miss_error", "false_alarm_error", "total_error")


def multipitch_values(hz):
    """Pitches in Hz -> (midi, chroma) float64 as mir_eval.multipitch sees them: frequencies_to_midi, then
    midi_to_chroma followed by the np.mod of util._outer_distance_mod_n (chroma in [0, 12)).  A pitch <= 0 gives a
    non-finite midi, which the library rejects."""
    hz = np.asarray(hz, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        midi = 69.0 + 12.0 * np.log2(hz / 440.0)
        chroma = np.mod(np.mod(midi, 12), 12)
    return midi, chroma


# Values of the MIDI numbers 0..127 as an estimated note's pitch, from the Hz of EST_LOG2_HZ (`note_creation.midi_to_hz`)
EST_MIDI, EST_CHROMA = (np.ascontiguousarray(a) for a in
                        multipitch_values(440.0 * 2.0 ** ((np.arange(128, dtype=np.float64) - 69.0) / 12.0)))


def notes_to_multipitch(intervals, pitches_hz, times) -> List[np.ndarray]:
    """Note annotations -> a multi-pitch series at `times` (non-decreasing, seconds): frame t holds the Hz of every note
    with onset <= t < offset, in note order.  This is how note annotations become frame references, and, at
    `note_creation.model_frames_to_time`, the estimate series the grid scorer builds from decoded notes."""
    iv = np.asarray(intervals, np.float64).reshape(-1, 2)
    hz = np.asarray(pitches_hz, np.float64).reshape(-1)
    t = np.asarray(times, np.float64).reshape(-1)
    if len(iv) != len(hz):
        raise ValueError(f"{len(iv)} intervals but {len(hz)} pitches")
    lo = np.searchsorted(t, iv[:, 0], side="left")  # first frame at or after the onset
    hi = np.maximum(np.searchsorted(t, iv[:, 1], side="left"), lo)  # first frame at or after the offset
    n = hi - lo
    frame = np.repeat(lo - np.cumsum(n) + n, n) + np.arange(n.sum())
    note = np.repeat(np.arange(len(hz)), n)
    if len(t) == 0:
        return []
    order = np.argsort(frame, kind="stable")
    cuts = np.searchsorted(frame[order], np.arange(1, len(t)))
    return np.split(hz[note[order]], cuts)


_SALIENCE_HZ = {"contour": constants.FREQ_BINS_CONTOURS, "note": constants.FREQ_BINS_NOTES}


def salience_bins(kind: str = "contour") -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(hz, midi, chroma) float64 of every bin of the contour (264 bins, a third of a semitone) or note (88 bins)
    posteriorgram: the reference's target grids constants.FREQ_BINS_CONTOURS / FREQ_BINS_NOTES, with their values as
    `multipitch_values` gives them."""
    if kind not in _SALIENCE_HZ:
        raise ValueError(f"kind must be 'contour' or 'note', got {kind!r}")
    hz = np.ascontiguousarray(_SALIENCE_HZ[kind], np.float64)
    midi, chroma = multipitch_values(hz)
    return hz, np.ascontiguousarray(midi), np.ascontiguousarray(chroma)


def salience_bin_range(kind: str, minimum_frequency: Optional[float], maximum_frequency: Optional[float]):
    """The bins [lo, hi) of a frequency range: lo is the first bin with Hz >= minimum_frequency, hi the first bin with
    Hz > maximum_frequency (np.searchsorted on the bin table); None leaves that side open.  A range below its lower end
    is empty (hi = lo)."""
    hz = salience_bins(kind)[0]
    lo = 0 if minimum_frequency is None else int(np.searchsorted(hz, float(minimum_frequency), side="left"))
    hi = len(hz) if maximum_frequency is None else int(np.searchsorted(hz, float(maximum_frequency), side="right"))
    return lo, max(lo, hi)


def salience_to_multipitch(gram, threshold: float, peak_picking: bool = True, minimum_frequency: Optional[float] = None,
                           maximum_frequency: Optional[float] = None, kind: str = "contour"):
    """A posteriorgram (T, bins) as a multi-f0 estimate (times (T,), [Hz array per frame]), mir_eval.multipitch's
    convention: frame t at the model frame time holds, in ascending order, the Hz of every bin b in the frequency range
    (`salience_bin_range`) with float64(gram[t, b]) >= threshold and, with peak_picking, a local maximum of the whole
    row in float32 (scipy.signal.argrelmax(gram, axis=1): 1 <= b <= bins - 2 and strictly above both neighbours).
    NaN cells are never estimates.  This is the host definition of bp_score_salience_grid_* (include/bp_b200.h).

    The threshold is compared in float64 on purpose: NumPy 2 compares a float32 array with a Python float in float32,
    which answers differently for a threshold between two float32 values."""
    hz = salience_bins(kind)[0]
    g = np.asarray(gram, np.float32)
    if g.ndim != 2 or g.shape[1] != len(hz):
        raise ValueError(f"a {kind} posteriorgram must be (T, {len(hz)}), got {g.shape}")
    threshold = float(threshold)
    if not (np.isfinite(threshold) and threshold > 0):
        raise ValueError(f"threshold must be finite and > 0, got {threshold}")
    est = g.astype(np.float64) >= threshold
    if peak_picking:
        peak = np.zeros(g.shape, bool)
        mid = g[:, 1:-1]
        peak[:, 1:-1] = (mid > g[:, :-2]) & (mid > g[:, 2:])
        est &= peak
    lo, hi = salience_bin_range(kind, minimum_frequency, maximum_frequency)
    est[:, :lo] = False
    est[:, hi:] = False
    return model_frames_to_time(g.shape[0]), [hz[np.flatnonzero(row)] for row in est]


def frame_scores(counts) -> Dict[str, np.ndarray]:
    """counts (..., 7) as `Model.score_frames_grid` / `score_multipitch` return them -> dict of float64 arrays of shape
    counts.shape[:-1]: precision, recall, accuracy, substitution_error, miss_error, false_alarm_error, total_error and
    the same seven with a "chroma_" prefix, by mir_eval.multipitch's formulas (0 where a denominator is 0; every error
    is 0 when n_ref is 0).  "mean" holds them averaged over the last axis, as in `note_scores`."""
    c = np.asarray(counts, np.int64)
    if c.ndim < 1 or c.shape[-1] != 7:
        raise ValueError(f"counts must have shape (..., 7), got {c.shape}")
    n_ref, n_est, tp, tpc, n_min, miss, fa = (c[..., k].astype(np.float64) for k in range(7))

    def div(a, b):
        return np.where(b > 0, a / np.where(b > 0, b, 1.0), 0.0)

    out: Dict[str, np.ndarray] = {}
    for prefix, t in (("", tp), ("chroma_", tpc)):
        vals = (div(t, n_est), div(t, n_ref), div(t, n_est + n_ref - t), div(n_min - t, n_ref), div(miss, n_ref),
                div(fa, n_ref), div(n_min + miss + fa - t, n_ref))
        out.update({prefix + k: v for k, v in zip(_METRICS, vals)})
    if c.ndim >= 2:
        n = c.shape[-2]
        out["mean"] = {k: (v.mean(axis=-1) if n else np.zeros(v.shape[:-1])) for k, v in out.items()}
    else:
        out["mean"] = {k: (v.mean() if v.size else np.float64(0.0)) for k, v in out.items()}
    return out


def note_scores(counts) -> Dict[str, np.ndarray]:
    """counts (..., 4) as `Model.score_grid` / `score_notes` return them -> dict of float64 arrays of shape counts.shape[:-1]:
    precision, recall, f_measure (with offsets) and precision_no_offset, recall_no_offset, f_measure_no_offset.
    P = m / n_est, R = m / n_ref, F = 2 P R / (P + R) (0 when P = R = 0); all three 0 when either side is empty.
    "mean" holds the same six names averaged over the last axis (over files for a grid: one value per setting; 0 where
    that axis is empty)."""
    c = np.asarray(counts, np.int64)
    if c.ndim < 1 or c.shape[-1] != 4:
        raise ValueError(f"counts must have shape (..., 4), got {c.shape}")
    n_ref, n_est = c[..., 0], c[..., 1]
    empty = (n_ref == 0) | (n_est == 0)
    out: Dict[str, np.ndarray] = {}
    for suffix, m in (("", c[..., 3]), ("_no_offset", c[..., 2])):
        with np.errstate(divide="ignore", invalid="ignore"):
            p = np.where(empty, 0.0, m / n_est)
            r = np.where(empty, 0.0, m / n_ref)
            f = np.where((p == 0) & (r == 0), 0.0, 2.0 * p * r / (p + r))
        out["precision" + suffix], out["recall" + suffix], out["f_measure" + suffix] = p, r, f
    if c.ndim >= 2:
        n = c.shape[-2]
        out["mean"] = {k: (v.mean(axis=-1) if n else np.zeros(v.shape[:-1])) for k, v in out.items()}
    else:
        out["mean"] = {k: (v.mean() if v.size else np.float64(0.0)) for k, v in out.items()}
    return out


# Columns of `Model.score_onset_offset_grid` / `score_onsets_offsets`
ONSET_OFFSET_FIELDS = ("n_ref", "n_est", "onset_matched", "offset_matched")

# mir_eval.transcription.evaluate's keys, in its order, and the names the evaluate_* functions give those values
TRANSCRIPTION_KEYS = {
    "Precision": "precision",
    "Recall": "recall",
    "F-measure": "f_measure",
    "Average_Overlap_Ratio": "average_overlap_ratio",
    "Precision_no_offset": "precision_no_offset",
    "Recall_no_offset": "recall_no_offset",
    "F-measure_no_offset": "f_measure_no_offset",
    "Average_Overlap_Ratio_no_offset": "average_overlap_ratio_no_offset",
    "Onset_Precision": "onset_precision",
    "Onset_Recall": "onset_recall",
    "Onset_F-measure": "onset_f_measure",
    "Offset_Precision": "offset_precision",
    "Offset_Recall": "offset_recall",
    "Offset_F-measure": "offset_f_measure",
}

_ONSET_OFFSET_NAMES = {"precision_no_offset": "onset_precision", "recall_no_offset": "onset_recall",
                       "f_measure_no_offset": "onset_f_measure", "precision": "offset_precision",
                       "recall": "offset_recall", "f_measure": "offset_f_measure"}


def onset_offset_scores(counts) -> Dict[str, np.ndarray]:
    """counts (..., 4) as `Model.score_onset_offset_grid` / `score_onsets_offsets` return them -> dict of float64
    arrays of shape counts.shape[:-1]: onset_precision, onset_recall, onset_f_measure (mir_eval.transcription's
    onset_precision_recall_f1) and offset_precision, offset_recall, offset_f_measure (offset_precision_recall_f1).
    The formulas are `note_scores`' on the same four columns (0 when either side is empty); "mean" as there."""
    c = np.asarray(counts, np.int64)
    if c.ndim < 1 or c.shape[-1] != 4:
        raise ValueError(f"counts must have shape (..., 4), got {c.shape}")
    s = note_scores(c)
    out = {name: s[k] for k, name in _ONSET_OFFSET_NAMES.items()}
    out["mean"] = {name: s["mean"][k] for k, name in _ONSET_OFFSET_NAMES.items()}
    return out


# Keys of `matching_scores`; each also exists with a "_no_offset" suffix (the pass without the offset test)
MATCH_FIELDS = ("average_overlap_ratio", "velocity_precision", "velocity_recall", "velocity_f_measure",
                "velocity_average_overlap_ratio")


def note_velocities(amplitude) -> np.ndarray:
    """The MIDI velocity the library writes for a note of this amplitude (note_events_to_midi, csrc/midi_events.h
    velocity_of): int(np.round(np.float32(127) * amplitude)), in float32."""
    return np.round(np.float32(127) * np.asarray(amplitude, np.float32)).astype(np.int64)


def check_velocities(velocities, what: str = "velocities") -> np.ndarray:
    """float64 copy of one file's velocities; ValueError naming the first that is not finite or is < 0 (mir_eval's
    transcription_velocity.validate rejects them)."""
    v = np.asarray(velocities, np.float64).reshape(-1)
    bad = np.flatnonzero(~(np.isfinite(v) & (v >= 0)))
    if len(bad):
        raise ValueError(f"{what} note {int(bad[0])}: velocity must be finite and >= 0, got {v[bad[0]]}")
    return v


def _overlap_ratio(ref_iv, est_iv, r, e) -> float:
    """transcription.average_overlap_ratio over the pairs (r[k], e[k]), in that order; 0 without pairs."""
    if len(r) == 0:
        return 0.0
    a, b = ref_iv[r], est_iv[e]
    return np.mean((np.minimum(a[:, 1], b[:, 1]) - np.maximum(a[:, 0], b[:, 0])) /
                   (np.maximum(a[:, 1], b[:, 1]) - np.minimum(a[:, 0], b[:, 0])))


def matching_scores(ref_intervals, ref_velocities, est_intervals, est_velocities, match,
                    velocity_tolerance: float = 0.1) -> Dict[str, np.float64]:
    """The scores of one file that depend on which pairs mir_eval 0.7 matches, from the library's matchings.

    ref_intervals (n_ref, 2) and est_intervals (n_est, 2) in seconds; velocities finite and >= 0 (an estimated note's is
    `note_velocities` of its amplitude); match (2, n_ref) as `Model.match_grid` / `match_notes` return it: per reference
    note the estimate index or -1, row 0 without and row 1 with the offset test.  Returns float64 values for
    average_overlap_ratio (transcription.precision_recall_f1_overlap's fourth value) and velocity_precision,
    velocity_recall, velocity_f_measure, velocity_average_overlap_ratio (transcription_velocity.precision_recall_f1_overlap,
    velocity_tolerance as there), each with offsets and with a "_no_offset" suffix without.

    The velocity step is mir_eval's: reference velocities become (v - min) / max(1, max - min); a least-squares line
    np.linalg.lstsq([est_v, 1], ref_v) through the matched pairs rescales the estimated ones; a pair is kept when
    |slope est_v + intercept - ref_v| < velocity_tolerance.  Every value is 0 when either side is empty."""
    ref_iv = np.asarray(ref_intervals, np.float64).reshape(-1, 2)
    est_iv = np.asarray(est_intervals, np.float64).reshape(-1, 2)
    rv = check_velocities(ref_velocities, "references")
    ev = check_velocities(est_velocities, "estimates")
    m = np.asarray(match, np.int64).reshape(2, -1)
    n_ref, n_est = len(rv), len(ev)
    if len(ref_iv) != n_ref or len(est_iv) != n_est or m.shape[1] != n_ref:
        raise ValueError(f"{len(ref_iv)} reference intervals, {n_ref} velocities, {m.shape[1]} matches; "
                         f"{len(est_iv)} estimated intervals, {n_est} velocities")
    out: Dict[str, np.float64] = {}
    for suffix, row in (("", m[1]), ("_no_offset", m[0])):
        r = np.flatnonzero(row >= 0)  # sorted(matching.items()): ascending reference index
        e = row[r]
        if len(r) and (e.max() >= n_est):
            raise ValueError(f"match refers to estimate {int(e.max())} of {n_est}")
        vals = dict.fromkeys(MATCH_FIELDS, np.float64(0.0))
        if n_ref and n_est:
            vals["average_overlap_ratio"] = np.float64(_overlap_ratio(ref_iv, est_iv, r, e))
            if len(r):
                v_min, v_max = np.min(rv), np.max(rv)
                rn = (rv - v_min) / float(max(1, v_max - v_min))
                slope, intercept = np.linalg.lstsq(np.vstack([ev[e], np.ones(len(e))]).T, rn[r])[0]
                keep = np.abs(slope * ev[e] + intercept - rn[r]) < velocity_tolerance
                r, e = r[keep], e[keep]
            p, rc = float(len(r)) / n_est, float(len(r)) / n_ref
            vals["velocity_precision"], vals["velocity_recall"] = np.float64(p), np.float64(rc)
            vals["velocity_f_measure"] = np.float64(0.0 if p == 0 and rc == 0 else 2 * p * rc / (p + rc))
            vals["velocity_average_overlap_ratio"] = np.float64(_overlap_ratio(ref_iv, est_iv, r, e))
        out.update({k + suffix: v for k, v in vals.items()})
    return out
