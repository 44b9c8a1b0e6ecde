"""NumPy / SciPy restatement of mir_eval.melody 0.7 (tests only).

`to_cent_voicing`, `resample_melody_series` and the five metric functions follow mir_eval.melody.evaluate with its
default arguments (hop=None, kind='linear', base_frequency=10, cent_tolerance=50, no est_voicing / ref_reward), with
scipy.interpolate.interp1d doing the interpolation, so SciPy decides every edge case.  `counts` returns the seven
integers the library's melody scorers return per (setting, file) or item (include/bp_b200.h, bp_score_melody_*),
`counts_cents` the same for series given as cents and voicing (as the library takes them), and `evaluate` the five
floats, in mir_eval's order and under its key names.

One case mir_eval does not define (it indexes est_time[0]): an estimate of no frames is read as unvoiced, cents 0, at
every reference frame.
"""
from __future__ import annotations

import collections

import numpy as np
import scipy.interpolate


def hz2cents(freq_hz, base_frequency=10.0):
    freq_hz = np.asarray(freq_hz, np.float64)
    freq_cent = np.zeros(freq_hz.shape[0])
    nz = np.flatnonzero(freq_hz)
    freq_cent[nz] = 1200 * np.log2(np.abs(freq_hz[nz]) / base_frequency)
    return freq_cent


def freq_to_voicing(frequencies):
    frequencies = np.asarray(frequencies, np.float64)
    return np.abs(frequencies), (frequencies > 0).astype(float)


def resample_melody_series(times, frequencies, voicing, times_new, kind="linear"):
    """The binary-voicing branch of mir_eval.melody.resample_melody_series (without its warning)."""
    if times.shape == times_new.shape and np.allclose(times, times_new):
        return frequencies, voicing
    times = np.round(times, 10)
    times_new = np.round(times_new, 10)
    if times_new.max() > times.max():
        times = np.append(times, times_new.max())
        frequencies = np.append(frequencies, 0)
        voicing = np.append(voicing, 0)
    frequencies_held = np.array(frequencies)
    for n, frequency in enumerate(frequencies[1:]):
        if frequency == 0:
            frequencies_held[n + 1] = frequencies_held[n]
    frequencies_resampled = scipy.interpolate.interp1d(times, frequencies_held, kind)(times_new)
    frequency_mask = scipy.interpolate.interp1d(times, frequencies, "zero")(times_new)
    frequencies_resampled *= frequency_mask != 0
    voicing_resampled = scipy.interpolate.interp1d(times, voicing, "zero")(times_new)
    return frequencies_resampled, voicing_resampled


def to_cent_voicing(ref_time, ref_freq, est_time, est_freq, base_frequency=10.0, kind="linear"):
    ref_time, ref_freq = np.asarray(ref_time, np.float64), np.asarray(ref_freq, np.float64)
    est_time, est_freq = np.asarray(est_time, np.float64), np.asarray(est_freq, np.float64)
    if len(ref_time) and ref_time[0] > 0:
        ref_time = np.insert(ref_time, 0, 0)
        ref_freq = np.insert(ref_freq, 0, ref_freq[0])
    if len(est_time) and est_time[0] > 0:
        est_time = np.insert(est_time, 0, 0)
        est_freq = np.insert(est_freq, 0, est_freq[0])
    ref_freq, ref_voicing = freq_to_voicing(ref_freq)
    est_freq, est_voicing = freq_to_voicing(est_freq)
    ref_cent = hz2cents(ref_freq, base_frequency)
    est_cent = hz2cents(est_freq, base_frequency)
    if len(est_time) == 0:
        return ref_voicing, ref_cent, np.zeros(len(ref_time)), np.zeros(len(ref_time))
    if len(ref_time) == 0:
        return ref_voicing, ref_cent, np.zeros(0), np.zeros(0)
    est_cent, est_voicing = resample_melody_series(est_time, est_cent, est_voicing, ref_time, kind=kind)
    return ref_voicing, ref_cent, est_voicing, est_cent


def voicing_recall(ref_voicing, est_voicing):
    if ref_voicing.size == 0 or est_voicing.size == 0:
        return 0.0
    ref_indicator = (ref_voicing > 0).astype(float)
    if np.sum(ref_indicator) == 0:
        return 1
    return np.sum(est_voicing * ref_indicator) / np.sum(ref_indicator)


def voicing_false_alarm(ref_voicing, est_voicing):
    if ref_voicing.size == 0 or est_voicing.size == 0:
        return 0.0
    ref_indicator = (ref_voicing == 0).astype(float)
    if np.sum(ref_indicator) == 0:
        return 0
    return np.sum(est_voicing * ref_indicator) / np.sum(ref_indicator)


def raw_pitch_accuracy(ref_voicing, ref_cent, est_voicing, est_cent, cent_tolerance=50):
    if ref_voicing.size == 0 or ref_voicing.sum() == 0 or ref_cent.size == 0 or est_cent.size == 0:
        return 0.0
    nonzero_freqs = np.logical_and(est_cent != 0, ref_cent != 0)
    if sum(nonzero_freqs) == 0:
        return 0.0
    freq_diff_cents = np.abs(ref_cent - est_cent)[nonzero_freqs]
    correct_frequencies = freq_diff_cents < cent_tolerance
    return np.sum(ref_voicing[nonzero_freqs] * correct_frequencies) / np.sum(ref_voicing)


def raw_chroma_accuracy(ref_voicing, ref_cent, est_voicing, est_cent, cent_tolerance=50):
    if ref_voicing.size == 0 or ref_voicing.sum() == 0 or ref_cent.size == 0 or est_cent.size == 0:
        return 0.0
    nonzero_freqs = np.logical_and(est_cent != 0, ref_cent != 0)
    if sum(nonzero_freqs) == 0:
        return 0.0
    freq_diff_cents = np.abs(ref_cent - est_cent)[nonzero_freqs]
    octave = 1200.0 * np.floor(freq_diff_cents / 1200 + 0.5)
    correct_chroma = np.abs(freq_diff_cents - octave) < cent_tolerance
    return np.sum(ref_voicing[nonzero_freqs] * correct_chroma) / np.sum(ref_voicing)


def overall_accuracy(ref_voicing, ref_cent, est_voicing, est_cent, cent_tolerance=50):
    if ref_voicing.size == 0 or est_voicing.size == 0 or ref_cent.size == 0 or est_cent.size == 0:
        return 0.0
    n_frames = float(len(ref_voicing))
    ratio = 0.0 if np.sum(ref_voicing) == 0 else 1.0
    nonzero_freqs = np.logical_and(est_cent != 0, ref_cent != 0)
    freq_diff_cents = np.abs(ref_cent - est_cent)[nonzero_freqs]
    correct_frequencies = freq_diff_cents < cent_tolerance
    ref_binary = (ref_voicing > 0).astype(float)
    return (ratio * np.sum(ref_voicing[nonzero_freqs] * est_voicing[nonzero_freqs] * correct_frequencies) +
            np.sum((1.0 - ref_binary) * (1.0 - est_voicing))) / n_frames


def evaluate(ref_time, ref_freq, est_time, est_freq, cent_tolerance=50):
    """mir_eval.melody.evaluate's five scores (an OrderedDict under mir_eval's keys)."""
    rv, rc, ev, ec = to_cent_voicing(ref_time, ref_freq, est_time, est_freq)
    scores = collections.OrderedDict()
    scores["Voicing Recall"] = voicing_recall(rv, ev)
    scores["Voicing False Alarm"] = voicing_false_alarm(rv, ev)
    scores["Raw Pitch Accuracy"] = raw_pitch_accuracy(rv, rc, ev, ec, cent_tolerance)
    scores["Raw Chroma Accuracy"] = raw_chroma_accuracy(rv, rc, ev, ec, cent_tolerance)
    scores["Overall Accuracy"] = overall_accuracy(rv, rc, ev, ec, cent_tolerance)
    return scores


def counts_resampled(rv, rc, ev, ec, cent_tolerance=50):
    """[n_frames, ref_voiced, voiced_hit, false_alarm, pitch_correct, chroma_correct, oa_voiced_correct] of the
    arrays to_cent_voicing returns."""
    rvb, evb = rv > 0, ev > 0
    nz = (ec != 0) & (rc != 0)
    d = np.abs(rc - ec)
    pitch = nz & rvb & (d < cent_tolerance)
    chroma = nz & rvb & (np.abs(d - 1200.0 * np.floor(d / 1200 + 0.5)) < cent_tolerance)
    return [len(rv), int(rvb.sum()), int((rvb & evb).sum()), int((~rvb & evb).sum()), int(pitch.sum()),
            int(chroma.sum()), int((pitch & evb).sum())]


def counts(ref_time, ref_freq, est_time, est_freq, cent_tolerance=50):
    return counts_resampled(*to_cent_voicing(ref_time, ref_freq, est_time, est_freq), cent_tolerance)


def counts_cents(ref_time, ref_cent, ref_voicing, est_time, est_cent, est_voicing, cent_tolerance=50):
    """`counts` of series given as cents and voicing (what the library takes, include/bp_b200.h): the steps of
    `to_cent_voicing` after hz2cents, then `resample_melody_series` and `counts_resampled`."""
    ref_time, est_time = np.asarray(ref_time, np.float64), np.asarray(est_time, np.float64)
    ref_cent, est_cent = np.asarray(ref_cent, np.float64), np.asarray(est_cent, np.float64)
    ref_voicing, est_voicing = np.asarray(ref_voicing, np.float64), np.asarray(est_voicing, np.float64)
    if len(ref_time) and ref_time[0] > 0:
        ref_time = np.insert(ref_time, 0, 0)
        ref_cent = np.insert(ref_cent, 0, ref_cent[0])
        ref_voicing = np.insert(ref_voicing, 0, ref_voicing[0])
    if len(est_time) and est_time[0] > 0:
        est_time = np.insert(est_time, 0, 0)
        est_cent = np.insert(est_cent, 0, est_cent[0])
        est_voicing = np.insert(est_voicing, 0, est_voicing[0])
    if len(est_time) == 0:
        ev, ec = np.zeros(len(ref_time)), np.zeros(len(ref_time))
    elif len(ref_time) == 0:
        ev, ec = np.zeros(0), np.zeros(0)
    else:
        ec, ev = resample_melody_series(est_time, est_cent, est_voicing, ref_time)
    return counts_resampled(ref_voicing, ref_cent, ev, ec, cent_tolerance)
