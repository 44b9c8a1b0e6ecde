"""Note decode host interface (mirrors the names of reference: basic_pitch/note_creation.py).

The arithmetic of the reference's `output_to_notes_polyphonic` / `get_pitch_bends`
(note_creation.py:360-511, 182-219) runs on the GPU (csrc/decode.cu via `bp_decode_host`); this
module converts arguments, maps frames to seconds and assembles the MIDI object.
"""
from __future__ import annotations

import os
from collections import defaultdict
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from .constants import (
    ANNOT_N_FRAMES,
    ANNOTATIONS_BASE_FREQUENCY,
    ANNOTATIONS_N_SEMITONES,
    AUDIO_N_SAMPLES,
    AUDIO_SAMPLE_RATE,
    CONTOURS_BINS_PER_SEMITONE,
    DEFAULT_MIN_NOTE_LEN,
    ENERGY_TOLERANCE,
    FFT_HOP,
    MAGIC_ALIGNMENT_OFFSET,
    MAX_FREQ_IDX,
    MIDI_OFFSET,
    MIDI_VELOCITY_SCALE,
    N_FREQ_BINS_CONTOURS,
    N_PITCH_BEND_TICKS,
    PITCH_BEND_SCALE,
)

try:  # the real package when present, else the bundled minimal containers
    import pretty_midi  # type: ignore
except ImportError:  # pragma: no cover - depends on the environment
    from . import midi as pretty_midi

NoteEvent = Tuple[float, float, int, float, Optional[List[int]]]


def hz_to_midi(hz):
    return 12 * (np.log2(np.asanyarray(hz)) - np.log2(440.0)) + 69


def midi_to_hz(midi):
    return 440.0 * (2.0 ** ((np.asanyarray(midi) - 69.0) / 12.0))


def midi_pitch_to_contour_bin(pitch_midi: int) -> np.ndarray:
    """reference: note_creation.py:168-179"""
    return 12.0 * CONTOURS_BINS_PER_SEMITONE * np.log2(midi_to_hz(pitch_midi) / ANNOTATIONS_BASE_FREQUENCY)


def frequency_to_column_range(min_freq: Optional[float], max_freq: Optional[float], n_cols: int = ANNOTATIONS_N_SEMITONES) -> Tuple[int, int]:
    """Columns kept by the reference's `constrain_frequency` (note_creation.py:329-341), as [lo, hi).

    The reference writes `m[:, :min_idx] = 0; m[:, max_idx:] = 0` with unclamped indices, so NumPy's
    slice rules apply (a negative index counts from the end); this reproduces them exactly.
    """
    lo, hi = 0, n_cols
    if min_freq is not None:
        lo = int(np.round(hz_to_midi(min_freq) - MIDI_OFFSET))
    if max_freq is not None:
        hi = int(np.round(hz_to_midi(max_freq) - MIDI_OFFSET))
    lo = slice(None, lo).indices(n_cols)[1]  # end of the zeroed prefix
    hi = slice(hi, None).indices(n_cols)[0]  # start of the zeroed suffix
    return lo, hi


def constrain_frequency(onsets: np.ndarray, frames: np.ndarray, max_freq: Optional[float], min_freq: Optional[float]):
    """Zero pitch columns outside the range, IN PLACE like the reference (note_creation.py:314-343)."""
    lo, hi = frequency_to_column_range(min_freq, max_freq, onsets.shape[1])
    for m in (onsets, frames):
        m[:, :lo] = 0
        m[:, hi:] = 0
    return onsets, frames


def model_frames_to_time(n_frames: int) -> np.ndarray:
    """reference: note_creation.py:346-357 (librosa.frames_to_time inlined)."""
    idx = np.arange(n_frames)
    original_times = (idx * FFT_HOP).astype(int) / float(AUDIO_SAMPLE_RATE)
    window_numbers = np.floor(idx / ANNOT_N_FRAMES)
    window_offset = (FFT_HOP / AUDIO_SAMPLE_RATE) * (ANNOT_N_FRAMES - (AUDIO_N_SAMPLES / FFT_HOP)) + MAGIC_ALIGNMENT_OFFSET
    return original_times - (window_offset * window_numbers)


def _decode(output, onset_thresh, frame_thresh, infer_onsets, min_note_len, min_freq, max_freq, include_pitch_bends,
            melodia_trick, energy_tol=ENERGY_TOLERANCE, model=None):
    from .inference import default_model

    mdl = model if model is not None else default_model()
    frames, onsets, contours = output["note"], output["onset"], output.get("contour")
    lo, hi = frequency_to_column_range(min_freq, max_freq, frames.shape[1])
    res = mdl.decode_arrays(
        [frames], [onsets], [contours] if contours is not None else None,
        onset_thresh=onset_thresh, frame_thresh=frame_thresh, min_note_len=min_note_len, energy_tol=energy_tol,
        infer_onsets=infer_onsets, melodia_trick=melodia_trick, include_pitch_bends=include_pitch_bends,
        min_pitch_idx=lo, max_pitch_idx=hi,
    )[0]
    # the reference zeroes the out-of-range columns of the caller's arrays (note_creation.py:338-341)
    if min_freq is not None or max_freq is not None:
        for m in (onsets, frames):
            if m.flags.writeable:
                m[:, :lo] = 0
                m[:, hi:] = 0
    return res


def output_to_notes_polyphonic(frames, onsets, onset_thresh, frame_thresh, min_note_len, infer_onsets, max_freq,
                               min_freq, melodia_trick=True, energy_tol=ENERGY_TOLERANCE, model=None):
    """reference: note_creation.py:360-511 -> [(start_frame, end_frame, pitch_midi, amplitude)]"""
    res = _decode({"note": frames, "onset": onsets}, onset_thresh, frame_thresh, infer_onsets, min_note_len, min_freq,
                  max_freq, False, melodia_trick, energy_tol, model)
    return [(int(a), int(b), int(p), np.float32(amp)) for a, b, p, amp in zip(res["start"], res["end"], res["pitch"], res["amp"])]


def model_output_to_notes(
    output: Dict[str, np.ndarray],
    onset_thresh: float,
    frame_thresh: float,
    infer_onsets: bool = True,
    min_note_len: int = DEFAULT_MIN_NOTE_LEN,
    min_freq: Optional[float] = None,
    max_freq: Optional[float] = None,
    include_pitch_bends: bool = True,
    multiple_pitch_bends: bool = False,
    melodia_trick: bool = True,
    midi_tempo: float = 120,
    model=None,
):
    """reference: note_creation.py:52-116 -> (PrettyMIDI, note events in seconds)."""
    res = _decode(output, onset_thresh, frame_thresh, infer_onsets, min_note_len, min_freq, max_freq,
                  include_pitch_bends, melodia_trick, model=model)
    events = note_events_from_arrays(res, output["contour"].shape[0], include_pitch_bends)
    return note_events_to_midi(events, multiple_pitch_bends, midi_tempo), events


_NOTES_SETTING = dict(onset_thresh=None, frame_thresh=None, infer_onsets=True, min_note_len=DEFAULT_MIN_NOTE_LEN,
                      min_freq=None, max_freq=None, include_pitch_bends=True, multiple_pitch_bends=False,
                      melodia_trick=True, midi_tempo=120)
# predict's keyword names (inference.py) -> model_output_to_notes'; minimum_note_length is in milliseconds
_PREDICT_SETTING = dict(onset_threshold=("onset_thresh", 0.5), frame_threshold=("frame_thresh", 0.3),
                        minimum_note_length=("min_note_len", 127.7), minimum_frequency=("min_freq", None),
                        maximum_frequency=("max_freq", None), multiple_pitch_bends=("multiple_pitch_bends", False),
                        melodia_trick=("melodia_trick", True), midi_tempo=("midi_tempo", 120))


def grid_setting(setting: Dict, predict_names: bool = False) -> Tuple[Dict, Dict]:
    """One setting of a grid decode -> (`Model.decode_arrays` keyword arguments, `note_events_to_midi` keyword arguments),
    with the arithmetic `model_output_to_notes` (`_decode`) and `predict` apply to the same arguments: Hz limits to the
    columns `frequency_to_column_range` gives, and with predict_names=True `predict`'s keyword names and defaults
    (onset_threshold, frame_threshold, minimum_note_length in ms -> frames, minimum_frequency, maximum_frequency,
    multiple_pitch_bends, melodia_trick, midi_tempo).  Otherwise `model_output_to_notes`' names; onset_thresh and
    frame_thresh are required as there.  Unknown names raise TypeError."""
    s = dict(setting)
    if predict_names:
        unknown = set(s) - set(_PREDICT_SETTING)
        if unknown:
            raise TypeError(f"unknown predict argument(s) {sorted(unknown)}")
        s = {name: s.get(k, default) for k, (name, default) in _PREDICT_SETTING.items()}
        s["min_note_len"] = int(np.round(s["min_note_len"] / 1000 * (AUDIO_SAMPLE_RATE / FFT_HOP)))
    unknown = set(s) - set(_NOTES_SETTING)
    if unknown:
        raise TypeError(f"unknown model_output_to_notes argument(s) {sorted(unknown)}")
    s = {**_NOTES_SETTING, **s}
    if s["onset_thresh"] is None or s["frame_thresh"] is None:
        raise TypeError("a setting needs onset_thresh and frame_thresh")
    lo, hi = frequency_to_column_range(s["min_freq"], s["max_freq"])
    decode = dict(onset_thresh=s["onset_thresh"], frame_thresh=s["frame_thresh"], min_note_len=s["min_note_len"],
                  energy_tol=ENERGY_TOLERANCE, infer_onsets=s["infer_onsets"], melodia_trick=s["melodia_trick"],
                  include_pitch_bends=s["include_pitch_bends"], min_pitch_idx=lo, max_pitch_idx=hi)
    return decode, dict(multiple_pitch_bends=s["multiple_pitch_bends"], midi_tempo=s["midi_tempo"])


def model_output_to_notes_grid(output: Dict[str, np.ndarray], settings: Sequence[Dict], model=None):
    """`model_output_to_notes(output, **setting)` for every setting of a grid, decoded in one library call
    (`Model.decode_grid`, `bp_decode_grid_host`).  A setting is a dict of `model_output_to_notes`' keyword arguments
    (min_freq / max_freq in Hz included).  Returns one (midi, note_events) per setting, each equal to that call's.

    Unlike `model_output_to_notes` (and the reference's `constrain_frequency`), the arrays of `output` are NOT modified:
    the settings may disagree on the frequency range, so no zeroing of the caller's columns would fit them all."""
    from .inference import default_model

    mdl = model if model is not None else default_model()
    conv = [grid_setting(s) for s in settings]
    contour = output.get("contour")
    res = mdl.decode_grid([output["note"]], [output["onset"]], None if contour is None else [contour], [d for d, _ in conv])
    n_frames = output["note"].shape[0]
    out = []
    for (d, midi_kw), r in zip(conv, res):
        events = note_events_from_arrays(r[0], n_frames, d["include_pitch_bends"])
        out.append((note_events_to_midi(events, **midi_kw), events))
    return out


def note_events_from_arrays(res: Dict[str, np.ndarray], n_frames: int, include_pitch_bends: bool = True) -> List[NoteEvent]:
    """Decode arrays (frames) -> the reference's list of (start_s, end_s, pitch, amplitude, bends)."""
    times = model_frames_to_time(n_frames)
    start, end, pitch, amp = res["start"], res["end"], res["pitch"], res["amp"]
    off, flat = res["bend_off"], res["bends"]
    events: List[NoteEvent] = []
    for j in range(len(start)):
        bends = list(flat[off[j] : off[j + 1]].astype(np.int64)) if include_pitch_bends else None
        events.append((times[start[j]], times[end[j]], np.int64(pitch[j]), np.float32(amp[j]), bends))
    return events


class NoteEventList(Sequence):
    """The note events of one file as a read-only sequence of the reference's tuples
    (start_s, end_s, pitch_midi, amplitude, [pitch bends]) backed by the arrays of the batch: tuples are made when an
    element is read.  A 1 250-clip batch has ~10^5 notes and ~2 x 10^6 pitch-bend values; turning all of them into
    Python objects costs more host time than the whole GPU pass, and most callers hand the events straight to a writer.
    Compares equal to the equivalent list; `to_list()` materialises it."""

    __slots__ = ("_st", "_en", "_pitch", "_amp", "_boff", "_flat")

    def __init__(self, st, en, pitch, amp, boff, flat):
        self._st, self._en, self._pitch, self._amp, self._boff, self._flat = st, en, pitch, amp, boff, flat

    def __len__(self) -> int:
        return len(self._st)

    def _one(self, j: int) -> NoteEvent:
        bends = None if self._flat is None else self._flat[self._boff[j] : self._boff[j + 1]].tolist()
        return (self._st[j], self._en[j], self._pitch[j], self._amp[j], bends)

    def __getitem__(self, i):
        if isinstance(i, slice):
            return [self._one(j) for j in range(*i.indices(len(self)))]
        n = len(self)
        if i < 0:
            i += n
        if not 0 <= i < n:
            raise IndexError("note event index out of range")
        return self._one(i)

    def __iter__(self):
        return iter(self.to_list())

    def to_list(self) -> List[NoteEvent]:
        n = len(self)
        if self._flat is None:
            bends: list = [None] * n
        else:
            bo = self._boff.tolist()
            fl = self._flat[bo[0] : bo[n]].tolist() if n else []
            b0 = bo[0] if n else 0
            bends = [fl[bo[j] - b0 : bo[j + 1] - b0] for j in range(n)]
        return list(zip(list(self._st), list(self._en), list(self._pitch), list(self._amp), bends))

    def __eq__(self, other) -> bool:
        if isinstance(other, (list, tuple, NoteEventList)):
            return self.to_list() == (other.to_list() if isinstance(other, NoteEventList) else list(other))
        return NotImplemented

    def __repr__(self) -> str:
        return f"NoteEventList({self.to_list()!r})"


def note_events_batch(arrs: Dict[str, np.ndarray], n_files: int, include_pitch_bends: bool = True,
                      lazy: bool = True) -> List[Sequence]:
    """`note_events_from_arrays` for every file of a batch at once (the concatenated arrays of one library call): the
    frame -> seconds mapping and the type conversions are vectorised over all notes of the batch.  Same values and
    element types as the per-file function (np.float64 times, np.int64 pitch, np.float32 amplitude; the pitch bends
    are Python ints).  lazy=True returns `NoteEventList`s, lazy=False plain lists."""
    noff = arrs["note_off"]
    n = int(noff[n_files])
    start, end = arrs["start"][:n], arrs["end"][:n]
    times = model_frames_to_time(int(max(int(start.max(initial=0)), int(end.max(initial=0)))) + 1)
    st, en = times[start], times[end]
    pitch, amp = arrs["pitch"][:n].astype(np.int64), arrs["amp"][:n]
    boff = arrs["bend_off"][: n + 1] if include_pitch_bends else None
    flat = arrs["bends"] if include_pitch_bends else None
    offs = noff[: n_files + 1].tolist()
    out = [NoteEventList(st[a:b], en[a:b], pitch[a:b], amp[a:b], None if boff is None else boff[a : b + 1], flat)
           for a, b in zip(offs[:-1], offs[1:])]
    return out if lazy else [e.to_list() for e in out]


def _pack_note_events(event_lists: Sequence[Sequence]):
    """The events of a batch as the concatenated arrays of the batch entry points (include/bp_b200.h: bp_write_note_files,
    bp_sonify_notes_host) -> (note_off int32, start_s f64, end_s f64, pitch int32, amplitude f32, bend_off int32, bends
    int32).  event_lists: one `NoteEventList` (or list of event tuples) per file."""
    n_files = len(event_lists)
    per = []
    for ev in event_lists:
        if isinstance(ev, NoteEventList):
            n = len(ev)
            if ev._flat is None or n == 0:
                boff, flat = np.zeros(n + 1, np.int64), np.zeros(0, np.int32)
            else:
                b0, b1 = int(ev._boff[0]), int(ev._boff[n])
                boff, flat = ev._boff.astype(np.int64) - b0, ev._flat[b0:b1]
            per.append((ev._st, ev._en, ev._pitch, ev._amp, boff, flat))
        else:
            ev = list(ev)
            bl = [list(e[4]) if e[4] else [] for e in ev]
            boff = np.zeros(len(ev) + 1, np.int64)
            boff[1:] = np.cumsum([len(b) for b in bl])
            per.append((np.array([e[0] for e in ev], np.float64), np.array([e[1] for e in ev], np.float64),
                        np.array([e[2] for e in ev], np.int64), np.array([e[3] for e in ev], np.float32), boff,
                        np.array([x for b in bl for x in b], np.int32)))
    cat = lambda k, dt: np.ascontiguousarray(np.concatenate([p[k] for p in per]) if per else np.zeros(0), dtype=dt)  # noqa: E731
    noff = np.zeros(n_files + 1, np.int32)
    noff[1:] = np.cumsum([len(p[0]) for p in per])
    st, en, pitch, amp, flat = cat(0, np.float64), cat(1, np.float64), cat(2, np.int32), cat(3, np.float32), cat(5, np.int32)
    boff = np.zeros(int(noff[-1]) + 1, np.int32)
    base = 0
    for i, p in enumerate(per):
        a, b = int(noff[i]), int(noff[i + 1])
        boff[a : b + 1] = p[4] + base
        base += int(p[4][-1])
    return noff, st, en, pitch, amp, boff, flat


def write_note_files(event_lists: Sequence[Sequence], midi_paths: Optional[Sequence], csv_paths: Optional[Sequence],
                     multiple_pitch_bends: bool = False, midi_tempo: float = 120, n_threads: int = 0) -> None:
    """One MIDI file and / or one note-event CSV per file of a batch in a single library call (`bp_write_note_files`,
    csrc/writers.cu: host threads over the files, no per-note Python objects).  Same bytes as
    `note_events_to_midi(events, ...).write(path)` with this package's MIDI writer and `inference.save_note_events`.
    event_lists: one `NoteEventList` (or list of event tuples) per file; paths: one per file, None entries are skipped."""
    import ctypes as C

    from . import _lib

    n_files = len(event_lists)
    noff, st, en, pitch, amp, boff, flat = _pack_note_events(event_lists)

    def c_paths(paths):
        if paths is None:
            return None
        assert len(paths) == n_files
        return (C.c_char_p * max(n_files, 1))(*[None if q is None else os.fsencode(str(q)) for q in paths])

    _lib.load().bp_write_note_files(n_files, c_paths(midi_paths), c_paths(csv_paths), noff.ctypes.data, st.ctypes.data,
                                    en.ctypes.data, pitch.ctypes.data, amp.ctypes.data, boff.ctypes.data, flat.ctypes.data,
                                    int(bool(multiple_pitch_bends)), float(midi_tempo), int(n_threads))


def sonify_batch(event_lists: Sequence[Sequence], sr: int = 44100, multiple_pitch_bends: bool = False,
                 model=None) -> List[np.ndarray]:
    """`note_events_to_midi(events, multiple_pitch_bends).synthesize(sr)` of the bundled `midi` stand-in for every file
    of a batch, rendered on the GPU in one library call (`bp_sonify_notes_host`, csrc/sonify.cu).  Returns one float64
    array per file (empty for a file without notes), views of one page-locked block.  The samples differ from the
    stand-in's only by the rounding of the phase (DESIGN.md §4.4).  event_lists: one `NoteEventList` (or list of event
    tuples) per file."""
    from .inference import default_model

    mdl = model if model is not None else default_model()
    n_files = len(event_lists)
    noff, st, en, pitch, amp, boff, flat = _pack_note_events(event_lists)
    soff = np.zeros(n_files + 1, np.int64)
    args = (n_files, noff.ctypes.data, st.ctypes.data, en.ctypes.data, pitch.ctypes.data, amp.ctypes.data,
            boff.ctypes.data, flat.ctypes.data, int(bool(multiple_pitch_bends)), int(sr), soff.ctypes.data)
    mdl._lib.bp_sonify_notes_host(mdl.handle, *args, None, 0)  # size query
    total = int(soff[-1])
    out = mdl._pinned.array((total,), np.float64)
    mdl._lib.bp_sonify_notes_host(mdl.handle, *args, out.ctypes.data, total)
    offs = soff.tolist()
    return [out[a:b] for a, b in zip(offs[:-1], offs[1:])]


def drop_overlapping_pitch_bends(note_events_with_pitch_bends: List[NoteEvent]) -> List[NoteEvent]:
    """reference: note_creation.py:274-286 — notes overlapping in time lose their pitch bends."""
    ev = sorted(note_events_with_pitch_bends)
    for i in range(len(ev) - 1):
        for j in range(i + 1, len(ev)):
            if ev[j][0] >= ev[i][1]:
                break
            ev[i] = ev[i][:-1] + (None,)
            ev[j] = ev[j][:-1] + (None,)
    return ev


class LazyPrettyMIDI(pretty_midi.PrettyMIDI):
    """The MIDI object of `note_events_to_midi`, assembled on first use.  A batch call returns one per file; most
    callers only ever `write()` a few of them or hand them to a batch writer, so the Instrument / Note / PitchBend
    objects (a dozen Python objects per note) are not created until `instruments` is first read."""

    def __init__(self, note_events: List[NoteEvent], multiple_pitch_bends: bool = False, midi_tempo: float = 120):
        self._pending = None
        self._instruments: list = []
        super().__init__(initial_tempo=midi_tempo)
        self._pending = (note_events, multiple_pitch_bends, midi_tempo)

    @property
    def instruments(self):
        if self._pending is not None:
            pending, self._pending = self._pending, None
            self._instruments = note_events_to_midi(*pending).instruments
        return self._instruments

    @instruments.setter
    def instruments(self, value):
        self._instruments = value


def note_events_to_midi(note_events_with_pitch_bends: List[NoteEvent], multiple_pitch_bends: bool = False,
                        midi_tempo: float = 120):
    """reference: note_creation.py:222-271"""
    mid = pretty_midi.PrettyMIDI(initial_tempo=midi_tempo)
    if not multiple_pitch_bends:
        note_events_with_pitch_bends = drop_overlapping_pitch_bends(note_events_with_pitch_bends)
    program = pretty_midi.instrument_name_to_program("Electric Piano 1")
    instruments = defaultdict(lambda: pretty_midi.Instrument(program=program))
    for start_time, end_time, note_number, amplitude, pitch_bend in note_events_with_pitch_bends:
        inst = instruments[note_number] if multiple_pitch_bends else instruments[0]
        inst.notes.append(
            pretty_midi.Note(velocity=int(np.round(MIDI_VELOCITY_SCALE * amplitude)), pitch=note_number,
                             start=start_time, end=end_time)
        )
        if not pitch_bend:
            continue
        bend_times = np.linspace(start_time, end_time, len(pitch_bend))
        ticks = np.round(np.array(pitch_bend) * PITCH_BEND_SCALE / CONTOURS_BINS_PER_SEMITONE).astype(int)
        ticks[ticks > N_PITCH_BEND_TICKS - 1] = N_PITCH_BEND_TICKS - 1
        ticks[ticks < -N_PITCH_BEND_TICKS] = -N_PITCH_BEND_TICKS
        for t, b in zip(bend_times, ticks):
            inst.pitch_bends.append(pretty_midi.PitchBend(b, t))
    mid.instruments.extend(instruments.values())
    return mid


def sonify_midi(midi, save_path, sr: Optional[int] = 44100) -> None:
    """reference: note_creation.py:119-128 — `midi.synthesize(sr)` written as a WAV.  With the real `pretty_midi` that is
    its synthesiser; the bundled `midi.PrettyMIDI` (and `LazyPrettyMIDI`) has an additive stand-in of the same shape."""
    from scipy.io import wavfile

    wavfile.write(save_path, sr, midi.synthesize(sr))


SONIFY_FS = 3000  # reference: note_creation.py:41


def sonify_salience(gram, semitone_resolution: float, save_path: Optional[str] = None, thresh: float = 0.2):
    """reference: note_creation.py:131-165 -> (audio at SONIFY_FS, SONIFY_FS).  gram: (n_freqs, n_times) salience in 0..1,
    log-spaced from ANNOTATIONS_BASE_FREQUENCY with `semitone_resolution` bins per semitone; values below `thresh` are
    zeroed IN PLACE like the reference.  The reference calls mir_eval.sonify.time_frequency and resampy; neither is a
    dependency here, so this restates what they do for this call: one sinusoid per frequency bin below SONIFY_FS / 2,
    amplitude = the bin's salience held from frame to frame (nearest frame time), summed and peak-normalised; the saved
    file is resampled to 44.1 kHz with this package's Kaiser polyphase resampler.  Not sample-identical to mir_eval."""
    gram = np.asarray(gram)
    n_bins = int(ANNOTATIONS_N_SEMITONES * semitone_resolution)
    freqs = ANNOTATIONS_BASE_FREQUENCY * 2.0 ** (np.arange(n_bins) / (12.0 * semitone_resolution))
    max_freq_idx = int(np.where(freqs > SONIFY_FS / 2)[0][0])
    hop = AUDIO_N_SAMPLES / ANNOT_N_FRAMES  # "THIS IS THE CORRECT HOP" (reference :154)
    times = (np.arange(gram.shape[1]) * hop).astype(int) / float(AUDIO_SAMPLE_RATE)
    gram[gram < thresh] = 0
    g = gram[:max_freq_idx, :]
    n_samples = int(times[-1] * SONIFY_FS) if len(times) else 0
    y = np.zeros(n_samples)
    if n_samples:
        t = np.arange(n_samples) / SONIFY_FS
        # nearest frame of every output sample (mir_eval interpolates the gram with kind="nearest")
        mid = 0.5 * (times[1:] + times[:-1])
        frame = np.searchsorted(mid, t, side="right")
        for k in np.flatnonzero(g.any(axis=1)):
            y += np.sin(2.0 * np.pi * freqs[k] * t) * g[k, frame]
        peak = np.abs(y).max()
        if peak > 0:
            y /= peak
    if save_path:
        from scipy.io import wavfile

        from .audio_io import resample

        wavfile.write(save_path, 44100, resample(y, SONIFY_FS, 44100))
    return y, SONIFY_FS


def get_pitch_bends(contours, note_events, n_bins_tolerance: int = 25, model=None):
    """reference: note_creation.py:182-219 -> [(start_frame, end_frame, pitch_midi, amplitude, [bends])].  Runs the
    decode's pitch-bend kernel (csrc/decode.cu: note_finish_kernel via `bp_pitch_bends_host`) on the given notes."""
    if n_bins_tolerance != 25:
        raise NotImplementedError("the device kernel implements the reference's default n_bins_tolerance = 25")
    from .inference import default_model

    mdl = model if model is not None else default_model()
    ev = list(note_events)
    off, bends = mdl.pitch_bends_arrays(contours, [e[0] for e in ev], [e[1] for e in ev], [e[2] for e in ev])
    return [(e[0], e[1], e[2], e[3], [int(x) for x in bends[off[i] : off[i + 1]]]) for i, e in enumerate(ev)]


def get_infered_onsets(onsets, frames, n_diff: int = 2, model=None):
    """reference: note_creation.py:289-311 -> float64 (T, 88).  Runs the decode's two cell-parallel kernels
    (csrc/decode.cu via `bp_infer_onsets_host`)."""
    if n_diff != 2:
        raise NotImplementedError("the device kernels implement the reference's default n_diff = 2")
    from .inference import default_model

    mdl = model if model is not None else default_model()
    return mdl.infer_onsets_array(onsets, frames)


__all__ = [
    "model_output_to_notes", "model_output_to_notes_grid", "grid_setting", "output_to_notes_polyphonic", "note_events_to_midi", "write_note_files", "sonify_batch",
    "note_events_batch",
    "NoteEventList", "LazyPrettyMIDI", "drop_overlapping_pitch_bends",
    "model_frames_to_time", "constrain_frequency", "midi_pitch_to_contour_bin", "sonify_midi", "sonify_salience",
    "get_pitch_bends", "get_infered_onsets", "SONIFY_FS",
    "MIDI_OFFSET", "MAX_FREQ_IDX", "N_FREQ_BINS_CONTOURS",
]  # fmt: skip
