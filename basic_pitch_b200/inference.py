"""Inference API — drop-in for reference: basic_pitch/inference.py, backed by libbp_b200.so.

Same public names, argument meaning, defaults, return types and error behaviour as the reference
module (`Model`, `predict`, `predict_and_save`, `run_inference`, `window_audio_file`,
`get_audio_input`, `unwrap_output`, `OutputExtensions`, `verify_*`, `build_output_path`,
`save_note_events`, `DEFAULT_*`).  What differs is what sits behind `Model`: instead of dispatching
to TensorFlow / CoreML / TFLite / onnxruntime (reference: inference.py:78-182) there is one runtime —
the hand-written sm_90a kernels in `csrc/` reached through the C ABI of include/bp_b200.h — and no
CPU fallback.  Batch entry points (`Model.transcribe_arrays`, `Model.transcribe_pcm`, `predict_batch`) are additions.
"""
from __future__ import annotations

import csv
import ctypes as C
import enum
import itertools
import json
import os
import pathlib
from typing import Any, Dict, Iterable, List, Mapping, Optional, Sequence, Tuple, Union

import numpy as np

from . import ICASSP_2022_MODEL_PATH, _lib, evaluate, weights
from . import note_creation as infer
from .audio_io import WavRegion, load_audio, load_audio_device, pcm_descriptors, pcm_sources, probe_wav, read_pcm
from .constants import (
    ANNOTATIONS_FPS,
    AUDIO_N_SAMPLES,
    AUDIO_SAMPLE_RATE,
    AUDIO_WINDOW_LENGTH,
    FFT_HOP,
    N_FREQ_BINS_CONTOURS,
    N_FREQ_BINS_NOTES,
)

DEFAULT_ONSET_THRESHOLD = 0.5
DEFAULT_FRAME_THRESHOLD = 0.3
DEFAULT_MINIMUM_NOTE_LENGTH_MS = 127.7
DEFAULT_MINIMUM_MIDI_TEMPO = 120
DEFAULT_SONIFICATION_SAMPLERATE = 44100
DEFAULT_OVERLAPPING_FRAMES = 30
DEFAULT_MIDI_VELOCITY_SCALE = 127

_F32 = np.float32


def _ptr(a: Optional[np.ndarray]) -> Optional[int]:
    return None if a is None else a.ctypes.data


def _cat_rows(xs: List[np.ndarray], w: int) -> np.ndarray:
    """Per-file (T, w) arrays -> one C-contiguous float32 (sum T, w) array."""
    cat = np.concatenate([np.asarray(x, _F32).reshape(-1, w) for x in xs]) if xs else np.zeros((0, w), _F32)
    return np.ascontiguousarray(cat, dtype=_F32)


class _PinnedBlock:
    """One page-locked host allocation (bp_host_alloc).  NumPy arrays carved out of it keep it alive through their
    `.base` chain; when the last of them dies the block goes back to the pool (or is freed)."""

    __slots__ = ("ptr", "nbytes", "pool")

    def __init__(self, ptr: int, nbytes: int, pool: "_PinnedPool"):
        self.ptr, self.nbytes, self.pool = ptr, nbytes, pool

    def __del__(self):
        pool, ptr = self.pool, self.ptr
        self.ptr = 0
        if ptr:
            try:
                pool._release(ptr, self.nbytes)
            except Exception:  # interpreter shutdown
                pass


class _PinnedPool:
    """Pool of page-locked output buffers: device->host copies into them are asynchronous (~50 GB/s instead of the
    ~10 GB/s of pageable memory) and `cudaHostAlloc` itself (~0.2 s per GB) is paid once, not per call."""

    GRANULE = 32 << 20
    KEEP = 3  # free blocks kept per size class

    def __init__(self, lib):
        self._lib = lib
        self._free: Dict[int, List[int]] = {}

    def array(self, shape: Tuple[int, ...], dtype=np.float32) -> np.ndarray:
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        cls = max(1, -(-n // self.GRANULE)) * self.GRANULE
        lst = self._free.get(cls)
        ptr = lst.pop() if lst else self._lib.bp_host_alloc(cls)
        if not ptr:
            raise MemoryError(f"cannot allocate {cls} bytes of page-locked host memory")
        carr = (C.c_byte * max(n, 1)).from_address(ptr)
        carr._block = _PinnedBlock(ptr, cls, self)  # lifetime: carr <- ndarray.base <- every view
        return np.frombuffer(carr, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def _release(self, ptr: int, cls: int) -> None:
        lst = self._free.setdefault(cls, [])
        if len(lst) < self.KEEP:
            lst.append(ptr)
        else:
            self._lib.bp_host_free(ptr)

    def __del__(self):
        for lst in self._free.values():
            for ptr in lst:
                try:
                    self._lib.bp_host_free(ptr)
                except Exception:
                    pass
        self._free = {}


def _default_device() -> int:
    for var in ("BP_B200_DEVICE", "LOCAL_RANK"):
        if os.environ.get(var, "") != "":
            return int(os.environ[var])
    return 0


class Model:
    """A loaded network bound to one H100 (reference: inference.py:71-182).

    `model_path` may be the packed blob shipped with this package (`ICASSP_2022_MODEL_PATH`) or an
    `.onnx` export of the same graph (e.g. the reference's `saved_models/icassp_2022/nmp.onnx`).
    Raises ValueError if the file is not a basic-pitch model (like the reference, inference.py:148-154)
    and `_lib.BpError` / ImportError if the CUDA library or an H100 is missing.
    """

    class MODEL_TYPES(enum.Enum):
        B200 = enum.auto()

    def __init__(self, model_path: Union[pathlib.Path, str], device: Optional[int] = None):
        self.model_type = Model.MODEL_TYPES.B200
        self.model_path = pathlib.Path(model_path)
        try:
            w = weights.load(self.model_path)
        except Exception as e:
            raise ValueError(
                f"File {model_path} cannot be loaded as a basic-pitch model (expected the packed .bpw blob or an "
                f"ONNX export of the ICASSP 2022 graph): {e!r}"
            )
        self._lib = _lib.load()
        blob = weights.pack(w)
        self._h = C.c_void_p()
        self.device = _default_device() if device is None else int(device)
        self._lib.bp_model_create(blob, len(blob), self.device, C.byref(self._h))
        self._pinned = _PinnedPool(self._lib)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and getattr(self, "_lib", None) is not None:
            try:
                self._lib.bp_model_destroy(h)
            except Exception:
                pass

    @property
    def handle(self) -> C.c_void_p:
        return self._h

    def set_path(self, path: int) -> None:
        """0 = FP32 FFMA kernels everywhere (on-device accuracy reference), 1 = tensor-core (wgmma) kernels with fused
        epilogues (default), 2 = tensor-core kernels keeping the 8-channel contour activations (for activation-level tests)."""
        self._lib.bp_model_set_path(self._h, int(path))

    @property
    def launch_count(self) -> int:
        return int(self._lib.bp_model_launch_count(self._h))

    # ------------------------------------------------------------------ stage 1+2
    def predict(self, x: np.ndarray) -> Dict[str, np.ndarray]:
        """(B, 43844, 1) or (B, 43844) float32 -> {"note","onset","contour"} (reference: inference.py:156-182)."""
        x = np.asarray(x)
        if x.ndim == 3 and x.shape[2] == 1:
            x = x[:, :, 0]
        if x.ndim != 2 or x.shape[1] != AUDIO_N_SAMPLES:
            raise ValueError(f"expected audio of shape (B, {AUDIO_N_SAMPLES}, 1), got {x.shape}")
        x = np.ascontiguousarray(x, dtype=_F32)
        n = x.shape[0]
        note = np.empty((n, 172, N_FREQ_BINS_NOTES), _F32)
        onset = np.empty((n, 172, N_FREQ_BINS_NOTES), _F32)
        contour = np.empty((n, 172, N_FREQ_BINS_CONTOURS), _F32)
        self._lib.bp_forward_host(self._h, _ptr(x), n, _ptr(note), _ptr(onset), _ptr(contour))
        return {"note": note, "onset": onset, "contour": contour}

    # ------------------------------------------------------------------ whole files
    @staticmethod
    def _pack_audio(audios: Sequence[np.ndarray]) -> Tuple[np.ndarray, np.ndarray]:
        offs = np.zeros(len(audios) + 1, dtype=np.int64)
        for i, a in enumerate(audios):
            if a.ndim != 1:
                raise ValueError("audio must be mono (1-D)")
            offs[i + 1] = offs[i] + a.shape[0]
        flat = np.empty(max(int(offs[-1]), 1), dtype=_F32)
        for i, a in enumerate(audios):
            flat[offs[i] : offs[i + 1]] = a
        return flat, offs

    def run_inference_arrays(self, audios: Sequence[np.ndarray]) -> List[Dict[str, np.ndarray]]:
        """Windowing + model + unwrap for a batch of mono 22 050 Hz signals (reference: inference.py:282-330)."""
        flat, offs = self._pack_audio(audios)
        n_files = len(audios)
        frames = [int(self._lib.bp_num_frames(int(offs[i + 1] - offs[i]))) for i in range(n_files)]
        total = sum(frames)
        note = np.empty((total, N_FREQ_BINS_NOTES), _F32)
        onset = np.empty((total, N_FREQ_BINS_NOTES), _F32)
        contour = np.empty((total, N_FREQ_BINS_CONTOURS), _F32)
        foff = np.zeros(n_files + 1, dtype=np.int64)
        self._lib.bp_run_inference_host(self._h, _ptr(flat), _ptr(offs), n_files, _ptr(note), _ptr(onset), _ptr(contour), _ptr(foff))
        return [
            {"note": note[foff[i] : foff[i + 1]], "onset": onset[foff[i] : foff[i + 1]], "contour": contour[foff[i] : foff[i + 1]]}
            for i in range(n_files)
        ]

    # ------------------------------------------------------------------ stage 3
    def _params(self, onset_thresh, frame_thresh, min_note_len, energy_tol, infer_onsets, melodia_trick,
                include_pitch_bends, min_pitch_idx, max_pitch_idx) -> _lib.DecodeParams:
        p = _lib.DecodeParams()
        p.onset_thresh, p.frame_thresh = float(onset_thresh), float(frame_thresh)
        p.min_note_len, p.energy_tol = int(min_note_len), int(energy_tol)
        p.infer_onsets, p.melodia_trick = int(bool(infer_onsets)), int(bool(melodia_trick))
        p.include_pitch_bends = int(bool(include_pitch_bends))
        p.min_pitch_idx, p.max_pitch_idx = int(min_pitch_idx), int(max_pitch_idx)
        return p

    @staticmethod
    def _alloc_notes(n_files: int, note_cap: int, bend_cap: int):
        arrs = {
            "note_off": np.zeros(n_files + 1, np.int32),
            "start": np.empty(note_cap, np.int32),
            "end": np.empty(note_cap, np.int32),
            "pitch": np.empty(note_cap, np.int32),
            "amp": np.empty(note_cap, _F32),
            "bend_off": np.zeros(note_cap + 1, np.int32),
            "bends": np.empty(max(bend_cap, 1), np.int32),
        }
        n = _lib.Notes()
        n.note_capacity, n.bend_capacity = note_cap, bend_cap
        n.note_off, n.start_frame, n.end_frame = _ptr(arrs["note_off"]), _ptr(arrs["start"]), _ptr(arrs["end"])
        n.pitch_midi, n.amplitude = _ptr(arrs["pitch"]), _ptr(arrs["amp"])
        n.bend_off, n.bends = _ptr(arrs["bend_off"]), _ptr(arrs["bends"])
        return n, arrs

    @staticmethod
    def _split_notes(arrs, n_files: int) -> List[Dict[str, np.ndarray]]:
        out = []
        noff, boff = arrs["note_off"], arrs["bend_off"]
        for i in range(n_files):
            a, b = int(noff[i]), int(noff[i + 1])
            b0 = int(boff[a])
            out.append({
                "start": arrs["start"][a:b].copy(), "end": arrs["end"][a:b].copy(), "pitch": arrs["pitch"][a:b].copy(),
                "amp": arrs["amp"][a:b].copy(), "bend_off": (boff[a : b + 1] - b0).copy(),
                "bends": arrs["bends"][b0 : int(boff[b])].copy(),
            })  # fmt: skip
        return out

    def _with_capacity(self, n_files: int, total_frames: int, call, n_params: int = 1):
        """call(notes) with capacities grown from bp_last_required; n_params: settings of a grid decode (the note offsets
        have n_params * n_files + 1 entries, the first guess scales with n_params)."""
        note_cap = max(4096, 2 * total_frames * n_params)
        bend_cap = max(65536, 24 * total_frames * n_params)
        for _ in range(3):  # at most: notes too small, then bends too small, then success
            notes, arrs = self._alloc_notes(n_files * n_params, note_cap, bend_cap)
            try:
                call(notes)
                return arrs
            except _lib.BpError as e:
                if e.code != _lib.BP_E_CAPACITY:
                    raise
                need_n, need_b = C.c_int64(0), C.c_int64(0)
                self._lib.bp_last_required(C.byref(need_n), C.byref(need_b))
                if need_n.value <= note_cap and need_b.value <= bend_cap:
                    raise
                note_cap, bend_cap = max(note_cap, need_n.value), max(bend_cap, need_b.value)
        raise RuntimeError("decode capacity negotiation failed")

    def decode_arrays(self, notes: Sequence[np.ndarray], onsets: Sequence[np.ndarray],
                      contours: Optional[Sequence[np.ndarray]], onset_thresh=0.5, frame_thresh=0.3, min_note_len=11,
                      energy_tol=11, infer_onsets=True, melodia_trick=True, include_pitch_bends=True,
                      min_pitch_idx=0, max_pitch_idx=88) -> List[Dict[str, np.ndarray]]:
        """Posteriorgrams of a batch of files -> note arrays per file (reference: note_creation.py:52-111)."""
        n_files = len(notes)
        foff, n_all, o_all, c_all = self._cat_posteriorgrams(notes, onsets, contours, include_pitch_bends)
        p = self._params(onset_thresh, frame_thresh, min_note_len, energy_tol, infer_onsets, melodia_trick,
                         include_pitch_bends, min_pitch_idx, max_pitch_idx)
        arrs = self._with_capacity(
            n_files, int(foff[-1]),
            lambda nt: self._lib.bp_decode_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(c_all), _ptr(foff), n_files, C.byref(p), C.byref(nt)),
        )
        return self._split_notes(arrs, n_files)

    def note_stream(self, onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, min_freq: Optional[float] = None,
                    max_freq: Optional[float] = None, melodia_trick=True, include_pitch_bends=True,
                    max_segment_frames: Optional[int] = None) -> "NoteStream":
        """A note decode for a recording whose posteriorgrams arrive piecewise (`bp_stream_*`, include/bp_b200.h): the
        stream cuts at quiet stretches and returns each stretch's notes as soon as the cut after it is known, holding
        only the frames since the last cut on the device.  Arguments as `note_creation.model_output_to_notes`
        (infer_onsets on, energy_tol 11); max_segment_frames > 0 also cuts when that many frames passed without a quiet
        cut, at the price of exactness there (DESIGN.md §4.5)."""
        lo, hi = infer.frequency_to_column_range(min_freq, max_freq)
        p = self._params(onset_thresh, frame_thresh, min_note_len, 11, True, melodia_trick, include_pitch_bends, lo, hi)
        return NoteStream(self, p, max_segment_frames)

    def stream_group(self, onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, min_freq: Optional[float] = None,
                     max_freq: Optional[float] = None, melodia_trick=True, include_pitch_bends=True,
                     max_segment_frames: Optional[int] = None) -> "StreamGroup":
        """Many streamed recordings with one set of note settings (`bp_stream_group_*`, include/bp_b200.h), each push
        served by one device pass over all of them; arguments as `note_stream`, whose notes every stream's equal."""
        lo, hi = infer.frequency_to_column_range(min_freq, max_freq)
        p = self._params(onset_thresh, frame_thresh, min_note_len, 11, True, melodia_trick, include_pitch_bends, lo, hi)
        return StreamGroup(self, p, max_segment_frames)

    @staticmethod
    def _cat_note_onset(notes, onsets):
        """Per-file note / onset posteriorgrams -> (frame offsets, note, onset) back to back."""
        n_files = len(notes)
        foff = np.zeros(n_files + 1, np.int64)
        for i, a in enumerate(notes):
            if a.shape[1:] != (N_FREQ_BINS_NOTES,) or onsets[i].shape != a.shape:
                raise ValueError("note/onset posteriorgrams must be (T, 88) and of equal shape")
            foff[i + 1] = foff[i] + a.shape[0]
        return foff, _cat_rows(list(notes), N_FREQ_BINS_NOTES), _cat_rows(list(onsets), N_FREQ_BINS_NOTES)

    @staticmethod
    def _cat_posteriorgrams(notes, onsets, contours, need_contours: bool):
        """Per-file posteriorgrams -> (frame offsets, note, onset, contour) back to back, as the decode entry points
        take them."""
        foff, n_all, o_all = Model._cat_note_onset(notes, onsets)
        total = int(foff[-1])
        if contours is None:
            if need_contours:
                raise ValueError("pitch bends need the contour posteriorgram")
            c_all = np.zeros((max(total, 1), N_FREQ_BINS_CONTOURS), _F32)
        else:
            c_all = _cat_rows(list(contours), N_FREQ_BINS_CONTOURS)
            if c_all.shape[0] != total:
                raise ValueError("contour posteriorgrams must have as many frames as note posteriorgrams")
        return foff, n_all, o_all, c_all

    _DECODE_DEFAULTS = dict(onset_thresh=0.5, frame_thresh=0.3, min_note_len=11, energy_tol=11, infer_onsets=True,
                            melodia_trick=True, include_pitch_bends=True, min_pitch_idx=0, max_pitch_idx=88)

    def decode_grid(self, notes: Sequence[np.ndarray], onsets: Sequence[np.ndarray],
                    contours: Optional[Sequence[np.ndarray]], settings: Sequence[Dict[str, Any]],
                    split_notes: bool = True):
        """Posteriorgrams of a batch of files decoded under every setting of a grid in ONE library call
        (`bp_decode_grid_host`: the posteriorgrams go up once, settings sharing a pitch range share the per-cell work,
        the greedy loops of all (setting, file) pairs run in parallel).  A setting is a dict of `decode_arrays`' keyword
        arguments (missing ones take its defaults).  Returns [setting][file] note-array dicts, each what `decode_arrays`
        gives for that setting; with split_notes=False the concatenated arrays of the call instead (note_off has
        len(settings) * n_files + 1 entries, setting-major)."""
        n_files, n_params = len(notes), len(settings)
        ps = self._grid_params(settings)
        need_contours = any(bool(p.include_pitch_bends) for p in ps[:n_params])
        foff, n_all, o_all, c_all = self._cat_posteriorgrams(notes, onsets, contours, need_contours)
        arrs = self._with_capacity(
            n_files, int(foff[-1]),
            lambda nt: self._lib.bp_decode_grid_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(c_all), _ptr(foff), n_files,
                                                     ps, n_params, C.byref(nt)),
            n_params=n_params,
        )
        if not split_notes:
            return arrs
        flat = self._split_notes(arrs, n_params * n_files)
        return [flat[k * n_files : (k + 1) * n_files] for k in range(n_params)]

    def _grid_params(self, settings: Sequence[Dict[str, Any]]):
        ps = (_lib.DecodeParams * max(len(settings), 1))()
        for k, s in enumerate(settings):
            unknown = set(s) - set(self._DECODE_DEFAULTS)
            if unknown:
                raise TypeError(f"settings[{k}]: unknown decode argument(s) {sorted(unknown)}")
            ps[k] = self._params(**{**self._DECODE_DEFAULTS, **s})
        return ps

    # ------------------------------------------------------------------ note-level scores
    @staticmethod
    def _score_params(tolerances: Dict[str, float]) -> _lib.ScoreParams:
        unknown = set(tolerances) - set(evaluate.TOLERANCES)
        if unknown:
            raise TypeError(f"unknown tolerance(s) {sorted(unknown)}")
        return _lib.ScoreParams(**{k: float(v) for k, v in {**evaluate.TOLERANCES, **tolerances}.items()})

    @staticmethod
    def _note_set(sets: Sequence, what: str, pitched: bool = True):
        """[(intervals (n, 2) in seconds, pitches (n,) in Hz)], or without `pitched` [intervals (n, 2)] ->
        (bp_note_set_t, the arrays it points at); log2 of the pitches as np.log2 takes it (a pitch <= 0 gives a
        non-finite log2, which the library rejects)."""
        off = np.zeros(len(sets) + 1, np.int64)
        ivs, hzs = [], []
        for i, s in enumerate(sets):
            iv, hz = s if pitched else (s, None)
            iv = np.asarray(iv, np.float64)
            if iv.size == 0:
                iv = iv.reshape(0, 2)
            if pitched:
                hz = np.asarray(hz, np.float64).reshape(-1)
                if iv.ndim != 2 or iv.shape[1] != 2 or len(hz) != len(iv):
                    raise ValueError(f"{what}[{i}]: need intervals (n, 2) and pitches (n,), got {iv.shape} and {hz.shape}")
                hzs.append(hz)
            elif iv.ndim != 2 or iv.shape[1] != 2:
                raise ValueError(f"{what}[{i}]: need intervals (n, 2), got {iv.shape}")
            off[i + 1] = off[i] + len(iv)
            ivs.append(iv)
        iv = np.concatenate(ivs) if ivs else np.zeros((0, 2))
        arrs = (off, np.ascontiguousarray(iv[:, 0]), np.ascontiguousarray(iv[:, 1]))
        if pitched:
            with np.errstate(divide="ignore", invalid="ignore"):
                arrs += (np.log2(np.concatenate(hzs) if hzs else np.zeros(0)),)
        ns = _lib.NoteSet(*(_ptr(a) for a in arrs))
        return ns, arrs

    @staticmethod
    def _interval_set(sets: Sequence[np.ndarray], what: str):
        """[intervals (n, 2) in seconds] -> (bp_note_set_t without pitches, the arrays it points at)."""
        return Model._note_set(sets, what, pitched=False)

    def score_grid(self, notes: Sequence[np.ndarray], onsets: Sequence[np.ndarray], settings: Sequence[Dict[str, Any]],
                   references: Sequence[Tuple[np.ndarray, np.ndarray]], **tolerances) -> np.ndarray:
        """Note-level match counts of a batch of files decoded under every setting of a grid, scored against one
        reference set per file, in ONE library call (`bp_score_grid_host`): the notes never leave the device.
        A setting is a dict of `decode_arrays`' keyword arguments (include_pitch_bends is ignored); a reference set is
        (intervals (n, 2) in seconds, pitches (n,) in Hz), mir_eval's convention; tolerances are those of
        `evaluate.TOLERANCES`.  Returns int64 counts (n_settings, n_files, 4): n_ref, n_est, matched without offsets,
        matched (`evaluate.note_scores` turns them into precision, recall and F)."""
        n_files, n_params = len(notes), len(settings)
        if len(references) != n_files:
            raise ValueError(f"{n_files} files but {len(references)} reference sets")
        ps = self._grid_params(settings)
        sp = self._score_params(tolerances)
        refs, keep = self._note_set(references, "references")
        foff, n_all, o_all = self._cat_note_onset(notes, onsets)
        counts = np.zeros((n_params, n_files, 4), np.int64)
        self._lib.bp_score_grid_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(foff), n_files, ps, n_params, C.byref(refs),
                                     C.byref(sp), _ptr(evaluate.EST_LOG2_HZ), _ptr(counts))
        return counts

    def score_notes(self, estimates: Sequence[Tuple[np.ndarray, np.ndarray]],
                    references: Sequence[Tuple[np.ndarray, np.ndarray]], **tolerances) -> np.ndarray:
        """Item i's estimated notes against item i's reference notes (`bp_score_notes_host`, one kernel launch), both
        as (intervals (n, 2) in seconds, pitches (n,) in Hz).  Returns int64 counts (n_items, 4) as `score_grid`."""
        if len(estimates) != len(references):
            raise ValueError(f"{len(estimates)} estimated but {len(references)} reference sets")
        sp = self._score_params(tolerances)
        est, keep_e = self._note_set(estimates, "estimates")
        refs, keep_r = self._note_set(references, "references")
        counts = np.zeros((len(estimates), 4), np.int64)
        self._lib.bp_score_notes_host(self._h, C.byref(est), C.byref(refs), len(estimates), C.byref(sp), _ptr(counts))
        return counts

    def match_grid(self, notes: Sequence[np.ndarray], onsets: Sequence[np.ndarray], settings: Sequence[Dict[str, Any]],
                   references: Sequence[Tuple[np.ndarray, np.ndarray]], **tolerances):
        """mir_eval 0.7's note matching, pair for pair, of a batch of files decoded under every setting of a grid, in ONE
        library call (`bp_match_grid_host`).  Arguments as `score_grid` (include_pitch_bends is ignored).

        Returns (res, match): res[setting][file] the note arrays `decode_grid` gives for that setting (amplitudes, no
        pitch bends); match[setting][file] int32 (2, n_ref): per reference note, in the caller's order, the index of the
        estimated note in res[setting][file] it is matched to, or -1; row 0 without, row 1 with the offset test.
        mir_eval's matching depends on the order of the estimate list: here it is the decode's order; `match_notes`
        takes another.  `evaluate.matching_scores` turns a file's matchings into its overlap and velocity scores."""
        n_files, n_params = len(notes), len(settings)
        if len(references) != n_files:
            raise ValueError(f"{n_files} files but {len(references)} reference sets")
        ps = self._grid_params(settings)
        sp = self._score_params(tolerances)
        refs, keep = self._note_set(references, "references")
        foff, n_all, o_all = self._cat_note_onset(notes, onsets)
        roff = keep[0]
        h_match = np.full((max(n_params, 1), 2, max(int(roff[-1]), 1)), -1, np.int32)
        arrs = self._with_capacity(
            n_files, int(foff[-1]),
            lambda nt: self._lib.bp_match_grid_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(foff), n_files, ps, n_params,
                                                    C.byref(refs), C.byref(sp), _ptr(evaluate.EST_LOG2_HZ), C.byref(nt),
                                                    _ptr(h_match)),
            n_params=n_params,
        )
        flat = self._split_notes(arrs, n_params * n_files)
        res = [flat[k * n_files : (k + 1) * n_files] for k in range(n_params)]
        match = [[h_match[k, :, roff[i] : roff[i + 1]].copy() for i in range(n_files)] for k in range(n_params)]
        return res, match

    def match_notes(self, estimates: Sequence[Tuple[np.ndarray, np.ndarray]],
                    references: Sequence[Tuple[np.ndarray, np.ndarray]], **tolerances) -> List[np.ndarray]:
        """mir_eval 0.7's note matching of item i's estimated notes, in the order given, against item i's reference
        notes (`bp_match_notes_host`), both as (intervals (n, 2) in seconds, pitches (n,) in Hz).  Returns per item an
        int32 (2, n_ref) array as `match_grid`."""
        if len(estimates) != len(references):
            raise ValueError(f"{len(estimates)} estimated but {len(references)} reference sets")
        sp = self._score_params(tolerances)
        est, keep_e = self._note_set(estimates, "estimates")
        refs, keep_r = self._note_set(references, "references")
        roff = keep_r[0]
        h_match = np.full((2, max(int(roff[-1]), 1)), -1, np.int32)
        self._lib.bp_match_notes_host(self._h, C.byref(est), C.byref(refs), len(estimates), C.byref(sp), _ptr(h_match))
        return [h_match[:, roff[i] : roff[i + 1]].copy() for i in range(len(estimates))]

    def score_onset_offset_grid(self, notes: Sequence[np.ndarray], onsets: Sequence[np.ndarray],
                                settings: Sequence[Dict[str, Any]], references: Sequence[np.ndarray],
                                **tolerances) -> np.ndarray:
        """Onset-only and offset-only match counts (mir_eval.transcription's match_note_onsets / match_note_offsets;
        pitch plays no part) of a batch of files decoded under every setting of a grid, in ONE library call
        (`bp_score_onset_offset_grid_host`): the notes never leave the device.  Settings as `score_grid`;
        `references[i]` is file i's intervals (n, 2) in seconds; tolerances those of `evaluate.TOLERANCES`
        (pitch_tolerance is checked and unused).  Returns int64 counts (n_settings, n_files, 4): n_ref, n_est, onsets
        matched, offsets matched (`evaluate.onset_offset_scores` turns them into precision, recall and F)."""
        n_files, n_params = len(notes), len(settings)
        if len(references) != n_files:
            raise ValueError(f"{n_files} files but {len(references)} reference sets")
        ps = self._grid_params(settings)
        sp = self._score_params(tolerances)
        refs, keep = self._interval_set(references, "references")
        foff, n_all, o_all = self._cat_note_onset(notes, onsets)
        counts = np.zeros((n_params, n_files, 4), np.int64)
        self._lib.bp_score_onset_offset_grid_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(foff), n_files, ps, n_params,
                                                  C.byref(refs), C.byref(sp), None, _ptr(counts))
        return counts

    def score_onsets_offsets(self, estimates: Sequence[np.ndarray], references: Sequence[np.ndarray],
                             **tolerances) -> np.ndarray:
        """Item i's estimated intervals against item i's reference intervals, (n, 2) in seconds
        (`bp_score_onset_offset_notes_host`, one kernel launch).  Returns int64 counts (n_items, 4) as
        `score_onset_offset_grid`."""
        if len(estimates) != len(references):
            raise ValueError(f"{len(estimates)} estimated but {len(references)} reference sets")
        sp = self._score_params(tolerances)
        est, keep_e = self._interval_set(estimates, "estimates")
        refs, keep_r = self._interval_set(references, "references")
        counts = np.zeros((len(estimates), 4), np.int64)
        self._lib.bp_score_onset_offset_notes_host(self._h, C.byref(est), C.byref(refs), len(estimates), C.byref(sp),
                                                   _ptr(counts))
        return counts

    # ------------------------------------------------------------------ frame-level scores
    @staticmethod
    def _multipitch_set(series: Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]], what: str):
        """[(times (n,) in seconds, [Hz array per frame])] (mir_eval.multipitch's convention) -> (bp_multipitch_set_t,
        the arrays it points at), values as `evaluate.multipitch_values` gives them."""
        f_off = np.zeros(len(series) + 1, np.int64)
        times, counts, hzs = [], [], []
        for i, (t, freqs) in enumerate(series):
            t = np.asarray(t, np.float64).reshape(-1)
            if len(t) != len(freqs):
                raise ValueError(f"{what}[{i}]: {len(t)} times but {len(freqs)} frames of frequencies")
            f_off[i + 1] = f_off[i] + len(t)
            times.append(t)
            for fr in freqs:
                fr = np.asarray(fr, np.float64).reshape(-1)
                counts.append(len(fr))
                hzs.append(fr)
        v_off = np.zeros(len(counts) + 1, np.int64)
        np.cumsum(counts, out=v_off[1:])
        midi, chroma = evaluate.multipitch_values(np.concatenate(hzs) if hzs else np.zeros(0))
        arrs = (f_off, np.ascontiguousarray(np.concatenate(times) if times else np.zeros(0)), v_off,
                np.ascontiguousarray(midi), np.ascontiguousarray(chroma))
        ms = _lib.MultipitchSet()
        ms.frame_off, ms.time_s, ms.value_off, ms.midi, ms.chroma = (_ptr(a) for a in arrs)
        return ms, arrs

    def score_frames_grid(self, notes: Sequence[np.ndarray], onsets: Sequence[np.ndarray],
                          settings: Sequence[Dict[str, Any]], references: Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]],
                          window: float = evaluate.WINDOW, contours: Optional[Sequence[np.ndarray]] = None) -> np.ndarray:
        """Frame-level multi-pitch counts of a batch of files decoded under every setting of a grid, scored against one
        reference series per file, in ONE library call: the notes never leave the device.  A setting is a dict of
        `decode_arrays`' keyword arguments; a reference is (times (n,) in seconds, [Hz array per frame]), mir_eval's
        convention; window in semitones.  Without contours (`bp_score_frames_grid_host`) include_pitch_bends is ignored
        and the estimate of (setting, file) is the piano roll of its notes at the model frame times.  With the files'
        contour posteriorgrams (`bp_score_bent_frames_grid_host`) each setting's include_pitch_bends (default True)
        applies: the estimate is `evaluate.note_frames_to_multipitch` of its notes and bends, what `predict` returns.
        Returns int64 counts (n_settings, n_files, 7) in the order of `evaluate.FRAME_FIELDS` (`evaluate.frame_scores`
        turns them into mir_eval.multipitch's metrics)."""
        n_files, n_params = len(notes), len(settings)
        if len(references) != n_files:
            raise ValueError(f"{n_files} files but {len(references)} reference series")
        ps = self._grid_params(settings)
        refs, keep = self._multipitch_set(references, "references")
        counts = np.zeros((n_params, n_files, 7), np.int64)
        if contours is None:
            foff, n_all, o_all = self._cat_note_onset(notes, onsets)
            self._lib.bp_score_frames_grid_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(foff), n_files, ps, n_params,
                                                C.byref(refs), float(window), _ptr(evaluate.EST_MIDI),
                                                _ptr(evaluate.EST_CHROMA), _ptr(counts))
            return counts
        foff, n_all, o_all, c_all = self._cat_posteriorgrams(notes, onsets, contours, True)
        _, midi, chroma, _ = evaluate.bent_bins()
        self._lib.bp_score_bent_frames_grid_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(c_all), _ptr(foff), n_files, ps,
                                                 n_params, C.byref(refs), float(window), _ptr(midi), _ptr(chroma),
                                                 _ptr(counts))
        return counts

    def score_multipitch(self, estimates: Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]],
                         references: Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]],
                         window: float = evaluate.WINDOW) -> np.ndarray:
        """Item i's estimate series against item i's reference series (`bp_score_multipitch_host`, one kernel launch),
        both as (times (n,) in seconds, [Hz array per frame]): mir_eval.multipitch.metrics for arbitrary series, for
        example `evaluate.notes_to_multipitch` of another system's notes.  Returns int64 counts (n_items, 7) as
        `score_frames_grid`."""
        if len(estimates) != len(references):
            raise ValueError(f"{len(estimates)} estimate but {len(references)} reference series")
        est, keep_e = self._multipitch_set(estimates, "estimates")
        refs, keep_r = self._multipitch_set(references, "references")
        counts = np.zeros((len(estimates), 7), np.int64)
        self._lib.bp_score_multipitch_host(self._h, C.byref(est), C.byref(refs), len(estimates), float(window),
                                           _ptr(counts))
        return counts

    _SALIENCE_KEYS = ("threshold", "peak_picking", "minimum_frequency", "maximum_frequency")

    @staticmethod
    def _salience_params(settings: Sequence[Dict[str, Any]], kind: str):
        """Settings {threshold, peak_picking (default True), minimum_frequency, maximum_frequency (default None)} ->
        bp_salience_params_t array, the range in bins as `evaluate.salience_bin_range` gives it."""
        ps = (_lib.SalienceParams * max(len(settings), 1))()
        for k, s in enumerate(settings):
            unknown = set(s) - set(Model._SALIENCE_KEYS)
            if unknown:
                raise TypeError(f"settings[{k}]: unknown salience argument(s) {sorted(unknown)}")
            if "threshold" not in s:
                raise TypeError(f"settings[{k}]: a threshold is required")
            lo, hi = evaluate.salience_bin_range(kind, s.get("minimum_frequency"), s.get("maximum_frequency"))
            ps[k] = _lib.SalienceParams(float(s["threshold"]), int(bool(s.get("peak_picking", True))), lo, hi, 0)
        return ps

    def score_salience_grid(self, grams: Sequence[np.ndarray], settings: Sequence[Dict[str, Any]],
                            references: Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]], kind: str = "contour",
                            window: float = evaluate.WINDOW) -> np.ndarray:
        """Frame-level multi-pitch counts of a batch of posteriorgrams read as multi-f0 estimates under every setting of
        a grid, scored against one reference series per file, in ONE library call (`bp_score_salience_grid_host`: the
        posteriorgrams go up once, no estimate is built on the host).  grams[i] is file i's (T, 264) contour or (T, 88)
        note posteriorgram (`kind`); a setting is a dict {threshold, peak_picking=True, minimum_frequency=None,
        maximum_frequency=None} and its estimate is `evaluate.salience_to_multipitch` of the posteriorgram under it; a
        reference is (times (n,) in seconds, [Hz array per frame]); window in semitones.  Returns int64 counts
        (n_settings, n_files, 7) in the order of `evaluate.FRAME_FIELDS`."""
        hz, midi, chroma = evaluate.salience_bins(kind)
        n_files, n_params, width = len(grams), len(settings), len(hz)
        if len(references) != n_files:
            raise ValueError(f"{n_files} files but {len(references)} reference series")
        foff = np.zeros(n_files + 1, np.int64)
        for i, g in enumerate(grams):
            if np.ndim(g) != 2 or np.shape(g)[1] != width:
                raise ValueError(f"grams[{i}]: a {kind} posteriorgram must be (T, {width}), got {np.shape(g)}")
            foff[i + 1] = foff[i] + np.shape(g)[0]
        ps = self._salience_params(settings, kind)
        refs, keep = self._multipitch_set(references, "references")
        g_all = _cat_rows(list(grams), width)
        counts = np.zeros((n_params, n_files, 7), np.int64)
        self._lib.bp_score_salience_grid_host(self._h, _ptr(g_all), width, _ptr(foff), n_files, ps, n_params,
                                              C.byref(refs), float(window), _ptr(midi), _ptr(chroma), _ptr(counts))
        return counts

    # ------------------------------------------------------------------ melody scores
    @staticmethod
    def _melody_set(series: Sequence[Tuple[np.ndarray, np.ndarray]], what: str):
        """[(times (n,) in seconds, f0 (n,) in Hz)] (mir_eval.melody's convention: 0 or a negative f0 is unvoiced) ->
        (bp_melody_set_t, the arrays it points at), values as `evaluate.melody_values` gives them."""
        f_off = np.zeros(len(series) + 1, np.int64)
        times, hzs = [], []
        for i, (t, hz) in enumerate(series):
            t = np.asarray(t, np.float64).reshape(-1)
            hz = np.asarray(hz, np.float64).reshape(-1)
            if len(t) != len(hz):
                raise ValueError(f"{what}[{i}]: {len(t)} times but {len(hz)} frequencies")
            f_off[i + 1] = f_off[i] + len(t)
            times.append(t)
            hzs.append(hz)
        cents, voiced = evaluate.melody_values(np.concatenate(hzs) if hzs else np.zeros(0))
        arrs = (f_off, np.ascontiguousarray(np.concatenate(times) if times else np.zeros(0)), cents, voiced)
        ms = _lib.MelodySet()
        ms.frame_off, ms.time_s, ms.cent, ms.voiced = (_ptr(a) for a in arrs)
        return ms, arrs

    _MELODY_KEYS = ("threshold", "minimum_frequency", "maximum_frequency", "guess_unvoiced")

    @staticmethod
    def _melody_params(settings: Sequence[Dict[str, Any]], kind: str):
        """Settings {threshold, minimum_frequency, maximum_frequency (default None), guess_unvoiced (default True)} ->
        bp_melody_params_t array, the range in bins as `evaluate.salience_bin_range` gives it."""
        ps = (_lib.MelodyParams * max(len(settings), 1))()
        for k, s in enumerate(settings):
            unknown = set(s) - set(Model._MELODY_KEYS)
            if unknown:
                raise TypeError(f"settings[{k}]: unknown melody argument(s) {sorted(unknown)}")
            if "threshold" not in s:
                raise TypeError(f"settings[{k}]: a threshold is required")
            lo, hi = evaluate.salience_bin_range(kind, s.get("minimum_frequency"), s.get("maximum_frequency"))
            ps[k] = _lib.MelodyParams(float(s["threshold"]), lo, hi, int(bool(s.get("guess_unvoiced", True))), 0)
        return ps

    def score_melody_grid(self, grams: Sequence[np.ndarray], settings: Sequence[Dict[str, Any]],
                          references: Sequence[Tuple[np.ndarray, np.ndarray]], kind: str = "contour",
                          cent_tolerance: float = evaluate.CENT_TOLERANCE) -> np.ndarray:
        """Melody counts of a batch of posteriorgrams read as single-f0 estimates under every setting of a grid, scored
        against one reference f0 track per file, in ONE library call (`bp_score_melody_grid_host`: the posteriorgrams
        go up once, no estimate is built on the host).  grams[i] is file i's (T, 264) contour or (T, 88) note
        posteriorgram (`kind`); a setting is a dict {threshold, minimum_frequency=None, maximum_frequency=None,
        guess_unvoiced=True} and its estimate is `evaluate.salience_to_melody` of the posteriorgram under it; a
        reference is (times (n,) in seconds, f0 (n,) in Hz), mir_eval.melody's convention.  Returns int64 counts
        (n_settings, n_files, 7) in the order of `evaluate.MELODY_FIELDS` (`evaluate.melody_scores` turns them into
        mir_eval.melody.evaluate's scores)."""
        hz, cents = evaluate.melody_bins(kind)
        n_files, n_params, width = len(grams), len(settings), len(hz)
        if len(references) != n_files:
            raise ValueError(f"{n_files} files but {len(references)} reference tracks")
        foff = np.zeros(n_files + 1, np.int64)
        for i, g in enumerate(grams):
            if np.ndim(g) != 2 or np.shape(g)[1] != width:
                raise ValueError(f"grams[{i}]: a {kind} posteriorgram must be (T, {width}), got {np.shape(g)}")
            foff[i + 1] = foff[i] + np.shape(g)[0]
        ps = self._melody_params(settings, kind)
        refs, keep = self._melody_set(references, "references")
        g_all = _cat_rows(list(grams), width)
        counts = np.zeros((n_params, n_files, 7), np.int64)
        self._lib.bp_score_melody_grid_host(self._h, _ptr(g_all), width, _ptr(foff), n_files, ps, n_params,
                                            C.byref(refs), float(cent_tolerance), _ptr(cents), _ptr(counts))
        return counts

    def score_note_melody_grid(self, notes: Sequence[np.ndarray], onsets: Sequence[np.ndarray],
                               contours: Optional[Sequence[np.ndarray]], settings: Sequence[Dict[str, Any]],
                               references: Sequence[Tuple[np.ndarray, np.ndarray]],
                               cent_tolerance: float = evaluate.CENT_TOLERANCE) -> np.ndarray:
        """Melody counts of a batch of files decoded under every setting of a grid, each (setting, file)'s notes with
        their pitch bends read as a single-f0 track (`evaluate.note_frames_to_melody`) and scored against one reference
        f0 track per file, in ONE library call (`bp_score_note_melody_grid_host`): the notes never leave the device.  A
        setting is a dict of `decode_arrays`' keyword arguments, whose include_pitch_bends (default True) applies;
        contours may be None only when no setting has bends; a reference is (times (n,) in seconds, f0 (n,) in Hz),
        mir_eval.melody's convention.  Returns int64 counts (n_settings, n_files, 7) in the order of
        `evaluate.MELODY_FIELDS` (`evaluate.melody_scores` turns them into mir_eval.melody.evaluate's scores)."""
        n_files, n_params = len(notes), len(settings)
        if len(references) != n_files:
            raise ValueError(f"{n_files} files but {len(references)} reference tracks")
        ps = self._grid_params(settings)
        need_contours = any(bool(p.include_pitch_bends) for p in ps[:n_params])
        refs, keep = self._melody_set(references, "references")
        foff, n_all, o_all, c_all = self._cat_posteriorgrams(notes, onsets, contours, need_contours)
        cents = evaluate.bent_bins()[3]
        counts = np.zeros((n_params, n_files, 7), np.int64)
        self._lib.bp_score_note_melody_grid_host(self._h, _ptr(n_all), _ptr(o_all), None if contours is None else _ptr(c_all),
                                                 _ptr(foff), n_files, ps, n_params, C.byref(refs),
                                                 float(cent_tolerance), _ptr(cents), _ptr(counts))
        return counts

    def score_melody(self, estimates: Sequence[Tuple[np.ndarray, np.ndarray]],
                     references: Sequence[Tuple[np.ndarray, np.ndarray]],
                     cent_tolerance: float = evaluate.CENT_TOLERANCE) -> np.ndarray:
        """Item i's estimated f0 track against item i's reference track (`bp_score_melody_host`, one kernel launch),
        both as (times (n,) in seconds, f0 (n,) in Hz): mir_eval.melody.evaluate for arbitrary tracks, for example
        another system's output.  Estimate times must be strictly increasing (after rounding to 1e-10 s).  Returns int64
        counts (n_items, 7) as `score_melody_grid`."""
        if len(estimates) != len(references):
            raise ValueError(f"{len(estimates)} estimate but {len(references)} reference tracks")
        est, keep_e = self._melody_set(estimates, "estimates")
        refs, keep_r = self._melody_set(references, "references")
        counts = np.zeros((len(estimates), 7), np.int64)
        self._lib.bp_score_melody_host(self._h, C.byref(est), C.byref(refs), len(estimates), float(cent_tolerance),
                                       _ptr(counts))
        return counts

    # ------------------------------------------------------------------ every family in one pass
    EVAL_FAMILIES = ("notes", "onset_offset", "pairs", "frames", "bent_frames", "note_melody", "flat_note_melody",
                     "salience", "melody")

    def _eval_request(self, n_files: int, families: Sequence[str], settings: Sequence[Dict[str, Any]] = (),
                      note_refs=None, multipitch_refs=None, f0_refs=None, salience: Optional[Dict[str, Any]] = None,
                      melody: Optional[Dict[str, Any]] = None, window: float = evaluate.WINDOW,
                      cent_tolerance: float = evaluate.CENT_TOLERANCE, **tolerances):
        """The bp_eval_request_t of `evaluate` -> (request, the arrays it points at, {family: counts array}); the pairs'
        notes (`pair_notes`) are set per attempt by the caller.  Inputs as the standalone `score_*` / `match_grid`
        calls take them; salience / melody are dicts {settings, references, kind="contour"}."""
        unknown = set(families) - set(self.EVAL_FAMILIES)
        if unknown:
            raise ValueError(f"unknown famil(ies) {sorted(unknown)}; choose from {self.EVAL_FAMILIES}")
        r, keep, out = _lib.EvalRequest(), [], {}
        n_params = len(settings)

        def need(refs, what):
            if refs is None:
                raise ValueError(f"{what} references are required")
            if len(refs) != n_files:
                raise ValueError(f"{n_files} files but {len(refs)} {what} references")

        def counts(name, n, width):
            out[name] = np.zeros((n, n_files, width), np.int64)
            return _ptr(out[name])

        if {"notes", "onset_offset", "pairs", "frames", "bent_frames", "note_melody", "flat_note_melody"} & set(families):
            ps = self._grid_params(settings)
            r.params, r.n_params = C.addressof(ps), n_params
            keep.append(ps)
        if {"notes", "onset_offset", "pairs"} & set(families):
            need(note_refs, "note")
            sp = self._score_params(tolerances)
            pitched = [(ref[0], ref[1]) for ref in note_refs]
            ns, arrs = self._note_set(pitched, "references")
            keep += [sp, ns, arrs]
            r.note_refs, r.score, r.est_log2_hz = C.addressof(ns), C.addressof(sp), _ptr(evaluate.EST_LOG2_HZ)
            if "notes" in families:
                r.notes_counts = counts("notes", n_params, 4)
            if "onset_offset" in families:
                r.onset_offset_counts = counts("onset_offset", n_params, 4)
            if "pairs" in families:
                roff = arrs[0]
                h_match = np.full((max(n_params, 1), 2, max(int(roff[-1]), 1)), -1, np.int32)
                out["pairs"] = (h_match, roff)
                r.pair_match = _ptr(h_match)
        elif tolerances:
            self._score_params(tolerances)
        if {"frames", "bent_frames"} & set(families):
            need(multipitch_refs, "multi-pitch")
            ms, arrs = self._multipitch_set(multipitch_refs, "references")
            keep += [ms, arrs]
            r.mp_refs, r.window = C.addressof(ms), float(window)
            if "frames" in families:
                r.est_midi, r.est_chroma = _ptr(evaluate.EST_MIDI), _ptr(evaluate.EST_CHROMA)
                r.frames_counts = counts("frames", n_params, 7)
            if "bent_frames" in families:
                _, midi, chroma, _ = evaluate.bent_bins()
                keep += [midi, chroma]
                r.bin_midi, r.bin_chroma = _ptr(midi), _ptr(chroma)
                r.bent_frames_counts = counts("bent_frames", n_params, 7)
        if {"note_melody", "flat_note_melody"} & set(families):
            need(f0_refs, "f0")
            ms, arrs = self._melody_set(f0_refs, "references")
            cents = evaluate.bent_bins()[3]
            keep += [ms, arrs, cents]
            r.f0_refs, r.cent_tolerance, r.bin_cent = C.addressof(ms), float(cent_tolerance), _ptr(cents)
            if "note_melody" in families:
                r.note_melody_counts = counts("note_melody", n_params, 7)
            if "flat_note_melody" in families:
                r.flat_note_melody_counts = counts("flat_note_melody", n_params, 7)
        for name, spec in (("salience", salience), ("melody", melody)):
            if name not in families:
                continue
            if spec is None or "settings" not in spec:
                raise ValueError(f"{name} needs a dict with its settings and references")
            kind = spec.get("kind", "contour")
            if kind not in ("contour", "note"):
                raise ValueError(f"{name}: kind must be 'contour' or 'note', got {kind!r}")
            need(spec.get("references"), name)
            sets = spec["settings"]
            if name == "salience":
                ps = self._salience_params(sets, kind)
                ms, arrs = self._multipitch_set(spec["references"], "references")
                _, midi, chroma = evaluate.salience_bins(kind)
                keep += [ps, ms, arrs, midi, chroma]
                r.salience_params, r.n_salience, r.salience_gram = C.addressof(ps), len(sets), int(kind == "note")
                r.salience_refs, r.salience_window = C.addressof(ms), float(window)
                r.salience_midi, r.salience_chroma = _ptr(midi), _ptr(chroma)
                r.salience_counts = counts("salience", len(sets), 7)
            else:
                ps = self._melody_params(sets, kind)
                ms, arrs = self._melody_set(spec["references"], "references")
                cents = evaluate.melody_bins(kind)[1]
                keep += [ps, ms, arrs, cents]
                r.melody_params, r.n_melody, r.melody_gram = C.addressof(ps), len(sets), int(kind == "note")
                r.melody_refs, r.melody_tolerance, r.melody_cent = C.addressof(ms), float(cent_tolerance), _ptr(cents)
                r.melody_counts = counts("melody", len(sets), 7)
        return r, keep, out

    def evaluate(self, families: Sequence[str], settings: Sequence[Dict[str, Any]] = (), *, grams=None, audio=None,
                 pcm=None, return_model_output: bool = False, stream: int = 0, **request) -> Dict[str, Any]:
        """Every requested metric family of a batch in ONE library call (`bp_evaluate_*`): the batch is decoded once per
        chunk of settings and every note-derived family scores that decode; the posteriorgram families read the
        posteriorgrams where they are.  Exactly one input:
          grams  (notes, onsets, contours) lists of per-file host arrays (contours may be None when no family reads
                 them), or (note, onset, contour, frame_off) with device tensors (anything with data_ptr(); row-major,
                 work on `stream`) -> bp_evaluate_host / bp_evaluate_device;
          audio  mono 22 050 Hz float32 arrays -> bp_evaluate_audio_host (the model runs once);
          pcm    (samples, sample_rate) or `WavRegion` items as `transcribe_pcm` takes them -> bp_evaluate_pcm_files_host
                 (bp_evaluate_pcm_sources_host when a region is among them).
        families: names from EVAL_FAMILIES; settings: the decode grid of the note-derived families (as `score_grid`);
        request: note_refs, multipitch_refs, f0_refs, salience / melody dicts {settings, references, kind}, window,
        cent_tolerance and note tolerances, as the standalone calls take them.
        Returns {family: int64 counts} as the standalone `score_*` calls return them, "pairs" as `match_grid`'s (res,
        match), and with return_model_output (audio / pcm) "model_output": per-file posteriorgram dicts."""
        if sum(x is not None for x in (grams, audio, pcm)) != 1:
            raise ValueError("give exactly one of grams, audio, pcm")
        device = grams is not None and hasattr(grams[0], "data_ptr")
        if device:
            note, onset, contour, foff = grams
            foff = np.ascontiguousarray(foff, np.int64)
            n_files = len(foff) - 1
        elif grams is not None:
            notes, onsets, contours = grams
            n_files = len(notes)
            foff, n_all, o_all = self._cat_note_onset(notes, onsets)
            c_all = None if contours is None else _cat_rows(list(contours), N_FREQ_BINS_CONTOURS)
            if c_all is not None and c_all.shape[0] != foff[-1]:
                raise ValueError("contour posteriorgrams must have as many frames as note posteriorgrams")
        elif audio is not None:
            flat, offs = self._pack_audio(audio)
            n_files = len(audio)
            lens = np.diff(offs)
        else:
            from_files = any(isinstance(it, WavRegion) for it in pcm)
            if from_files:
                files, keep_pcm = pcm_sources(pcm)
                n_files = len(pcm)
                descs = [f.pcm for f in files[:n_files]]
            else:
                files, keep_pcm = pcm_descriptors(pcm)
                n_files = len(keep_pcm)
                descs = files[:n_files]
            lens = np.fromiter((self._lib.bp_resampled_length(int(f.n_frames), int(f.sample_rate)) for f in descs),
                               dtype=np.int64, count=n_files)
        req, keep, out = self._eval_request(n_files, families, settings, **request)
        n_params = len(settings)
        mo = {}
        if grams is None:
            foff = np.zeros(n_files + 1, np.int64)
            total = int(sum(self._lib.bp_num_frames(int(n)) for n in lens))
            if return_model_output:
                mo = {k: np.empty((total, w), _F32) for k, w in (("note", N_FREQ_BINS_NOTES), ("onset", N_FREQ_BINS_NOTES),
                                                                 ("contour", N_FREQ_BINS_CONTOURS))}

        def call(notes=None):
            req.pair_notes = C.addressof(notes) if notes is not None else None
            if device:
                self._lib.bp_evaluate_device(self._h, note.data_ptr(), onset.data_ptr(),
                                             None if contour is None else contour.data_ptr(), _ptr(foff), n_files,
                                             C.byref(req), stream or None)
            elif grams is not None:
                self._lib.bp_evaluate_host(self._h, _ptr(n_all), _ptr(o_all), _ptr(c_all), _ptr(foff), n_files, C.byref(req))
            elif audio is not None:
                self._lib.bp_evaluate_audio_host(self._h, _ptr(flat), _ptr(offs), n_files, C.byref(req), _ptr(mo.get("note")),
                                                 _ptr(mo.get("onset")), _ptr(mo.get("contour")), _ptr(foff))
            else:
                entry = self._lib.bp_evaluate_pcm_sources_host if from_files else self._lib.bp_evaluate_pcm_files_host
                entry(self._h, files, n_files, C.byref(req), _ptr(mo.get("note")), _ptr(mo.get("onset")),
                      _ptr(mo.get("contour")), _ptr(foff), None)

        if "pairs" in families:
            total = int(foff[-1]) if grams is not None else total
            arrs = self._with_capacity(n_files, total, call, n_params=n_params)
            flat_res = self._split_notes(arrs, n_params * n_files)
            h_match, roff = out["pairs"]
            out["pairs"] = ([flat_res[k * n_files : (k + 1) * n_files] for k in range(n_params)],
                            [[h_match[k, :, roff[i] : roff[i + 1]].copy() for i in range(n_files)] for k in range(n_params)])
        else:
            call()
        if grams is None:
            out["frame_off"] = foff
            if return_model_output:
                fo = foff.tolist()
                out["model_output"] = [{k: v[a:b] for k, v in mo.items()} for a, b in zip(fo[:-1], fo[1:])]
        return out

    def evaluate_chunk_params(self, total_frames: int, families: Sequence[str], settings: Sequence[Dict[str, Any]] = (),
                              **request) -> int:
        """`bp_evaluate_chunk_params`: settings per decode chunk of `evaluate` over a batch of this many frames."""
        n_files = max(len(request.get(k) or ()) for k in ("note_refs", "multipitch_refs", "f0_refs"))
        req, keep, _ = self._eval_request(n_files, families, settings, **request)
        return int(self._lib.bp_evaluate_chunk_params(int(total_frames), n_files, C.byref(req)))

    def infer_onsets_array(self, onsets: np.ndarray, frames: np.ndarray) -> np.ndarray:
        """reference: note_creation.py:289-311 `get_infered_onsets` (n_diff = 2) -> float64 (T, 88), on the device."""
        o = np.ascontiguousarray(onsets, dtype=_F32)
        f = np.ascontiguousarray(frames, dtype=_F32)
        if o.ndim != 2 or o.shape[1] != N_FREQ_BINS_NOTES or f.shape != o.shape:
            raise ValueError("onsets / frames must be (T, 88) and of equal shape")
        out = np.empty(o.shape, np.float64)
        self._lib.bp_infer_onsets_host(self._h, _ptr(o), _ptr(f), o.shape[0], _ptr(out))
        return out

    def pitch_bends_arrays(self, contours: np.ndarray, start: np.ndarray, end: np.ndarray, pitch: np.ndarray):
        """reference: note_creation.py:182-219 `get_pitch_bends` for given notes -> (bend_off int32[n+1], bends int32[])."""
        c = np.ascontiguousarray(contours, dtype=_F32)
        if c.ndim != 2 or c.shape[1] != N_FREQ_BINS_CONTOURS:
            raise ValueError("contours must be (T, 264)")
        st = np.ascontiguousarray(start, dtype=np.int32)
        en = np.ascontiguousarray(end, dtype=np.int32)
        pi = np.ascontiguousarray(pitch, dtype=np.int32)
        n = len(st)
        off = np.zeros(n + 1, np.int32)
        cap = int(np.maximum(en.astype(np.int64) - st.astype(np.int64), 0).sum())
        bends = np.empty(max(cap, 1), np.int32)
        self._lib.bp_pitch_bends_host(self._h, _ptr(c), c.shape[0], n, _ptr(st), _ptr(en), _ptr(pi), _ptr(off), _ptr(bends), cap)
        return off, bends[: int(off[n])]

    # ------------------------------------------------------------------ the whole path
    def transcribe_arrays(self, audios: Sequence[np.ndarray], onset_thresh=0.5, frame_thresh=0.3, min_note_len=11,
                          energy_tol=11, infer_onsets=True, melodia_trick=True, include_pitch_bends=True,
                          min_pitch_idx=0, max_pitch_idx=88, return_model_output: bool = True, split_notes: bool = True):
        """Audio of a batch of files -> (model outputs | None, note arrays) per file in ONE library call
        (reference: inference.py:431-506 `predict`, minus file I/O and the MIDI object).  With split_notes=False the
        second result is the concatenated arrays of the call (note_off, start, end, pitch, amp, bend_off, bends)."""
        n_files = len(audios)
        # one pointer per file: the library gathers the (pageable) arrays into pinned staging itself, sub-batch by
        # sub-batch, overlapped with the kernels (bp_transcribe_files_host) — no host-side concatenation
        keep = []
        for a in audios:
            if a.ndim != 1:
                raise ValueError("audio must be mono (1-D)")
            keep.append(a if (a.dtype == _F32 and a.flags.c_contiguous) else np.ascontiguousarray(a, dtype=_F32))
        ptrs = (C.c_void_p * max(n_files, 1))(*[a.ctypes.data for a in keep])
        lens = np.fromiter((a.shape[0] for a in keep), dtype=np.int64, count=n_files)
        p = self._params(onset_thresh, frame_thresh, min_note_len, energy_tol, infer_onsets, melodia_trick,
                         include_pitch_bends, min_pitch_idx, max_pitch_idx)
        return self._transcribe(
            lens, return_model_output, split_notes,
            lambda note, onset, contour, foff, nt: self._lib.bp_transcribe_files_host(
                self._h, ptrs, _ptr(lens), n_files, C.byref(p), _ptr(note), _ptr(onset), _ptr(contour), _ptr(foff), C.byref(nt)),
        )

    def transcribe_pcm(self, items: Sequence[Tuple[np.ndarray, int]], onset_thresh=0.5, frame_thresh=0.3, min_note_len=11,
                       energy_tol=11, infer_onsets=True, melodia_trick=True, include_pitch_bends=True,
                       min_pitch_idx=0, max_pitch_idx=88, return_model_output: bool = True, split_notes: bool = True):
        """`transcribe_arrays` for files given as their stored samples: an item is (samples, sample_rate) as
        `audio_io.read_pcm` returns them — (n,) or (n, channels), float32 / int16 / int32 / uint8, any rate — or a
        `WavRegion` from `audio_io.probe_wav`, whose samples the library reads from the file itself.  ONE library call
        (bp_transcribe_pcm_files_host; bp_transcribe_pcm_sources_host when a region is among the items): the samples go
        up as stored, one batched ingest per sub-batch converts, down-mixes and resamples them on the device, and the
        forward pass reads the result there.  Same results as `load_audio_device` per file followed by
        `transcribe_arrays`, same return value.  A region's file that cannot be read during the call raises OSError
        (`_lib.BpIOError`) naming it."""
        from_files = any(isinstance(it, WavRegion) for it in items)
        if from_files:
            files, keep = pcm_sources(items)
            n_files = len(items)
            descs = [f.pcm for f in files[:n_files]]
        else:
            files, keep = pcm_descriptors(items)
            n_files = len(keep)
            descs = files[:n_files]
        lens = np.fromiter((self._lib.bp_resampled_length(int(f.n_frames), int(f.sample_rate)) for f in descs),
                           dtype=np.int64, count=n_files)
        p = self._params(onset_thresh, frame_thresh, min_note_len, energy_tol, infer_onsets, melodia_trick,
                         include_pitch_bends, min_pitch_idx, max_pitch_idx)
        entry = self._lib.bp_transcribe_pcm_sources_host if from_files else self._lib.bp_transcribe_pcm_files_host
        return self._transcribe(
            lens, return_model_output, split_notes,
            lambda note, onset, contour, foff, nt: entry(
                self._h, files, n_files, C.byref(p), _ptr(note), _ptr(onset), _ptr(contour), _ptr(foff), None, C.byref(nt)),
        )

    def _transcribe(self, lens: np.ndarray, return_model_output: bool, split_notes: bool, call):
        """The part the whole-path calls share: outputs for files of `lens` samples at 22 050 Hz, capacity negotiation
        around call(note, onset, contour, frame_off, notes), and the per-file views."""
        n_files = len(lens)
        frames = [int(self._lib.bp_num_frames(int(n))) for n in lens]
        total = sum(frames)
        note = onset = contour = None
        if return_model_output:  # page-locked: the posteriorgrams stream back while later sub-batches compute
            note = self._pinned.array((total, N_FREQ_BINS_NOTES))
            onset = self._pinned.array((total, N_FREQ_BINS_NOTES))
            contour = self._pinned.array((total, N_FREQ_BINS_CONTOURS))
        foff = np.zeros(n_files + 1, np.int64)
        arrs = self._with_capacity(n_files, total, lambda nt: call(note, onset, contour, foff, nt))
        res = self._split_notes(arrs, n_files) if split_notes else arrs
        outs: List[Optional[Dict[str, np.ndarray]]] = [None] * n_files
        if return_model_output:
            fo = foff.tolist()
            outs = [{"note": note[a:b], "onset": onset[a:b], "contour": contour[a:b]} for a, b in zip(fo[:-1], fo[1:])]
        return outs, res, frames


_DEFAULT_MODELS: Dict[Tuple[str, int], Model] = {}


class NoteStream:
    """The note decode of one streamed recording (`Model.note_stream`).  `push(note, onset, contour)` takes the next
    frames ((T, 88), (T, 88), (T, 264) arrays; contour may be None without pitch bends) and `end()` closes the
    recording; both return the note events that became final, as the reference's (start_s, end_s, pitch, amplitude,
    bends) tuples with times at their frame index in the whole recording.  `held_frames` is the number of frames the
    device holds."""

    def __init__(self, model: Model, params: _lib.DecodeParams, max_segment_frames: Optional[int] = None):
        self._model, self._lib = model, model._lib
        self._bends = bool(params.include_pitch_bends)
        self._h = C.c_void_p()
        self._lib.bp_stream_create(model.handle, C.byref(params), int(max_segment_frames or 0), C.byref(self._h))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and getattr(self, "_lib", None) is not None:
            try:
                self._lib.bp_stream_destroy(h)
            except Exception:
                pass

    @property
    def held_frames(self) -> int:
        return int(self._lib.bp_stream_held_frames(self._h))

    def push(self, note: np.ndarray, onset: np.ndarray, contour: Optional[np.ndarray]) -> List[infer.NoteEvent]:
        note = np.ascontiguousarray(note, dtype=_F32).reshape(-1, N_FREQ_BINS_NOTES)
        onset = np.ascontiguousarray(onset, dtype=_F32).reshape(-1, N_FREQ_BINS_NOTES)
        if onset.shape != note.shape:
            raise ValueError("note and onset posteriorgrams must be (T, 88) and of equal shape")
        if contour is not None:
            contour = np.ascontiguousarray(contour, dtype=_F32).reshape(-1, N_FREQ_BINS_CONTOURS)
            if contour.shape[0] != note.shape[0]:
                raise ValueError("contour posteriorgrams must have as many frames as note posteriorgrams")
        elif self._bends:
            raise ValueError("pitch bends need the contour posteriorgram")
        self._lib.bp_stream_push_host(self._h, _ptr(note), _ptr(onset), _ptr(contour), note.shape[0])
        return self._take()

    def end(self) -> List[infer.NoteEvent]:
        self._lib.bp_stream_end(self._h)
        return self._take()

    def _take(self) -> List[infer.NoteEvent]:
        arrs = self._model._with_capacity(1, 0, lambda nt: self._lib.bp_stream_take(self._h, C.byref(nt)))
        return _note_events(arrs, 0, int(arrs["note_off"][1]), self._bends)


def _note_events(arrs, a: int, b: int, bends: bool) -> List[infer.NoteEvent]:
    """Notes a .. b of taken note arrays (global frame indices) -> the reference's event tuples."""
    start, end = arrs["start"][a:b], arrs["end"][a:b]
    t0, t1 = infer.frame_index_to_time(start.astype(np.int64)), infer.frame_index_to_time(end.astype(np.int64))
    off, flat = arrs["bend_off"], arrs["bends"]
    return [
        (t0[j - a], t1[j - a], np.int64(arrs["pitch"][j]), np.float32(arrs["amp"][j]),
         list(flat[off[j] : off[j + 1]].astype(np.int64)) if bends else None)
        for j in range(a, b)
    ]  # fmt: skip


def _pcm_block(block, dtype: np.dtype, channels: int) -> np.ndarray:
    """A PCM stream's block as the library takes it: C-contiguous (n, channels) of the stream's dtype.  (n,) stands for
    (n, 1).  ValueError for any other dtype, channel count or shape."""
    b = np.asarray(block)
    if b.dtype != dtype:
        raise ValueError(f"a block of this PCM stream must be {dtype}, got {b.dtype}")
    if b.ndim == 1 and channels == 1:
        b = b.reshape(-1, 1)
    if b.ndim != 2 or b.shape[1] != channels:
        raise ValueError(f"a block of this {channels}-channel PCM stream must be (n, {channels})"
                         + (" or (n,)" if channels == 1 else "") + f", got shape {b.shape}")
    return np.ascontiguousarray(b)


def _pcm_format(dtype) -> int:
    from .audio_io import _PCM_FORMATS

    dt = np.dtype(dtype)
    if dt not in _PCM_FORMATS:
        raise ValueError(f"PCM dtype must be float32, int16, int32 or uint8, got {dt}")
    return _PCM_FORMATS[dt]


class StreamGroup:
    """Many streamed recordings decoded together (`Model.stream_group`, `bp_stream_group_*`): each call serves every
    stream it lists with one device pass — one forward pass over the windows the new audio completes, one quiet scan,
    and the closed stretches of all streams decoded as one batch per round.  Every stream's notes are those a
    `NoteStream` (and `predict_stream_notes`) gives for the same recording on its own.

    `open()` adds a stream and returns its id.  `push({id: block})` takes the next mono 22 050 Hz audio block of some
    streams (any length, 0 included), `push_frames({id: (note, onset, contour)})` posteriorgrams instead (a stream takes
    one kind only), `end(ids)` closes streams.  Each returns {id: note_events} for the streams it lists, the events that
    became final; with `with_posteriorgrams` also {id: model_output_part}, the frames each stream committed in that call
    (concatenated, `run_inference_stream`'s output for the stream's blocks).  `held_frames(id)` is what
    `NoteStream.held_frames` reports.

    `open_pcm(sample_rate, channels, dtype)` adds a stream that takes its blocks as captured: (n,) or (n, channels)
    arrays of that dtype (float32, int16, int32 or uint8, as `audio_io.read_pcm` returns them) at that rate, resampled
    on the device with state carried across pushes, so that its signal is `bp_load_pcm_host` of the whole recording
    whatever the blocks (DESIGN.md §4.6)."""

    def __init__(self, model: Model, params: _lib.DecodeParams, max_segment_frames: Optional[int] = None):
        self._model, self._lib = model, model._lib
        self._pcm: Dict[int, Tuple[np.dtype, int]] = {}  # PCM stream id -> (dtype, channels)
        self._bends = bool(params.include_pitch_bends)
        self._h = C.c_void_p()
        self._lib.bp_stream_group_create(model.handle, C.byref(params), int(max_segment_frames or 0), C.byref(self._h))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and getattr(self, "_lib", None) is not None:
            try:
                self._lib.bp_stream_group_destroy(h)
            except Exception:
                pass

    def open(self) -> int:
        i = C.c_int32(0)
        self._lib.bp_stream_group_open(self._h, C.byref(i))
        return int(i.value)

    def open_pcm(self, sample_rate: int, channels: int, dtype) -> int:
        fmt = _pcm_format(dtype)
        i = C.c_int32(0)
        self._lib.bp_stream_group_open_pcm(self._h, fmt, int(channels), int(sample_rate), C.byref(i))
        self._pcm[int(i.value)] = (np.dtype(dtype), int(channels))
        return int(i.value)

    def held_frames(self, stream_id: int) -> int:
        return int(self._lib.bp_stream_group_held_frames(self._h, int(stream_id)))

    @staticmethod
    def _ids(ids) -> np.ndarray:
        return np.ascontiguousarray(np.asarray(list(ids), dtype=np.int64).reshape(-1).astype(np.int32))

    def _call(self, ids: np.ndarray, call, n_samples, with_posteriorgrams: bool):
        """call(note, onset, contour, frame_off) with output arrays sized by bp_stream_group_commit_offsets."""
        n = len(ids)
        off = np.zeros(n + 1, np.int64)
        outs = [None, None, None]
        if with_posteriorgrams:
            self._lib.bp_stream_group_commit_offsets(self._h, n, _ptr(ids), _ptr(n_samples), int(n_samples is None),
                                                     _ptr(off))
            total = int(off[-1])
            outs = [np.empty((total, w), _F32) for w in (N_FREQ_BINS_NOTES, N_FREQ_BINS_NOTES, N_FREQ_BINS_CONTOURS)]
        call(*(_ptr(o) for o in outs), _ptr(off))
        events = self._take(ids)
        if not with_posteriorgrams:
            return events
        parts = {int(i): {k: o[off[j] : off[j + 1]] for k, o in zip(("note", "onset", "contour"), outs)}
                 for j, i in enumerate(ids)}  # fmt: skip
        return events, parts

    def push(self, blocks: Mapping[int, np.ndarray], with_posteriorgrams: bool = False):
        ids = self._ids(blocks.keys())
        pcm = any(int(i) in self._pcm for i in ids)
        audio = [_pcm_block(b, *self._pcm[int(i)]) if int(i) in self._pcm
                 else np.ascontiguousarray(np.asarray(b, dtype=_F32).reshape(-1)) for i, b in zip(ids, blocks.values())]
        ptrs = (C.c_void_p * max(len(audio), 1))(*[a.ctypes.data for a in audio])
        lens = np.array([a.shape[0] for a in audio], np.int64)  # PCM frames of a PCM stream
        push = self._lib.bp_stream_group_push_pcm_host if pcm else self._lib.bp_stream_group_push_host
        return self._call(ids, lambda no, on, co, off: push(self._h, len(ids), _ptr(ids), ptrs, _ptr(lens), no, on, co, off),
                          lens, with_posteriorgrams)

    def debug_tail(self, stream_id: int) -> Tuple[int, np.ndarray]:
        """(first sample, samples) of the stream's held 22 050 Hz tail (`bp_stream_group_debug_tail`)."""
        first, n = C.c_int64(0), C.c_int64(0)
        try:
            self._lib.bp_stream_group_debug_tail(self._h, int(stream_id), None, 0, C.byref(first), C.byref(n))
            return int(first.value), np.zeros(0, _F32)
        except _lib.BpError as e:
            if e.code != _lib.BP_E_CAPACITY:
                raise
        out = np.empty(int(n.value), _F32)
        self._lib.bp_stream_group_debug_tail(self._h, int(stream_id), _ptr(out), out.shape[0], C.byref(first),
                                             C.byref(n))
        return int(first.value), out

    def push_frames(self, frames: Mapping[int, Tuple[np.ndarray, np.ndarray, Optional[np.ndarray]]]):
        ids = self._ids(frames.keys())
        keep, rows = [], []
        for note, onset, contour in frames.values():
            note = np.ascontiguousarray(note, dtype=_F32).reshape(-1, N_FREQ_BINS_NOTES)
            onset = np.ascontiguousarray(onset, dtype=_F32).reshape(-1, N_FREQ_BINS_NOTES)
            if onset.shape != note.shape:
                raise ValueError("note and onset posteriorgrams must be (T, 88) and of equal shape")
            if contour is not None:
                contour = np.ascontiguousarray(contour, dtype=_F32).reshape(-1, N_FREQ_BINS_CONTOURS)
                if contour.shape[0] != note.shape[0]:
                    raise ValueError("contour posteriorgrams must have as many frames as note posteriorgrams")
            elif self._bends:
                raise ValueError("pitch bends need the contour posteriorgram")
            keep.append((note, onset, contour))
            rows.append(note.shape[0])
        n = max(len(keep), 1)
        ptrs = [(C.c_void_p * n)(*[_ptr(k[c]) for k in keep]) for c in range(3)]
        lens = np.array(rows, np.int64)
        self._lib.bp_stream_group_push_frames_host(self._h, len(ids), _ptr(ids), *ptrs, _ptr(lens))
        return self._take(ids)

    def end(self, ids: Iterable[int], with_posteriorgrams: bool = False):
        ids = self._ids(ids)
        return self._call(ids, lambda no, on, co, off: self._lib.bp_stream_group_end(self._h, len(ids), _ptr(ids), no, on,
                                                                                    co, off),
                          None, with_posteriorgrams)

    def _take(self, ids: np.ndarray) -> Dict[int, List[infer.NoteEvent]]:
        arrs = self._model._with_capacity(
            len(ids), 0, lambda nt: self._lib.bp_stream_group_take(self._h, len(ids), _ptr(ids), C.byref(nt)))
        off = arrs["note_off"]
        return {int(i): _note_events(arrs, int(off[j]), int(off[j + 1]), self._bends) for j, i in enumerate(ids)}


def default_model(model_path: Union[pathlib.Path, str] = ICASSP_2022_MODEL_PATH, device: Optional[int] = None) -> Model:
    """One shared `Model` per (path, device); what `predict(path)` uses when given a path."""
    dev = _default_device() if device is None else int(device)
    key = (str(model_path), dev)
    if key not in _DEFAULT_MODELS:
        _DEFAULT_MODELS[key] = Model(model_path, dev)
    return _DEFAULT_MODELS[key]


# ---------------------------------------------------------------------------------------------
# Windowing helpers (host-side equivalents kept for API compatibility; the hot path does this
# arithmetic on the device, see bp_run_inference_* in include/bp_b200.h).
# ---------------------------------------------------------------------------------------------
def window_audio_file(audio_original: np.ndarray, hop_size: int) -> Iterable[Tuple[np.ndarray, Dict[str, float]]]:
    """reference: inference.py:194-219"""
    for i in range(0, audio_original.shape[0], hop_size):
        window = audio_original[i : i + AUDIO_N_SAMPLES]
        if len(window) < AUDIO_N_SAMPLES:
            window = np.pad(window, pad_width=[[0, AUDIO_N_SAMPLES - len(window)]])
        t_start = float(i) / AUDIO_SAMPLE_RATE
        yield np.expand_dims(window, axis=-1), {"start": t_start, "end": t_start + (AUDIO_N_SAMPLES / AUDIO_SAMPLE_RATE)}


def get_audio_input(audio_path: Union[pathlib.Path, str], overlap_len: int, hop_size: int):
    """reference: inference.py:222-244"""
    assert overlap_len % 2 == 0, f"overlap_length must be even, got {overlap_len}"
    audio_original, _ = load_audio(audio_path, sr=AUDIO_SAMPLE_RATE, mono=True)
    original_length = audio_original.shape[0]
    audio_original = np.concatenate([np.zeros((int(overlap_len / 2),), dtype=np.float32), audio_original])
    for window, window_time in window_audio_file(audio_original, hop_size):
        yield np.expand_dims(window, axis=0), window_time, original_length


def unwrap_output(output: np.ndarray, audio_original_length: int, n_overlapping_frames: int, hop_size: int):
    """reference: inference.py:247-279"""
    if len(output.shape) != 3:
        return None
    n_olap = int(0.5 * n_overlapping_frames)
    if n_olap > 0:
        output = output[:, n_olap:-n_olap, :]
    flat = output.reshape(output.shape[0] * output.shape[1], output.shape[2])
    n_expected_windows = audio_original_length / hop_size
    n_frames_per_window = (AUDIO_WINDOW_LENGTH * ANNOTATIONS_FPS) - n_overlapping_frames
    return flat[: int(n_expected_windows * n_frames_per_window), :]


def run_inference(audio_path: Union[pathlib.Path, str], model_or_model_path: Union[Model, pathlib.Path, str],
                  debug_file: Optional[pathlib.Path] = None) -> Dict[str, np.ndarray]:
    """reference: inference.py:282-330 — returns the unwrapped note / onset / contour posteriorgrams."""
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    audio, _ = load_audio(audio_path, sr=AUDIO_SAMPLE_RATE, mono=True)
    out = model.run_inference_arrays([audio])[0]
    if debug_file:
        n_overlap = DEFAULT_OVERLAPPING_FRAMES * FFT_HOP
        with open(debug_file, "w") as f:
            hop = AUDIO_N_SAMPLES - n_overlap
            padded = np.concatenate([np.zeros(n_overlap // 2, _F32), audio])
            last = padded[(max(len(padded) - 1, 0) // hop) * hop :][:AUDIO_N_SAMPLES]  # the reference dumps the LAST window
            json.dump({
                "audio_windowed": np.pad(last, (0, AUDIO_N_SAMPLES - len(last))).reshape(1, AUDIO_N_SAMPLES, 1).tolist(),
                "audio_original_length": int(audio.shape[0]),
                "hop_size_samples": AUDIO_N_SAMPLES - n_overlap,
                "overlap_length_samples": n_overlap,
                "unwrapped_output": {k: v.tolist() for k, v in out.items()},
            }, f)  # fmt: skip
    return out


def run_inference_stream(audio_blocks: Iterable[np.ndarray], model_or_model_path: Union["Model", pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
                         windows_per_step: int = 64) -> Iterable[Dict[str, np.ndarray]]:
    """Bounded-memory inference for long recordings (reference: README.md:196-198 — "we recommend streaming the audio of
    the file, processing windows of audio at a time").

    audio_blocks: an iterable of consecutive mono 22 050 Hz float blocks of any sizes (e.g. a file read piecewise).
    Yields dicts {"note", "onset", "contour"} of consecutive unwrapped frames; concatenated they equal
    `run_inference(whole_file)` bit for bit.  At any time the host holds at most `windows_per_step` windows of audio
    (~1.6 s each) plus two windows of held-back frames, the device one step of windows: memory does not grow with the
    length of the recording.  (The final trim of `unwrap_output`, inference.py:247-279, can reach two windows back, so
    the frames of the last two windows are yielded when the stream ends.)"""
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    n_overlap = DEFAULT_OVERLAPPING_FRAMES * FFT_HOP
    hop = AUDIO_N_SAMPLES - n_overlap
    n_olap = DEFAULT_OVERLAPPING_FRAMES // 2
    per_window = AUDIO_WINDOW_LENGTH * ANNOTATIONS_FPS - DEFAULT_OVERLAPPING_FRAMES  # 142 kept frames per window
    buf = np.zeros(n_overlap // 2, _F32)  # the reference prepends overlap_len / 2 zeros (inference.py:241)
    total = 0  # samples of the recording seen so far
    emitted = 0  # frames yielded so far
    held: List[Dict[str, np.ndarray]] = []  # frames of the newest windows, not yet safe to yield

    def run(windows: np.ndarray) -> None:
        out = model.predict(windows)
        for k in range(windows.shape[0]):
            held.append({key: out[key][k, n_olap : 172 - n_olap] for key in ("note", "onset", "contour")})

    def drain(keep: int):
        nonlocal emitted
        while len(held) > keep:
            w = held.pop(0)
            emitted += per_window
            yield w

    for block in audio_blocks:
        block = np.asarray(block, dtype=_F32).reshape(-1)
        total += block.shape[0]
        buf = np.concatenate([buf, block])
        n_ready = (buf.shape[0] - AUDIO_N_SAMPLES) // hop + 1 if buf.shape[0] >= AUDIO_N_SAMPLES else 0
        while n_ready > 0:
            n = min(n_ready, windows_per_step)
            idx = np.arange(n)[:, None] * hop + np.arange(AUDIO_N_SAMPLES)[None, :]
            run(buf[idx])
            buf = buf[n * hop :]
            n_ready -= n
            yield from drain(2)
    # end of stream: the windows that start inside the remaining samples, zero-padded (inference.py:194-219)
    tail = []
    for i in range(0, buf.shape[0], hop):
        w = buf[i : i + AUDIO_N_SAMPLES]
        tail.append(np.pad(w, (0, AUDIO_N_SAMPLES - w.shape[0])))
    for c0 in range(0, len(tail), windows_per_step):
        run(np.stack(tail[c0 : c0 + windows_per_step]))
    # the trim of unwrap_output: keep int(n_samples / hop * frames_per_window) frames in all
    n_final = int(total / hop * per_window)
    for w in held:
        take = max(0, min(per_window, n_final - emitted))
        emitted += take
        if take > 0:
            yield {k: v[:take] for k, v in w.items()}
    held.clear()


def predict_stream(audio_blocks: Iterable[np.ndarray], model_or_model_path: Union["Model", pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
                   onset_threshold: float = DEFAULT_ONSET_THRESHOLD, frame_threshold: float = DEFAULT_FRAME_THRESHOLD,
                   minimum_note_length: float = DEFAULT_MINIMUM_NOTE_LENGTH_MS, minimum_frequency: Optional[float] = None,
                   maximum_frequency: Optional[float] = None, multiple_pitch_bends: bool = False, melodia_trick: bool = True,
                   midi_tempo: float = DEFAULT_MINIMUM_MIDI_TEMPO, windows_per_step: int = 64):
    """`predict` for a recording delivered block by block: the model runs with bounded memory (`run_inference_stream`), the
    posteriorgrams (1.76 KB per frame, 86 frames per second) are collected on the host and decoded once — the note
    decode is global over a file (reference: note_creation.py:409-509).  Returns (model_output, midi_data, note_events)."""
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    parts = list(run_inference_stream(audio_blocks, model, windows_per_step))
    keys = ("note", "onset", "contour")
    widths = {"note": N_FREQ_BINS_NOTES, "onset": N_FREQ_BINS_NOTES, "contour": N_FREQ_BINS_CONTOURS}
    model_output = {k: (np.concatenate([p[k] for p in parts]) if parts else np.zeros((0, widths[k]), _F32)) for k in keys}
    min_note_len = int(np.round(minimum_note_length / 1000 * (AUDIO_SAMPLE_RATE / FFT_HOP)))
    midi_data, note_events = infer.model_output_to_notes(
        model_output, onset_thresh=onset_threshold, frame_thresh=frame_threshold, min_note_len=min_note_len,
        min_freq=minimum_frequency, max_freq=maximum_frequency, multiple_pitch_bends=multiple_pitch_bends,
        melodia_trick=melodia_trick, midi_tempo=midi_tempo, model=model,
    )
    return model_output, midi_data, note_events


def predict_stream_notes(audio_blocks: Iterable[np.ndarray],
                         model_or_model_path: Union["Model", pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
                         onset_threshold: float = DEFAULT_ONSET_THRESHOLD, frame_threshold: float = DEFAULT_FRAME_THRESHOLD,
                         minimum_note_length: float = DEFAULT_MINIMUM_NOTE_LENGTH_MS,
                         minimum_frequency: Optional[float] = None, maximum_frequency: Optional[float] = None,
                         melodia_trick: bool = True, max_segment_seconds: Optional[float] = None,
                         windows_per_step: int = 64):
    """`predict`'s note events for a recording delivered block by block, yielded as they become final: a generator of
    (model_output_part, note_events) per step.  The parts are `run_inference_stream`'s, in order, followed by one part
    of zero frames that carries the notes of the end of the recording; the events are the reference's
    (start_s, end_s, pitch, amplitude, bends) tuples with times in the whole recording.  The decode (`Model.note_stream`)
    holds only the frames since the last quiet stretch on the device, so memory does not grow with the recording.
    A stretch's notes equal `predict`'s once both of the recording's maxima that the inferred onsets use have arrived
    (DESIGN.md §4.5); max_segment_seconds also cuts a stretch that grows longer than that, where the notes may differ.
    The keyword arguments that shape the notes are `predict`'s, with its defaults; the MIDI ones do not apply."""
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    min_note_len = int(np.round(minimum_note_length / 1000 * (AUDIO_SAMPLE_RATE / FFT_HOP)))
    max_seg = None if max_segment_seconds is None else max(1, int(np.round(max_segment_seconds * AUDIO_SAMPLE_RATE / FFT_HOP)))
    stream = model.note_stream(onset_threshold, frame_threshold, min_note_len, minimum_frequency, maximum_frequency,
                               melodia_trick, True, max_seg)
    for part in run_inference_stream(audio_blocks, model, windows_per_step):
        yield part, stream.push(part["note"], part["onset"], part["contour"])
    widths = {"note": N_FREQ_BINS_NOTES, "onset": N_FREQ_BINS_NOTES, "contour": N_FREQ_BINS_CONTOURS}
    yield {k: np.zeros((0, w), _F32) for k, w in widths.items()}, stream.end()


def predict_streams_notes(audio_streams: Sequence[Iterable[np.ndarray]],
                          model_or_model_path: Union["Model", pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
                          onset_threshold: float = DEFAULT_ONSET_THRESHOLD, frame_threshold: float = DEFAULT_FRAME_THRESHOLD,
                          minimum_note_length: float = DEFAULT_MINIMUM_NOTE_LENGTH_MS,
                          minimum_frequency: Optional[float] = None, maximum_frequency: Optional[float] = None,
                          melodia_trick: bool = True, max_segment_seconds: Optional[float] = None,
                          sample_rates: Optional[Sequence[Optional[int]]] = None):
    """`predict_stream_notes` for many live recordings at once (`Model.stream_group`): each step pulls one block from
    every iterator that has not ended, pushes them together, ends the recordings whose iterator is exhausted and yields
    {index: note_events} for the recordings it served.  Every recording's events, concatenated over the steps, equal
    `predict_stream_notes`' on its blocks alone; the keyword arguments are that function's.

    sample_rates[i] (None: every recording's blocks are mono float32 at 22 050 Hz) is None for such a recording, or the
    capture rate of recording i, whose blocks are then PCM as captured: (n,) or (n, channels) float32, int16, int32 or
    uint8.  Its first block fixes the dtype and the channel count (a later block that differs raises ValueError), and
    its events are `predict_stream_notes`' on `bp_load_pcm_host` of the whole recording, however it was cut."""
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    min_note_len = int(np.round(minimum_note_length / 1000 * (AUDIO_SAMPLE_RATE / FFT_HOP)))
    max_seg = None if max_segment_seconds is None else max(1, int(np.round(max_segment_seconds * AUDIO_SAMPLE_RATE / FFT_HOP)))
    group = model.stream_group(onset_threshold, frame_threshold, min_note_len, minimum_frequency, maximum_frequency,
                               melodia_trick, True, max_seg)
    rates = list(sample_rates) if sample_rates is not None else [None] * len(audio_streams)
    if len(rates) != len(audio_streams):
        raise ValueError("sample_rates must give one entry per recording")
    live = {}
    for k, it in enumerate(audio_streams):
        it = iter(it)
        if rates[k] is None:
            live[group.open()] = (k, it)
            continue
        try:  # the first block fixes the stream's format
            first = np.asarray(next(it))
        except StopIteration:
            live[group.open()] = (k, it)  # an empty recording
            continue
        channels = 1 if first.ndim == 1 else (first.shape[1] if first.ndim == 2 else 0)
        if channels < 1:
            raise ValueError(f"recording {k}: PCM blocks must be (n,) or (n, channels), got shape {first.shape}")
        live[group.open_pcm(int(rates[k]), channels, first.dtype)] = (k, itertools.chain([first], it))
    while live:
        blocks, done = {}, []
        for sid, (_, it) in live.items():
            try:
                blocks[sid] = next(it)
            except StopIteration:
                done.append(sid)
        events = group.push(blocks) if blocks else {}
        events.update(group.end(done) if done else {})
        yield {live[sid][0]: ev for sid, ev in events.items()}
        for sid in done:
            del live[sid]


class OutputExtensions(enum.Enum):
    MIDI = "mid"
    MODEL_OUTPUT_NPZ = "npz"
    MIDI_SONIFICATION = "wav"
    NOTE_EVENTS = "csv"


def verify_input_path(audio_path: Union[pathlib.Path, str]) -> None:
    if not os.path.isfile(audio_path):
        raise ValueError(f"🚨 {audio_path} is not a file path.")
    if not os.path.exists(audio_path):
        raise ValueError(f"🚨 {audio_path} does not exist.")


def verify_output_dir(output_dir: Union[pathlib.Path, str]) -> None:
    if not os.path.isdir(output_dir):
        raise ValueError(f"🚨 {output_dir} is not a directory.")
    if not os.path.exists(output_dir):
        raise ValueError(f"🚨 {output_dir} does not exist.")


def build_output_path(audio_path: Union[pathlib.Path, str], output_directory: Union[pathlib.Path, str],
                      output_type: OutputExtensions) -> pathlib.Path:
    """reference: inference.py:372-406 — `<stem>_basic_pitch.<ext>`, never overwrites."""
    basename, _ = os.path.splitext(os.path.basename(str(audio_path)))
    output_path = pathlib.Path(output_directory) / f"{basename}_basic_pitch.{output_type.value}"
    print(f"\n\n  Creating {output_type.name.lower().replace('_', ' ')}...")
    if output_path.exists():
        raise IOError(f"  🚨 {str(output_path)} already exists and would be overwritten. Skipping output files for {audio_path}.")
    return output_path


def save_note_events(note_events: List[infer.NoteEvent], save_path: Union[pathlib.Path, str]) -> None:
    """reference: inference.py:409-428"""
    with open(save_path, "w") as fhandle:
        writer = csv.writer(fhandle, delimiter=",")
        writer.writerow(["start_time_s", "end_time_s", "pitch_midi", "velocity", "pitch_bend"])
        for start_time, end_time, note_number, amplitude, pitch_bend in note_events:
            row = [start_time, end_time, note_number, int(np.round(DEFAULT_MIDI_VELOCITY_SCALE * amplitude))]
            if pitch_bend:
                row.extend(pitch_bend)
            writer.writerow(row)


def _events_and_midi(model_output, res, n_frames, min_freq, max_freq, multiple_pitch_bends, midi_tempo):
    events = infer.note_events_from_arrays(res, n_frames, include_pitch_bends=True)
    if min_freq is not None or max_freq is not None:  # the reference zeroes these columns of the returned arrays
        lo, hi = infer.frequency_to_column_range(min_freq, max_freq)
        for k in ("note", "onset"):
            model_output[k][:, :lo] = 0
            model_output[k][:, hi:] = 0
    return infer.note_events_to_midi(events, multiple_pitch_bends, midi_tempo), events


def predict(
    audio_path: Union[pathlib.Path, str],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    onset_threshold: float = DEFAULT_ONSET_THRESHOLD,
    frame_threshold: float = DEFAULT_FRAME_THRESHOLD,
    minimum_note_length: float = DEFAULT_MINIMUM_NOTE_LENGTH_MS,
    minimum_frequency: Optional[float] = None,
    maximum_frequency: Optional[float] = None,
    multiple_pitch_bends: bool = False,
    melodia_trick: bool = True,
    debug_file: Optional[pathlib.Path] = None,
    midi_tempo: float = DEFAULT_MINIMUM_MIDI_TEMPO,
):
    """reference: inference.py:431-506 -> (model_output, midi_data, note_events)."""
    print(f"Predicting MIDI for {audio_path}...")
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    audio, _ = load_audio_device(audio_path, model)  # decode on the host, convert / down-mix / resample on the GPU
    min_note_len = int(np.round(minimum_note_length / 1000 * (AUDIO_SAMPLE_RATE / FFT_HOP)))
    lo, hi = infer.frequency_to_column_range(minimum_frequency, maximum_frequency)
    outs, res, frames = model.transcribe_arrays(
        [audio], onset_thresh=onset_threshold, frame_thresh=frame_threshold, min_note_len=min_note_len,
        melodia_trick=melodia_trick, min_pitch_idx=lo, max_pitch_idx=hi,
    )
    model_output = outs[0]
    midi_data, note_events = _events_and_midi(model_output, res[0], frames[0], minimum_frequency, maximum_frequency,
                                              multiple_pitch_bends, midi_tempo)
    if debug_file:
        with open(debug_file, "w") as f:
            json.dump({
                "audio_original_length": int(audio.shape[0]),
                "unwrapped_output": {k: v.tolist() for k, v in model_output.items()},
                "min_note_length": min_note_len,
                "onset_thresh": onset_threshold,
                "frame_thresh": frame_threshold,
                "estimated_notes": [
                    (float(s), float(e), int(p), float(a), [int(b) for b in pb] if pb else None)
                    for s, e, p, a, pb in note_events
                ],
            }, f)  # fmt: skip
    return model_output, midi_data, note_events


def _model_and_clips(audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
                     model_or_model_path: Union[Model, pathlib.Path, str]) -> Tuple[Model, List[np.ndarray]]:
    """The model, and `audio`'s items as mono 22 050 Hz arrays: arrays as given, paths decoded on the host and converted
    and resampled on the GPU (`load_audio_device`)."""
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    clips = []
    for a in audio:
        if isinstance(a, np.ndarray):
            if a.ndim != 1:
                raise ValueError("audio must be mono (1-D)")
            clips.append(a)
        else:
            clips.append(load_audio_device(a, model)[0])
    return model, clips


def _match_counts(n_frames, ref_ivs, res, match):
    """Of `Model.match_grid`'s (res, match) on files of n_frames model frames: the estimated intervals in seconds
    [setting][file], and counts (n_settings, n_files, 4) = n_ref, n_est, matched without offsets, matched."""
    times = [infer.model_frames_to_time(t + 1) for t in n_frames]
    counts = np.zeros((len(res), len(n_frames), 4), np.int64)
    est_ivs = []
    for k, per in enumerate(res):
        est_ivs.append([np.stack([times[i][r["start"]], times[i][r["end"]]], 1) for i, r in enumerate(per)])
        for i, m in enumerate(match[k]):
            counts[k, i] = (len(ref_ivs[i]), len(per[i]["start"]), (m[0] >= 0).sum(), (m[1] >= 0).sum())
    return est_ivs, counts


def predict_grid(
    audio: Union[np.ndarray, pathlib.Path, str],
    settings: Sequence[Dict[str, Any]],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
):
    """`predict` of one recording under every setting of a grid (addition; no reference counterpart): the model runs
    once (device ingest of a path, then `bp_run_inference_host`) and all settings are decoded in one
    `bp_decode_grid_host` call.  `audio` is a path or a mono 22 050 Hz array; a setting is a dict of `predict`'s
    keyword arguments (onset_threshold, frame_threshold, minimum_note_length in ms, minimum_frequency,
    maximum_frequency, multiple_pitch_bends, melodia_trick, midi_tempo), missing ones take its defaults.

    Returns (model_output, [(midi_data, note_events) per setting]); each pair equals what `predict` gives for that
    setting, with the events as `NoteEventList`s and the MIDI objects as `LazyPrettyMIDI`s (`predict_batch(lazy=True)`).
    The model output is not column-zeroed: the settings may disagree on the frequency range."""
    model, (audio,) = _model_and_clips([audio], model_or_model_path)
    conv = [infer.grid_setting(s, predict_names=True) for s in settings]
    model_output = model.run_inference_arrays([audio])[0]
    arrs = model.decode_grid([model_output["note"]], [model_output["onset"]], [model_output["contour"]],
                             [d for d, _ in conv], split_notes=False)
    events = infer.note_events_batch(arrs, len(conv), include_pitch_bends=True, lazy=True)
    return model_output, [(infer.LazyPrettyMIDI(ev, **midi_kw), ev) for (_, midi_kw), ev in zip(conv, events)]


def evaluate_grid(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    references: Sequence[Tuple[np.ndarray, np.ndarray]],
    settings: Sequence[Dict[str, Any]],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    **tolerances,
):
    """Note-level scores of a batch of annotated recordings under every setting of a grid (addition; no reference
    counterpart): the model runs once over the batch, and every (setting, file) is decoded and scored against its
    file's reference notes on the device in one `bp_score_grid_host` call.  `audio` items are paths (decoded on the host,
    converted and resampled on the GPU, as in `predict`) or mono 22 050 Hz arrays; `references[i]` is file i's
    (intervals (n, 2) in seconds, pitches (n,) in Hz); a setting is a dict of `predict`'s keyword arguments (as in
    `predict_grid`); tolerances as `evaluate.TOLERANCES`.

    Returns (counts (n_settings, n_files, 4), `evaluate.note_scores(counts)`)."""
    model, clips = _model_and_clips(audio, model_or_model_path)
    decode = [infer.grid_setting(s, predict_names=True)[0] for s in settings]
    outs = model.run_inference_arrays(clips)
    counts = model.score_grid([o["note"] for o in outs], [o["onset"] for o in outs], decode, references, **tolerances)
    return counts, evaluate.note_scores(counts)


def evaluate_velocity_grid(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    references: Sequence[Tuple[np.ndarray, np.ndarray, np.ndarray]],
    settings: Sequence[Dict[str, Any]],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    velocity_tolerance: float = 0.1,
    **tolerances,
):
    """Note-level scores with velocity and overlap of a batch of annotated recordings under every setting of a grid
    (addition; no reference counterpart): the model runs once over the batch, every (setting, file) is decoded and
    matched as mir_eval 0.7 matches it on the device in one `bp_match_grid_host` call, and `evaluate.matching_scores`
    turns each matching into mir_eval's floats on the host.  `audio`, `settings` and tolerances as in `evaluate_grid`;
    `references[i]` is file i's (intervals (n, 2) in seconds, pitches (n,) in Hz, velocities (n,), finite and >= 0).
    An estimated note's velocity is the one the MIDI writer gives it (`evaluate.note_velocities`).

    Returns (counts (n_settings, n_files, 4) as `evaluate_grid`, derived from the matchings; scores), scores holding
    `evaluate.note_scores(counts)` and every key of `evaluate.matching_scores` as (n_settings, n_files) float64 arrays,
    with "mean" over files as in `note_scores`."""
    refs = _velocity_references(references)
    model, clips = _model_and_clips(audio, model_or_model_path)
    decode = [infer.grid_setting(s, predict_names=True)[0] for s in settings]
    outs = model.run_inference_arrays(clips)
    res, match = model.match_grid([o["note"] for o in outs], [o["onset"] for o in outs], decode,
                                  [(iv, hz) for iv, hz, _ in refs], **tolerances)
    return _velocity_scores([o["note"].shape[0] for o in outs], refs, res, match, velocity_tolerance)


def _velocity_references(references):
    """evaluate_velocity_grid's references, checked: [(intervals, pitches_hz, velocities)]."""
    refs = []
    for i, ref in enumerate(references):
        if len(ref) != 3:
            raise ValueError(f"references[{i}]: need (intervals, pitches_hz, velocities)")
        iv, hz, vel = ref
        vel = evaluate.check_velocities(vel, f"references[{i}]")
        if len(vel) != len(np.asarray(hz).reshape(-1)):
            raise ValueError(f"references[{i}]: {len(vel)} velocities for {len(np.asarray(hz).reshape(-1))} notes")
        refs.append((iv, hz, vel))
    return refs


def _velocity_scores(n_frames, refs, res, match, velocity_tolerance):
    """evaluate_velocity_grid's return value from the pairs of files of n_frames model frames."""
    n_params, n_files = len(res), len(n_frames)
    ref_ivs = [np.asarray(iv, np.float64).reshape(-1, 2) for iv, _, _ in refs]
    est_ivs, counts = _match_counts(n_frames, ref_ivs, res, match)
    keys = [k + s for s in ("", "_no_offset") for k in evaluate.MATCH_FIELDS]
    extra = {k: np.zeros((n_params, n_files)) for k in keys}
    for k in range(n_params):
        for i in range(n_files):
            vals = evaluate.matching_scores(ref_ivs[i], refs[i][2], est_ivs[k][i], evaluate.note_velocities(res[k][i]["amp"]),
                                            match[k][i], velocity_tolerance)
            for key in keys:
                extra[key][k, i] = vals[key]
    scores = evaluate.note_scores(counts)
    scores.update(extra)
    scores["mean"].update({k: (v.mean(axis=-1) if n_files else np.zeros(n_params)) for k, v in extra.items()})
    return counts, scores


def evaluate_transcription_grid(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    references: Sequence[Tuple[np.ndarray, np.ndarray]],
    settings: Sequence[Dict[str, Any]],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    **tolerances,
):
    """Every value of mir_eval.transcription.evaluate (0.7) for a batch of annotated recordings under every setting of a
    grid (addition; no reference counterpart).  The model runs once over the batch; one `bp_match_grid_host` call
    decodes every (setting, file) and returns mir_eval's pairs with and without offsets, which give the note scores and
    both average overlap ratios; one `bp_score_onset_offset_notes_host` call scores the notes that came back for onsets
    and offsets alone, so the grid is decoded once.  `audio`, `settings` and tolerances as in `evaluate_grid`;
    `references[i]` is file i's (intervals (n, 2) in seconds, pitches (n,) in Hz).

    Returns (counts, scores): counts int64 (n_settings, n_files, 6) = n_ref, n_est, matched without offsets, matched,
    onsets matched, offsets matched; scores the 14 values under the names `evaluate.TRANSCRIPTION_KEYS` maps mir_eval's
    keys to, in its order, as (n_settings, n_files) float64 arrays, with "mean" over files as in `note_scores`."""
    model, clips = _model_and_clips(audio, model_or_model_path)
    decode = [infer.grid_setting(s, predict_names=True)[0] for s in settings]
    outs = model.run_inference_arrays(clips)
    res, match = model.match_grid([o["note"] for o in outs], [o["onset"] for o in outs], decode, references,
                                  **tolerances)
    n_frames = [o["note"].shape[0] for o in outs]
    ref_ivs = [np.asarray(iv, np.float64).reshape(-1, 2) for iv, _ in references]
    est_ivs, _ = _match_counts(n_frames, ref_ivs, res, match)
    ests = [iv for per in est_ivs for iv in per]
    onoff = model.score_onsets_offsets(ests, ref_ivs * len(res), **tolerances).reshape(len(res), len(outs), 4)
    return _transcription_scores(n_frames, ref_ivs, res, match, onoff)


def _transcription_scores(n_frames, ref_ivs, res, match, onoff):
    """evaluate_transcription_grid's return value from the pairs and the onset / offset counts of files of n_frames
    model frames."""
    n_params, n_files = len(res), len(n_frames)
    est_ivs, counts = _match_counts(n_frames, ref_ivs, res, match)
    overlap = {k: np.zeros((n_params, n_files)) for k in ("average_overlap_ratio", "average_overlap_ratio_no_offset")}
    for k in range(n_params):
        for i in range(n_files):
            m = match[k][i]
            for suffix, row in (("", m[1]), ("_no_offset", m[0])):
                ref_idx = np.flatnonzero(row >= 0)  # sorted(matching.items()): ascending reference index
                overlap["average_overlap_ratio" + suffix][k, i] = evaluate._overlap_ratio(ref_ivs[i], est_ivs[k][i],
                                                                                           ref_idx, row[ref_idx])
    scores = evaluate.note_scores(counts)
    counts = np.concatenate([counts, onoff[..., 2:]], axis=-1)
    scores.update(overlap)
    scores["mean"].update({k: (v.mean(axis=-1) if n_files else np.zeros(n_params)) for k, v in overlap.items()})
    oo = evaluate.onset_offset_scores(onoff)
    scores["mean"].update(oo.pop("mean"))
    scores.update(oo)
    names = list(evaluate.TRANSCRIPTION_KEYS.values())
    return counts, {**{k: scores[k] for k in names}, "mean": {k: scores["mean"][k] for k in names}}


def evaluate_frames_grid(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    references: Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]],
    settings: Sequence[Dict[str, Any]],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    window: float = evaluate.WINDOW,
    pitch_bends: bool = False,
):
    """Frame-level multi-pitch scores of a batch of annotated recordings under every setting of a grid (addition; no
    reference counterpart): the model runs once over the batch, and every (setting, file) is decoded and scored against
    its file's reference series on the device in one library call.  `audio` and `settings` as in `evaluate_grid`;
    `references[i]` is file i's (times (n,) in seconds, [Hz array per frame]), mir_eval.multipitch's convention
    (`evaluate.notes_to_multipitch` makes one from note annotations); window in semitones.  With pitch_bends=False the
    estimate is the piano roll of the notes (`bp_score_frames_grid_host`); with True it is the notes with their pitch
    bends, what `predict` returns (`bp_score_bent_frames_grid_host`, `evaluate.note_frames_to_multipitch`).

    Returns (counts (n_settings, n_files, 7), `evaluate.frame_scores(counts)`)."""
    model, clips = _model_and_clips(audio, model_or_model_path)
    decode = [infer.grid_setting(s, predict_names=True)[0] for s in settings]  # include_pitch_bends: predict's True
    outs = model.run_inference_arrays(clips)
    counts = model.score_frames_grid([o["note"] for o in outs], [o["onset"] for o in outs], decode, references,
                                     window=window, contours=[o["contour"] for o in outs] if pitch_bends else None)
    return counts, evaluate.frame_scores(counts)


def evaluate_salience_grid(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    references: Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]],
    settings: Sequence[Dict[str, Any]],
    kind: str = "contour",
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    window: float = evaluate.WINDOW,
):
    """Frame-level multi-pitch scores of the model's contour (or note) posteriorgram read as a multi-f0 estimate, for a
    batch of annotated recordings under every setting of a grid (addition; no reference counterpart): the model runs
    once over the batch, and every (setting, file) is scored on the device in one `bp_score_salience_grid_host` call.
    `audio` as in `evaluate_grid`; `references` as in `evaluate_frames_grid`; a setting is a dict {threshold,
    peak_picking=True, minimum_frequency=None, maximum_frequency=None} (`Model.score_salience_grid`); window in
    semitones.

    Returns (counts (n_settings, n_files, 7), `evaluate.frame_scores(counts)`)."""
    if kind not in ("contour", "note"):
        raise ValueError(f"kind must be 'contour' or 'note', got {kind!r}")
    model, clips = _model_and_clips(audio, model_or_model_path)
    outs = model.run_inference_arrays(clips)
    counts = model.score_salience_grid([o[kind] for o in outs], settings, references, kind=kind, window=window)
    return counts, evaluate.frame_scores(counts)


def evaluate_melody_grid(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    references: Sequence[Tuple[np.ndarray, np.ndarray]],
    settings: Sequence[Dict[str, Any]],
    kind: str = "contour",
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    cent_tolerance: float = evaluate.CENT_TOLERANCE,
):
    """mir_eval.melody's scores of the model's contour (or note) posteriorgram read as a single-f0 estimate, for a batch
    of f0-annotated recordings under every setting of a grid (addition; no reference counterpart): the model runs once
    over the batch, and every (setting, file) is scored on the device in one `bp_score_melody_grid_host` call.  `audio`
    as in `evaluate_grid`; `references[i]` is file i's (times (n,) in seconds, f0 (n,) in Hz, 0 or negative where
    unvoiced), mir_eval.melody's convention; a setting is a dict {threshold, minimum_frequency=None,
    maximum_frequency=None, guess_unvoiced=True} (`Model.score_melody_grid`); cent_tolerance in cents.

    Returns (counts (n_settings, n_files, 7), `evaluate.melody_scores(counts)`)."""
    if kind not in ("contour", "note"):
        raise ValueError(f"kind must be 'contour' or 'note', got {kind!r}")
    model, clips = _model_and_clips(audio, model_or_model_path)
    outs = model.run_inference_arrays(clips)
    counts = model.score_melody_grid([o[kind] for o in outs], settings, references, kind=kind,
                                     cent_tolerance=cent_tolerance)
    return counts, evaluate.melody_scores(counts)


def evaluate_note_melody_grid(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    references: Sequence[Tuple[np.ndarray, np.ndarray]],
    settings: Sequence[Dict[str, Any]],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    pitch_bends: bool = True,
    cent_tolerance: float = evaluate.CENT_TOLERANCE,
):
    """mir_eval.melody's scores of the decoded notes read as a single-f0 track (`evaluate.note_frames_to_melody`: per
    frame the sounding pitch with the largest note posteriorgram value, with its pitch bend when pitch_bends), for a
    batch of f0-annotated recordings under every setting of a grid (addition; no reference counterpart): the model runs
    once over the batch, and every (setting, file) is decoded and scored on the device in one
    `bp_score_note_melody_grid_host` call.  `audio` and `settings` as in `evaluate_grid`; `references[i]` is file i's
    (times (n,) in seconds, f0 (n,) in Hz, 0 or negative where unvoiced), mir_eval.melody's convention; cent_tolerance in
    cents.

    Returns (counts (n_settings, n_files, 7), `evaluate.melody_scores(counts)`)."""
    model, clips = _model_and_clips(audio, model_or_model_path)
    decode = [{**infer.grid_setting(s, predict_names=True)[0], "include_pitch_bends": bool(pitch_bends)} for s in settings]
    outs = model.run_inference_arrays(clips)
    counts = model.score_note_melody_grid([o["note"] for o in outs], [o["onset"] for o in outs],
                                          [o["contour"] for o in outs] if pitch_bends else None, decode, references,
                                          cent_tolerance=cent_tolerance)
    return counts, evaluate.melody_scores(counts)


EVALUATE_FAMILIES = ("notes", "transcription", "velocity", "frames", "bent_frames", "note_melody", "flat_note_melody",
                     "salience", "melody")


def evaluate_all(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    settings: Sequence[Dict[str, Any]],
    notes: Optional[Sequence[Tuple[np.ndarray, ...]]] = None,
    multipitch: Optional[Sequence[Tuple[np.ndarray, Sequence[np.ndarray]]]] = None,
    f0: Optional[Sequence[Tuple[np.ndarray, np.ndarray]]] = None,
    salience: Optional[Dict[str, Any]] = None,
    melody: Optional[Dict[str, Any]] = None,
    families: Optional[Sequence[str]] = None,
    return_model_output: bool = False,
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    window: float = evaluate.WINDOW,
    cent_tolerance: float = evaluate.CENT_TOLERANCE,
    velocity_tolerance: float = 0.1,
    **tolerances,
):
    """Several metric families of a batch of annotated recordings under one grid of settings, in one device pass
    (addition; no reference counterpart): the batch is ingested and run through the model once, its posteriorgrams stay
    on the device, each chunk of settings is decoded once and every note-derived family scores that decode
    (`Model.evaluate`, `bp_evaluate_*`).  Items follow `predict_batch`: with any path the batch goes through the
    stored-PCM pipeline, otherwise the packed arrays.

    A family stands for one existing call, and its value equals that call's return value bit for bit:
      notes            evaluate_grid(audio, notes, settings)
      transcription    evaluate_transcription_grid(audio, notes, settings)
      velocity         evaluate_velocity_grid(audio, notes, settings, velocity_tolerance=...); notes with velocities
      frames           evaluate_frames_grid(audio, multipitch, settings, pitch_bends=False)
      bent_frames      evaluate_frames_grid(audio, multipitch, settings, pitch_bends=True)
      note_melody      evaluate_note_melody_grid(audio, f0, settings, pitch_bends=True)
      flat_note_melody evaluate_note_melody_grid(audio, f0, settings, pitch_bends=False)
      salience         evaluate_salience_grid(audio, refs, salience["settings"], kind=salience.get("kind", "contour"))
      melody           evaluate_melody_grid(audio, refs, melody["settings"], kind=melody.get("kind", "contour"))
    with the tolerances given here (window, cent_tolerance, note tolerances as `evaluate.TOLERANCES`).  salience /
    melody are dicts {settings, kind="contour", references}; their references default to `multipitch` / `f0`.
    families=None selects every family whose references are given (velocity when the note references carry
    velocities).  Returns {family: (counts, scores)}, plus "model_output" (per-file posteriorgram dicts) when asked."""
    salience = None if salience is None else {"references": multipitch, **salience}
    melody = None if melody is None else {"references": f0, **melody}
    if families is None:
        families = [f for f, given in (
            ("notes", notes), ("transcription", notes), ("velocity", notes and all(len(r) == 3 for r in notes)),
            ("frames", multipitch), ("bent_frames", multipitch), ("note_melody", f0), ("flat_note_melody", f0),
            ("salience", salience and salience.get("references")), ("melody", melody and melody.get("references")),
        ) if given is not None and given is not False]  # fmt: skip
    unknown = set(families) - set(EVALUATE_FAMILIES)
    if unknown:
        raise ValueError(f"unknown famil(ies) {sorted(unknown)}; choose from {EVALUATE_FAMILIES}")
    fam = set(families)
    refs = _velocity_references(notes) if "velocity" in fam else None
    lib_fams = [f for f in ("notes", "frames", "bent_frames", "note_melody", "flat_note_melody", "salience", "melody")
                if f in fam]
    if "transcription" in fam:
        lib_fams.append("onset_offset")
    if fam & {"transcription", "velocity"}:
        lib_fams.append("pairs")
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    decode = [infer.grid_setting(s, predict_names=True)[0] for s in settings]  # include_pitch_bends: predict's True
    request = dict(note_refs=notes, multipitch_refs=multipitch, f0_refs=f0, salience=salience, melody=melody,
                   window=window, cent_tolerance=cent_tolerance, **tolerances)
    if all(isinstance(a, np.ndarray) for a in audio):
        for a in audio:
            if a.ndim != 1:
                raise ValueError("audio must be mono (1-D)")
        out = model.evaluate(lib_fams, decode, audio=[np.ascontiguousarray(a, dtype=_F32) for a in audio],
                             return_model_output=return_model_output, **request)
    else:
        out = model.evaluate(lib_fams, decode, pcm=_pcm_items(audio), return_model_output=return_model_output, **request)
    n_frames = np.diff(out["frame_off"]).tolist()
    result: Dict[str, Any] = {}
    if "notes" in fam:
        result["notes"] = (out["notes"], evaluate.note_scores(out["notes"]))
    if "transcription" in fam:
        ref_ivs = [np.asarray(r[0], np.float64).reshape(-1, 2) for r in notes]
        result["transcription"] = _transcription_scores(n_frames, ref_ivs, *out["pairs"], out["onset_offset"])
    if "velocity" in fam:
        result["velocity"] = _velocity_scores(n_frames, refs, *out["pairs"], velocity_tolerance)
    for f in ("frames", "bent_frames", "salience"):
        if f in fam:
            result[f] = (out[f], evaluate.frame_scores(out[f]))
    for f in ("note_melody", "flat_note_melody", "melody"):
        if f in fam:
            result[f] = (out[f], evaluate.melody_scores(out[f]))
    if return_model_output:
        result["model_output"] = out["model_output"]
    return result


def _pcm_items(audio: Sequence[Union[np.ndarray, pathlib.Path, str]], wav_in_library: bool = True) -> List[Any]:
    """A batch of paths and arrays as the items of one `Model.transcribe_pcm` / `Model.evaluate(pcm=...)` call: files go
    to the device as the samples they store, arrays beside them as float32 mono at 22 050 Hz, which the ingest copies
    bit for bit.  With wav_in_library every path is probed (`audio_io.probe_wav`): an accepted WAV file becomes a
    `WavRegion`, which the library reads itself; a declined one, and every path without wav_in_library, is read by
    `read_pcm` as always, with its result or exception."""
    paths = [i for i, a in enumerate(audio) if not isinstance(a, np.ndarray)]
    found = probe_wav([audio[i] for i in paths])[0] if wav_in_library else [None] * len(paths)
    regions = dict(zip(paths, found))
    items: List[Any] = []
    for i, a in enumerate(audio):
        if isinstance(a, np.ndarray):
            if a.ndim != 1:
                raise ValueError("audio must be mono (1-D)")
            items.append((np.ascontiguousarray(a, dtype=_F32), AUDIO_SAMPLE_RATE))
        else:
            items.append(regions[i] if regions[i] is not None else read_pcm(a))
    return items


def predict_batch(
    audio: Sequence[Union[np.ndarray, pathlib.Path, str]],
    model_or_model_path: Union[Model, pathlib.Path, str] = ICASSP_2022_MODEL_PATH,
    onset_threshold: float = DEFAULT_ONSET_THRESHOLD,
    frame_threshold: float = DEFAULT_FRAME_THRESHOLD,
    minimum_note_length: float = DEFAULT_MINIMUM_NOTE_LENGTH_MS,
    minimum_frequency: Optional[float] = None,
    maximum_frequency: Optional[float] = None,
    multiple_pitch_bends: bool = False,
    melodia_trick: bool = True,
    midi_tempo: float = DEFAULT_MINIMUM_MIDI_TEMPO,
    return_model_output: bool = True,
    build_midi: bool = True,
    lazy: bool = True,
    wav_in_library: bool = False,
):
    """`predict` for many clips in one device pass (addition; no reference counterpart).

    Items are paths or mono 22 050 Hz float arrays.  With a path among them the batch goes through
    `Model.transcribe_pcm`: the files cross to the device once, as the samples they store, and are converted, down-mixed
    and resampled there.  The files are read by `read_pcm` on this thread (`bp_transcribe_pcm_files_host`); with
    wav_in_library=True (what `predict_and_save` and the CLI use) WAV files the header probe accepts
    (`audio_io.probe_wav`) are read by the library's gather threads straight into pinned staging, 24-bit and float64
    ones as stored (`bp_transcribe_pcm_sources_host`), and only declined files by `read_pcm`.  The results are the same
    bit for bit, in one library call either way.  Returns a list of
    (model_output | None, midi_data | None, note_events) in input order.  The model outputs are views of three
    page-locked arrays shared by the batch.  With lazy=True (default) the note events are `NoteEventList`s and the MIDI
    objects `LazyPrettyMIDI`s: both turn into the reference's Python objects when first read; lazy=False builds
    everything before returning."""
    model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
    min_note_len = int(np.round(minimum_note_length / 1000 * (AUDIO_SAMPLE_RATE / FFT_HOP)))
    lo, hi = infer.frequency_to_column_range(minimum_frequency, maximum_frequency)
    decode = dict(onset_thresh=onset_threshold, frame_thresh=frame_threshold, min_note_len=min_note_len,
                  melodia_trick=melodia_trick, min_pitch_idx=lo, max_pitch_idx=hi, return_model_output=return_model_output,
                  split_notes=False)
    if all(isinstance(a, np.ndarray) for a in audio):
        outs, arrs, frames = model.transcribe_arrays(audio, **decode)
    else:
        outs, arrs, frames = model.transcribe_pcm(_pcm_items(audio, wav_in_library), **decode)
    n = len(audio)
    events = infer.note_events_batch(arrs, n, include_pitch_bends=True, lazy=lazy)
    if return_model_output and (minimum_frequency is not None or maximum_frequency is not None):
        # the reference zeroes these columns of the returned arrays (note_creation.py:338-341); all files share two arrays
        flo, fhi = infer.frequency_to_column_range(minimum_frequency, maximum_frequency)
        for k in ("note", "onset"):
            whole = outs[0][k].base if n and outs[0][k].base is not None else None
            for m in ([whole] if isinstance(whole, np.ndarray) and whole.ndim == 2 else [o[k] for o in outs]):
                m[:, :flo] = 0
                m[:, fhi:] = 0
    midis = [infer.LazyPrettyMIDI(ev, multiple_pitch_bends, midi_tempo) if build_midi else None for ev in events]
    if build_midi and not lazy:
        for m in midis:
            m.instruments  # assemble the Instrument / Note / PitchBend objects now
    return list(zip(outs, midis, events))


def predict_and_save(
    audio_path_list: Sequence[Union[pathlib.Path, str]],
    output_directory: Union[pathlib.Path, str],
    save_midi: bool,
    sonify_midi: bool,
    save_model_outputs: bool,
    save_notes: bool,
    model_or_model_path: Union[Model, str, pathlib.Path],
    onset_threshold: float = DEFAULT_ONSET_THRESHOLD,
    frame_threshold: float = DEFAULT_FRAME_THRESHOLD,
    minimum_note_length: float = DEFAULT_MINIMUM_NOTE_LENGTH_MS,
    minimum_frequency: Optional[float] = None,
    maximum_frequency: Optional[float] = None,
    multiple_pitch_bends: bool = False,
    melodia_trick: bool = True,
    debug_file: Optional[pathlib.Path] = None,
    sonification_samplerate: int = DEFAULT_SONIFICATION_SAMPLERATE,
    midi_tempo: float = DEFAULT_MINIMUM_MIDI_TEMPO,
) -> None:
    """reference: inference.py:509-604 — same files, names and failure behaviour (print, then re-raise).

    Several files without `debug_file` go through the batch path: one device pass per `BATCH_FILES` files
    (`predict_batch(wav_in_library=True)`: GPU ingest, one library call, WAV files read by the library), one
    `bp_write_note_files` call for their MIDI / CSV files
    (csrc/writers.cu) and, for `sonify_midi` with the bundled MIDI stand-in, one `bp_sonify_notes_host` call for their
    WAV samples (csrc/sonify.cu) instead of a Python loop over files and notes."""

    def _saved(kind: str, path) -> None:
        print(f"  ✅ Saved {kind.lower().replace('_', ' ')} to {path}")

    def _failed(kind: str, path) -> None:
        print(f"\n🚨 Failed to save {kind.lower().replace('_', ' ')} to {path} \n")

    paths = list(audio_path_list)
    if len(paths) > 1 and debug_file is None:
        from scipy.io import wavfile

        from . import midi as bundled_midi

        model = model_or_model_path if isinstance(model_or_model_path, Model) else default_model(model_or_model_path)
        BATCH_FILES = 64
        for c0 in range(0, len(paths), BATCH_FILES):
            chunk = paths[c0 : c0 + BATCH_FILES]
            for q in chunk:
                print(f"\nPredicting MIDI for {q}...")
            results = predict_batch([pathlib.Path(q) for q in chunk], model, onset_threshold, frame_threshold, minimum_note_length,
                                    minimum_frequency, maximum_frequency, multiple_pitch_bends, melodia_trick, midi_tempo,
                                    wav_in_library=True)
            # the GPU renders the bundled stand-in's synthesiser; with the real pretty_midi installed, its own synthesiser
            # makes the file, one by one
            gpu_sonify = sonify_midi and infer.pretty_midi is bundled_midi
            sonified: Optional[List[np.ndarray]] = None
            midi_paths: List[Optional[pathlib.Path]] = [None] * len(chunk)
            csv_paths: List[Optional[pathlib.Path]] = [None] * len(chunk)
            for i, (audio_path, (model_output, midi_data, _events)) in enumerate(zip(chunk, results)):
                if save_model_outputs:
                    path = build_output_path(audio_path, output_directory, OutputExtensions.MODEL_OUTPUT_NPZ)
                    try:
                        np.savez(path, basic_pitch_model_output=model_output)
                        _saved(OutputExtensions.MODEL_OUTPUT_NPZ.name, path)
                    except Exception:
                        _failed(OutputExtensions.MODEL_OUTPUT_NPZ.name, path)
                        raise
                if save_midi:
                    midi_paths[i] = build_output_path(audio_path, output_directory, OutputExtensions.MIDI)
                if sonify_midi:
                    path = build_output_path(audio_path, output_directory, OutputExtensions.MIDI_SONIFICATION)
                    try:
                        if gpu_sonify:  # the whole chunk rendered in one library call, when the first file needs it
                            if sonified is None:
                                sonified = infer.sonify_batch([r[2] for r in results], sonification_samplerate,
                                                              multiple_pitch_bends, model)
                            wavfile.write(path, sonification_samplerate, sonified[i])
                        else:
                            infer.sonify_midi(midi_data, path, sr=sonification_samplerate)
                        _saved(OutputExtensions.MIDI_SONIFICATION.name, path)
                    except Exception:
                        _failed(OutputExtensions.MIDI_SONIFICATION.name, path)
                        raise
                if save_notes:
                    csv_paths[i] = build_output_path(audio_path, output_directory, OutputExtensions.NOTE_EVENTS)
            if save_midi or save_notes:
                try:
                    infer.write_note_files([r[2] for r in results], midi_paths if save_midi else None,
                                           csv_paths if save_notes else None, multiple_pitch_bends, midi_tempo)
                except Exception:
                    for kind, plist in ((OutputExtensions.MIDI, midi_paths), (OutputExtensions.NOTE_EVENTS, csv_paths)):
                        for path in plist:
                            if path is not None and not path.exists():
                                _failed(kind.name, path)
                    raise
                for mp, cp in zip(midi_paths, csv_paths):
                    if mp is not None:
                        _saved(OutputExtensions.MIDI.name, mp)
                    if cp is not None:
                        _saved(OutputExtensions.NOTE_EVENTS.name, cp)
        return

    for audio_path in audio_path_list:
        print("")
        model_output, midi_data, note_events = predict(
            pathlib.Path(audio_path), model_or_model_path, onset_threshold, frame_threshold, minimum_note_length,
            minimum_frequency, maximum_frequency, multiple_pitch_bends, melodia_trick, debug_file, midi_tempo,
        )
        if save_model_outputs:
            path = build_output_path(audio_path, output_directory, OutputExtensions.MODEL_OUTPUT_NPZ)
            try:
                np.savez(path, basic_pitch_model_output=model_output)
                _saved(OutputExtensions.MODEL_OUTPUT_NPZ.name, path)
            except Exception:
                _failed(OutputExtensions.MODEL_OUTPUT_NPZ.name, path)
                raise
        if save_midi:
            path = build_output_path(audio_path, output_directory, OutputExtensions.MIDI)
            try:
                midi_data.write(str(path))
                _saved(OutputExtensions.MIDI.name, path)
            except Exception:
                _failed(OutputExtensions.MIDI.name, path)
                raise
        if sonify_midi:
            path = build_output_path(audio_path, output_directory, OutputExtensions.MIDI_SONIFICATION)
            try:
                infer.sonify_midi(midi_data, path, sr=sonification_samplerate)
                _saved(OutputExtensions.MIDI_SONIFICATION.name, path)
            except Exception:
                _failed(OutputExtensions.MIDI_SONIFICATION.name, path)
                raise
        if save_notes:
            path = build_output_path(audio_path, output_directory, OutputExtensions.NOTE_EVENTS)
            try:
                save_note_events(note_events, path)
                _saved(OutputExtensions.NOTE_EVENTS.name, path)
            except Exception:
                _failed(OutputExtensions.NOTE_EVENTS.name, path)
                raise
