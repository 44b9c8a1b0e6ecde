"""Audio file -> mono float32 at 22 050 Hz, in front of the hot path: `load_audio` on the host (NumPy / SciPy),
`load_audio_device` with the conversion, down-mix and resampling on the GPU (csrc/ingest.cu, same filter); `read_pcm` +
`pcm_descriptors` hand the stored samples of a whole batch of files to the batched ingest (`Model.transcribe_pcm`), and
`probe_wav` finds the WAV files whose samples the library reads itself (`WavRegion`).

Stands in for `librosa.load(path, sr=22050, mono=True)` (reference: basic_pitch/inference.py:239).
WAV files are decoded with scipy; other containers need `soundfile` (optional).  Files that are not
already at 22 050 Hz are resampled with a Kaiser-windowed polyphase FIR (pass band 0.913·Nyquist,
125 dB stop band — the shape of soxr's HQ preset, which is what librosa uses by default).  The
resampler is NOT parity-pinned against librosa/soxr (neither is available offline); on the reference's
44.1 kHz test clip it reproduces the golden posteriorgrams to 2e-4 (tests/golden/README.md).
"""
from __future__ import annotations

import os
import pathlib
from dataclasses import dataclass
from math import gcd
from typing import List, Optional, Sequence, Tuple, Union

import ctypes as C

import numpy as np

from .constants import AUDIO_SAMPLE_RATE


def _to_float32(x: np.ndarray) -> np.ndarray:
    if x.dtype.kind == "f":
        return x.astype(np.float32)
    if x.dtype.kind == "i":
        return x.astype(np.float32) / np.float32(2 ** (8 * x.dtype.itemsize - 1))
    if x.dtype.kind == "u":  # 8-bit WAV is unsigned
        return (x.astype(np.float32) - 128.0) / 128.0
    raise ValueError(f"unsupported sample dtype {x.dtype}")


_FILTERS = {}


def _resample_filter(up: int, down: int) -> np.ndarray:
    key = (up, down)
    if key not in _FILTERS:
        import scipy.signal

        m = max(up, down)
        pass_edge, stop_edge = 0.913 / m, 1.0 / m
        numtaps, beta = scipy.signal.kaiserord(125.0, stop_edge - pass_edge)
        numtaps |= 1
        _FILTERS[key] = scipy.signal.firwin(numtaps, 0.5 * (pass_edge + stop_edge), window=("kaiser", beta))
    return _FILTERS[key]


def resample(x: np.ndarray, sr_in: int, sr_out: int = AUDIO_SAMPLE_RATE) -> np.ndarray:
    if sr_in == sr_out:
        return x.astype(np.float32)
    import scipy.signal

    g = gcd(int(sr_in), int(sr_out))
    up, down = int(sr_out) // g, int(sr_in) // g
    y = scipy.signal.resample_poly(x.astype(np.float64), up, down, window=_resample_filter(up, down))
    return y.astype(np.float32)


_PCM_FORMATS = {np.dtype(np.float32): 0, np.dtype(np.int16): 1, np.dtype(np.int32): 2, np.dtype(np.uint8): 3}


def read_pcm(path: Union[str, pathlib.Path]) -> Tuple[np.ndarray, int]:
    """Decode a file to its stored samples — (n,) or (n, channels) in one of the dtypes the device ingest converts
    itself (float32, int16, int32, uint8) — plus the sample rate."""
    try:
        from scipy.io import wavfile

        sr, x = wavfile.read(str(path))
        x = np.asarray(x)
        if x.dtype not in _PCM_FORMATS:  # e.g. float64 WAV
            x = _to_float32(x)
        return x, int(sr)
    except Exception:
        x, sr = read_audio(path)
        return x, sr


def pcm_descriptors(items: Sequence[Tuple[np.ndarray, int]]):
    """Stored samples of a batch of files -> the `bp_pcm_file_t` array the batched ingest takes (`bp_load_pcm_files_device`,
    `bp_transcribe_pcm_files_host`) plus the arrays it points into, which the caller keeps alive for the call.  An item is
    (samples, sample_rate) as `read_pcm` returns them: (n,) or (n, channels) float32 / int16 / int32 / uint8; samples
    that are not C-contiguous are copied.  The library packs the PCM itself, sub-batch by sub-batch."""
    from . import _lib

    keep = []
    files = (_lib.PcmFile * max(len(items), 1))()
    for f, (x, sr) in zip(files, items):
        x = np.asarray(x)
        if x.dtype not in _PCM_FORMATS:
            raise ValueError(f"unsupported sample dtype {x.dtype}: the device ingest takes float32, int16, int32 and uint8")
        if x.ndim not in (1, 2):
            raise ValueError(f"samples must be (n,) or (n, channels), got shape {x.shape}")
        x = np.ascontiguousarray(x)
        keep.append(x)
        f.pcm = x.ctypes.data if x.size else None
        f.n_frames, f.channels = (x.shape[0], 1) if x.ndim == 1 else x.shape
        f.sample_format, f.sample_rate = _PCM_FORMATS[x.dtype], int(sr)
    return files, keep


@dataclass(frozen=True)
class WavRegion:
    """The samples of a WAV file as `probe_wav` found them: bytes [data_offset, data_offset + n_frames x channels x
    bytes per sample) of `path`, interleaved, in library format `sample_format` (0 float32, 1 int16, 2 int32, 3 uint8,
    4 packed 24-bit, 5 float64).  An item of `Model.transcribe_pcm` / `Model.evaluate(pcm=...)` beside
    (samples, sample_rate) pairs: the library reads the bytes itself, and they cross PCIe as stored."""

    path: str
    data_offset: int
    n_frames: int
    sample_format: int
    channels: int
    sample_rate: int


def probe_wav(paths: Sequence[Union[str, pathlib.Path]]) -> Tuple[List[Optional[WavRegion]], List[int]]:
    """The WAV headers of `paths`, read by the library (`bp_probe_wav_files`, no GPU): (regions, declined), regions[i]
    the `WavRegion` of an accepted file and None for a declined one, whose indices `declined` lists.  A file is accepted
    only when its reading is unambiguous and equals `scipy.io.wavfile.read`'s (include/bp_b200.h); a declined file is
    for `read_pcm`, which gives it the result or the exception it always did."""
    from . import _lib

    lib = _lib.load()
    names = [os.fsencode(p) for p in paths]
    n = len(names)
    arg = (C.c_char_p * max(n, 1))(*names)
    out = (_lib.PcmSource * max(n, 1))()
    accepted = np.zeros(max(n, 1), np.int32)
    lib.bp_probe_wav_files(arg, n, out, accepted.ctypes.data)
    regions: List[Optional[WavRegion]] = []
    for i in range(n):
        s = out[i]
        regions.append(WavRegion(os.fsdecode(names[i]), int(s.data_offset), int(s.pcm.n_frames), int(s.pcm.sample_format),
                                 int(s.pcm.channels), int(s.pcm.sample_rate)) if accepted[i] else None)
    return regions, [i for i in range(n) if not accepted[i]]


def pcm_sources(items: Sequence[Union[Tuple[np.ndarray, int], WavRegion]]):
    """`pcm_descriptors` for batches that may hold `WavRegion`s: the `bp_pcm_source_t` array of
    `bp_transcribe_pcm_sources_host` / `bp_evaluate_pcm_sources_host` plus what it points into (kept by the caller for
    the call).  (samples, sample_rate) items are described as `pcm_descriptors` describes them."""
    from . import _lib

    n = len(items)
    sources = (_lib.PcmSource * max(n, 1))()
    arrays = [it for it in items if not isinstance(it, WavRegion)]
    files, keep = pcm_descriptors(arrays)
    keep = list(keep)
    k = 0
    for s, it in zip(sources, items):
        if isinstance(it, WavRegion):
            name = os.fsencode(it.path)
            keep.append(name)
            s.path, s.data_offset = name, it.data_offset
            s.pcm.pcm = None
            s.pcm.n_frames, s.pcm.sample_format = it.n_frames, it.sample_format
            s.pcm.channels, s.pcm.sample_rate = it.channels, it.sample_rate
        else:
            s.pcm = files[k]
            k += 1
    return sources, keep


def load_audio_device(path: Union[str, pathlib.Path], model) -> Tuple[np.ndarray, int]:
    """`load_audio(path, 22050, mono=True)` with the sample conversion, down-mix and resampling done on the GPU
    (csrc/ingest.cu through `bp_load_pcm_host`): the file crosses PCIe as the PCM it was stored as."""
    x, file_sr = read_pcm(path)
    x = np.ascontiguousarray(x)
    n, ch = (x.shape[0], 1) if x.ndim == 1 else x.shape
    lib = model._lib
    out = np.empty(int(lib.bp_resampled_length(n, file_sr)), np.float32)
    lib.bp_load_pcm_host(model.handle, x.ctypes.data, _PCM_FORMATS[x.dtype], n, ch, file_sr, out.ctypes.data)
    return out, AUDIO_SAMPLE_RATE


def read_audio(path: Union[str, pathlib.Path]) -> Tuple[np.ndarray, int]:
    """Decode to float32 (n,) or (n, channels) plus the file's sample rate."""
    path = str(path)
    try:
        from scipy.io import wavfile

        sr, x = wavfile.read(path)
        return _to_float32(np.asarray(x)), int(sr)
    except Exception as wav_err:  # not a WAV scipy can read
        try:
            import soundfile  # type: ignore

            x, sr = soundfile.read(path, dtype="float32", always_2d=False)
            return np.asarray(x, dtype=np.float32), int(sr)
        except ImportError:
            raise ValueError(
                f"cannot decode {path}: scipy.io.wavfile failed ({wav_err}) and `soundfile` is not installed; "
                "convert the file to WAV"
            ) from wav_err


def load_audio(path: Union[str, pathlib.Path], sr: int = AUDIO_SAMPLE_RATE, mono: bool = True) -> Tuple[np.ndarray, int]:
    x, file_sr = read_audio(path)
    if x.ndim == 2 and mono:
        x = x.mean(axis=1, dtype=np.float32)
    x = resample(x, file_sr, sr)
    return np.ascontiguousarray(x, dtype=np.float32), sr
