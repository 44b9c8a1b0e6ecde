#!/usr/bin/env python
"""Where the time goes when a batch of audio FILES is transcribed: the input side of `predict_batch` /
`predict_and_save`, measured without the output side (no MIDI objects, no files written).

Workload: N seeded `random_notes_clip` clips written to a temporary directory as WAV files at a chosen rate, sample
format and channel count (default 64 x 10 s, 44.1 kHz, int16, stereo; int24 writes packed 24-bit PCM).  Three sequences
are timed in the same process, alternating, each leg ending in a device synchronise:

  per_file  `audio_io.load_audio_device` per file (one upload, one ingest launch and one download each), then
            `Model.transcribe_arrays` on the 22 050 Hz signals (a second upload);
  batched   `audio_io.read_pcm` per file, then `Model.transcribe_pcm` (one library call: the stored PCM goes up once,
            one batched ingest per sub-batch, the forward pass reads its output on the device);
  library   `audio_io.probe_wav` on all files (headers only), then `Model.transcribe_pcm` on the regions it returns: the
            library's gather threads read the samples straight into pinned staging (`bp_transcribe_pcm_sources_host`),

and within `batched` / `library` the host split: reading the files (or their headers) against the library call.  Every
sequence reads the same files, so all read from a warm page cache after the first round.  `batched` and `library` must
return bit-identical posteriorgrams and notes (asserted).  Prints one JSON line with the medians, the spread of each
sequence, audio-seconds per second, and the device name and power limit read in the same run.  Needs a GPU: there is
nothing to fall back to."""
import argparse
import json
import os
import pathlib
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = pathlib.Path(__file__).resolve().parent.parent

FORMATS = {"int16": np.int16, "int32": np.int32, "uint8": np.uint8, "float32": np.float32, "int24": "int24"}


def write_wav24(path, rate, pcm):
    """A 24-bit PCM WAV of int32 samples (n, channels) in [-2^23, 2^23) (scipy.io.wavfile cannot write one)."""
    import struct

    data = pcm.astype("<i4").reshape(-1).view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    ch = pcm.shape[1]
    fmt = struct.pack("<HHIIHH", 1, ch, rate, rate * ch * 3, ch * 3, 24)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(data)) + data
    pathlib.Path(path).write_bytes(b"RIFF" + struct.pack("<I", len(body)) + body + b"\0" * (len(data) % 2))


def device_info():
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("file_path_profile: no CUDA device; this measurement only exists on the GPU")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"device": torch.cuda.get_device_name(0), "power_limit": power}


def write_clips(directory, n_clips, seconds, rate, dtype, channels):
    from scipy import signal
    from scipy.io import wavfile

    from basic_pitch_b200 import synth

    paths = []
    for i in range(n_clips):
        x = synth.random_notes_clip(seconds, seed=7000 + i).astype(np.float64)
        if rate != 22050:
            x = signal.resample_poly(x, rate, 22050)
        x = np.clip(x, -1.0, 1.0)
        cols = np.stack([x * (1.0 - 0.1 * c) for c in range(channels)], 1)
        paths.append(os.path.join(directory, f"clip{i:03d}.wav"))
        if dtype == "int24":
            write_wav24(paths[-1], rate, np.round(cols * 0.9 * (2**23 - 1)).astype(np.int32))
            continue
        if dtype == np.uint8:
            pcm = np.round(cols * 120 + 128).astype(dtype)
        elif np.dtype(dtype).kind == "i":
            pcm = np.round(cols * 0.9 * np.iinfo(dtype).max).astype(dtype)
        else:
            pcm = cols.astype(dtype)
        wavfile.write(paths[-1], rate, pcm[:, 0] if channels == 1 else pcm)
    return paths


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--rate", type=int, default=44100)
    ap.add_argument("--format", choices=sorted(FORMATS), default="int16")
    ap.add_argument("--channels", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    sys.path.insert(0, str(HERE))
    out = device_info()
    import torch

    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, audio_io
    from basic_pitch_b200.inference import Model

    model = Model(ICASSP_2022_MODEL_PATH)
    kw = dict(return_model_output=True, split_notes=False)

    def sync():
        torch.cuda.synchronize(model.device)

    with tempfile.TemporaryDirectory() as tmp:
        paths = write_clips(tmp, args.clips, args.seconds, args.rate, FORMATS[args.format], args.channels)
        file_bytes = sum(os.path.getsize(p) for p in paths)

        def per_file():
            t0 = time.perf_counter()
            audios = [audio_io.load_audio_device(p, model)[0] for p in paths]
            sync()
            t1 = time.perf_counter()
            _outs, arrs, _frames = model.transcribe_arrays(audios, **kw)
            sync()
            return {"load_audio_device": t1 - t0, "transcribe_arrays": time.perf_counter() - t1}, arrs

        def batched():
            t0 = time.perf_counter()
            items = [audio_io.read_pcm(p) for p in paths]
            t1 = time.perf_counter()
            _outs, arrs, _frames = model.transcribe_pcm(items, **kw)
            sync()
            return {"read_pcm": t1 - t0, "transcribe_pcm": time.perf_counter() - t1}, (outs, arrs)

        def library():
            t0 = time.perf_counter()
            regions, declined = audio_io.probe_wav(paths)
            assert not declined
            t1 = time.perf_counter()
            outs, arrs, _frames = model.transcribe_pcm(regions, **kw)
            sync()
            return {"probe_wav": t1 - t0, "transcribe_pcm": time.perf_counter() - t1}, (outs, arrs)

        def batched():
            t0 = time.perf_counter()
            items = [audio_io.read_pcm(p) for p in paths]
            t1 = time.perf_counter()
            outs, arrs, _frames = model.transcribe_pcm(items, **kw)
            sync()
            return {"read_pcm": t1 - t0, "transcribe_pcm": time.perf_counter() - t1}, (outs, arrs)

        def snapshot(res):  # the page-locked outputs are reused by the next call
            outs, arrs = res
            grams = {k: np.concatenate([o[k] for o in outs]).view(np.uint32).copy() for k in ("note", "onset", "contour")}
            n_notes = int(arrs["note_off"][args.clips])
            used = {"note_off": args.clips + 1, "bend_off": n_notes + 1, "bends": int(arrs["bend_off"][n_notes])}
            return grams, {k: np.asarray(v)[: used.get(k, n_notes)].copy() for k, v in arrs.items()}

        legs = {"per_file": per_file, "batched": batched, "library": library}
        times = {name: [] for name in legs}
        notes, first = {}, {}
        for r in range(args.warmup + args.rounds):
            for name, fn in legs.items():
                t, res = fn()
                arrs = res if name == "per_file" else res[1]
                notes[name] = int(arrs["note_off"][args.clips])
                if name != "per_file" and name not in first:
                    first[name] = snapshot(res)
                if r >= args.warmup:
                    times[name].append(t)
        assert notes["per_file"] == notes["batched"] == notes["library"] > 0, notes  # the same notes on every route
        (gb, ab), (gl, al) = first["batched"], first["library"]
        identical = all(np.array_equal(gb[k], gl[k]) for k in gb) and all(
            np.array_equal(ab[k].view(np.uint8), al[k].view(np.uint8)) for k in ab)
        assert identical, "the library route must return read_pcm's posteriorgrams and notes bit for bit"

    audio_s = args.clips * args.seconds
    out.update({"clips": args.clips, "clip_seconds": args.seconds, "rate": args.rate, "format": args.format,
                "channels": args.channels, "file_mbytes": file_bytes / 1e6, "rounds": args.rounds, "notes": notes["batched"],
                "page_cache": "warm (every sequence reads the same files, round after round)",
                "library_equals_batched_bitwise": identical})
    for name, rows in times.items():
        total = [sum(t.values()) for t in rows]
        for leg in rows[0]:  # (per leg, over the rounds)
            out[f"{name}.{leg}_ms"] = 1e3 * float(np.median([t[leg] for t in rows]))
        out[f"{name}_ms"] = 1e3 * float(np.median(total))
        out[f"{name}_ms_min_max"] = [1e3 * min(total), 1e3 * max(total)]
        out[f"{name}_audio_s_per_s"] = audio_s / float(np.median(total))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
