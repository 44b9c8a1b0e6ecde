#!/usr/bin/env python
"""Where the time goes when a batch of audio FILES is transcribed: the input side of `predict_batch` /
`predict_and_save`, measured without the output side (no MIDI objects, no files written).

Workload: N seeded `random_notes_clip` clips written to a temporary directory as WAV files at a chosen rate, sample
format and channel count (default 64 x 10 s, 44.1 kHz, int16, stereo).  Two sequences are timed in the same process,
alternating, each leg ending in a device synchronise:

  per_file  `audio_io.load_audio_device` per file (one upload, one ingest launch and one download each), then
            `Model.transcribe_arrays` on the 22 050 Hz signals (a second upload);
  batched   `audio_io.read_pcm` per file, then `Model.transcribe_pcm` (one library call: the stored PCM goes up once,
            one batched ingest per sub-batch, the forward pass reads its output on the device),

and within `batched` the host split: reading the files against the library call.  Prints one JSON line with the
medians, audio-seconds per second, and the device name and power limit read in the same run.  Needs a GPU: there is
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

FORMATS = {"int16": np.int16, "int32": np.int32, "uint8": np.uint8, "float32": np.float32}


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
        if dtype == np.uint8:
            pcm = np.round(cols * 120 + 128).astype(dtype)
        elif np.dtype(dtype).kind == "i":
            pcm = np.round(cols * 0.9 * np.iinfo(dtype).max).astype(dtype)
        else:
            pcm = cols.astype(dtype)
        paths.append(os.path.join(directory, f"clip{i:03d}.wav"))
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
            return {"read_pcm": t1 - t0, "transcribe_pcm": time.perf_counter() - t1}, arrs

        legs = {"per_file": per_file, "batched": batched}
        times = {name: [] for name in legs}
        notes = {}
        for r in range(args.warmup + args.rounds):
            for name, fn in legs.items():
                t, arrs = fn()
                notes[name] = int(arrs["note_off"][args.clips])
                if r >= args.warmup:
                    times[name].append(t)
        assert notes["per_file"] == notes["batched"] > 0, notes  # the two sequences transcribe the same notes

    audio_s = args.clips * args.seconds
    out.update({"clips": args.clips, "clip_seconds": args.seconds, "rate": args.rate, "format": args.format,
                "channels": args.channels, "file_mbytes": file_bytes / 1e6, "rounds": args.rounds, "notes": notes["batched"]})
    for name, rows in times.items():
        total = [sum(t.values()) for t in rows]
        for leg in rows[0]:
            out[f"{name}.{leg}_ms"] = 1e3 * float(np.median([t[leg] for t in rows]))
        out[f"{name}_ms"] = 1e3 * float(np.median(total))
        out[f"{name}_ms_min_max"] = [1e3 * min(total), 1e3 * max(total)]
        out[f"{name}_audio_s_per_s"] = audio_s / float(np.median(total))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
