#!/usr/bin/env python
"""The note stream (Model.note_stream, inference.predict_stream_notes) on a 180 s melody clip and a long synthetic
recording (the clip repeated, one hour by default) delivered in 1 s audio blocks: time per push (host clock around the synchronous call), emission latency
(frames from a note's end to the end of the push that returned it), the most frames held on the device, and the wall
time of predict_stream_notes against predict_stream over the same blocks, with the notes of both routes compared.
Writes one JSON line per recording (and to --out)."""
import argparse
import json
import pathlib
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))

from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, synth  # noqa: E402
from basic_pitch_b200.note_creation import model_frames_to_time  # noqa: E402
from basic_pitch_b200.inference import Model, predict_stream, predict_stream_notes, run_inference_stream  # noqa: E402


def blocks(audio, n=22050):
    return (audio[i : i + n] for i in range(0, len(audio), n))


def profile(model, name, audio, windows_per_step):
    parts = list(run_inference_stream(blocks(audio), model, windows_per_step))
    stream = model.note_stream()
    push_s, latency, held, pushed = [], [], 0, 0
    for part in parts:
        t0 = time.perf_counter()
        ev = stream.push(part["note"], part["onset"], part["contour"])
        push_s.append(time.perf_counter() - t0)
        pushed += part["note"].shape[0]
        held = max(held, stream.held_frames)
        times = model_frames_to_time(pushed + 1)
        latency += [pushed - int(np.searchsorted(times, e[1])) for e in ev]  # end time back to its frame
    t0 = time.perf_counter()
    tail = stream.end()
    end_s = time.perf_counter() - t0
    t0 = time.perf_counter()
    streamed = [e for _, ev in predict_stream_notes(blocks(audio), model, windows_per_step=windows_per_step) for e in ev]
    t_stream = time.perf_counter() - t0
    t0 = time.perf_counter()
    _, _, whole = predict_stream(blocks(audio), model, windows_per_step=windows_per_step)
    t_whole = time.perf_counter() - t0
    key = lambda e: (e[0], e[1], int(e[2]), float(e[3]), tuple(e[4] or ()))  # noqa: E731
    same = sorted(map(key, streamed)) == sorted(map(key, whole))
    return {
        "recording": name, "seconds": round(len(audio) / 22050, 1), "frames": pushed, "pushes": len(parts),
        "push_ms_median": round(1e3 * float(np.median(push_s)), 3), "push_ms_max": round(1e3 * max(push_s), 3),
        "end_ms": round(1e3 * end_s, 3), "notes": len(streamed), "notes_at_end": len(tail),
        "latency_frames_median": float(np.median(latency)) if latency else None,
        "latency_frames_max": int(max(latency)) if latency else None, "held_frames_max": held,
        "predict_stream_notes_s": round(t_stream, 3), "predict_stream_s": round(t_whole, 3),
        "notes_equal_predict_stream": same,
    }  # fmt: skip


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--long-repeats", type=int, default=20, help="the long recording: the 180 s clip this many times")
    ap.add_argument("--windows-per-step", type=int, default=64)
    ap.add_argument("--out", type=pathlib.Path, default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    model = Model(ICASSP_2022_MODEL_PATH)
    profile(model, "warm-up", synth.melody_clip(20.0, seed=1), args.windows_per_step)
    rows = []
    clip = synth.melody_clip(180.0, seed=3)
    for name, audio in (("melody 180 s", clip), (f"melody 180 s x {args.long_repeats}", np.tile(clip, args.long_repeats))):
        row = dict(profile(model, name, audio, args.windows_per_step), gpu=gpu)
        print(json.dumps(row), flush=True)
        rows.append(row)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
