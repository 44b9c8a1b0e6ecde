#!/usr/bin/env python
"""N live recordings transcribed at once: the stream group (Model.stream_group) against N predict_stream_notes
generators stepped in turn, over the same 1 s audio blocks of 180 s synthetic clips, the two routes alternated in one
run (group, interleaved generators, group again).  Reports per N the wall time per push round (host clock around each
synchronous call), audio-seconds transcribed per second, kernel launches per push, the most frames held by one stream,
the note latency (frames from a note's end to the last frame committed by the push that returned it) and whether both
routes gave the same notes; and the card's name and power limit from the same run.  One JSON line per N (and --out)."""
import argparse
import json
import pathlib
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))

from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, synth  # noqa: E402
from basic_pitch_b200.inference import Model, predict_stream_notes  # noqa: E402
from basic_pitch_b200.note_creation import model_frames_to_time  # noqa: E402

SR, HOP, LEAD, WIN, PER_WINDOW = 22050, 36164, 3840, 43844, 142


def committed(samples):
    """Frames a stream has committed after `samples` samples (run_inference_stream holds back its newest two windows)."""
    nw = (samples + LEAD - WIN) // HOP + 1 if samples + LEAD >= WIN else 0
    return max(0, (nw - 2) * PER_WINDOW)


def blocks(audio):
    return [audio[i : i + SR] for i in range(0, len(audio), SR)]


def key(e):
    return (float(e[0]), float(e[1]), int(e[2]), float(e[3]), tuple(e[4] or ()))


def end_frame(e, times):
    return int(np.searchsorted(times, e[1]))


def run_group(model, clips):
    g = model.stream_group()
    ids = [g.open() for _ in clips]
    n_blocks = max(-(-len(c) // SR) for c in clips)
    times = model_frames_to_time(max(len(c) for c in clips) // 256 + 200)
    notes = {i: [] for i in ids}
    push_s, launches, held, latency = [], [], 0, []
    t_all = time.perf_counter()
    for k in range(n_blocks + 1):
        l0 = model.launch_count
        t0 = time.perf_counter()
        if k < n_blocks:
            ev = g.push({i: c[k * SR : (k + 1) * SR] for i, c in zip(ids, clips)})
        else:
            ev = g.end(ids)
        push_s.append(time.perf_counter() - t0)
        launches.append(model.launch_count - l0)
        for i, c in zip(ids, clips):
            held = max(held, g.held_frames(i))
            if k < n_blocks:
                now = committed(min(len(c), (k + 1) * SR))
                latency += [now - end_frame(e, times) for e in ev[i]]
            notes[i] += ev[i]
    wall = time.perf_counter() - t_all
    return dict(wall=wall, push_s=push_s, launches=launches, held=held, latency=latency,
                notes=[list(map(key, notes[i])) for i in ids])  # fmt: skip


def run_interleaved(model, clips):
    gens = [predict_stream_notes(blocks(c), model) for c in clips]
    notes = [[] for _ in clips]
    live = list(range(len(clips)))
    rounds = []
    t_all = time.perf_counter()
    while live:
        t0 = time.perf_counter()
        for j in list(live):
            try:
                notes[j] += next(gens[j])[1]
            except StopIteration:
                live.remove(j)
        rounds.append(time.perf_counter() - t0)
    wall = time.perf_counter() - t_all
    return dict(wall=wall, rounds=rounds, notes=[list(map(key, n)) for n in notes])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,16,64,256")
    ap.add_argument("--seconds", type=float, default=180.0)
    ap.add_argument("--clips", type=int, default=8, help="distinct synthetic clips, cycled over the streams")
    ap.add_argument("--interleaved-max", type=int, default=64,
                    help="largest N for which the N separate generators run too (they take N times the pushes)")
    ap.add_argument("--out", type=pathlib.Path, default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    model = Model(ICASSP_2022_MODEL_PATH)
    base = [synth.melody_clip(args.seconds, seed=s) for s in range(args.clips)]
    run_group(model, base[:2])  # warm-up
    rows = []
    for n in (int(x) for x in args.streams.split(",")):
        clips = [base[i % len(base)] for i in range(n)]
        a = run_group(model, clips)
        sep = run_interleaved(model, clips) if n <= args.interleaved_max else None
        b = run_group(model, clips)
        audio_s = n * args.seconds
        row = {
            "streams": n, "seconds_per_stream": args.seconds, "pushes": len(a["push_s"]),
            "group_push_ms_median": round(1e3 * float(np.median(a["push_s"] + b["push_s"])), 3),
            "group_push_ms_max": round(1e3 * max(a["push_s"] + b["push_s"]), 3),
            "group_audio_s_per_s": [round(audio_s / a["wall"], 1), round(audio_s / b["wall"], 1)],
            "group_launches_per_push_median": float(np.median(a["launches"])),
            "group_launches_per_push_max": int(max(a["launches"])),
            "held_frames_max_per_stream": a["held"],
            "latency_frames_median": float(np.median(a["latency"])) if a["latency"] else None,
            "latency_frames_max": int(max(a["latency"])) if a["latency"] else None,
            "group_runs_equal": a["notes"] == b["notes"],
            "gpu": gpu,
        }  # fmt: skip
        if sep is not None:
            row.update({
                "interleaved_round_ms_median": round(1e3 * float(np.median(sep["rounds"])), 3),
                "interleaved_audio_s_per_s": round(audio_s / sep["wall"], 1),
                "speedup_vs_interleaved": round(sep["wall"] / min(a["wall"], b["wall"]), 2),
                "notes_equal_interleaved": sep["notes"] == a["notes"],
            })  # fmt: skip
        print(json.dumps(row), flush=True)
        rows.append(row)
    if args.out:
        args.out.parent.mkdir(parents=True, exist_ok=True)
        args.out.write_text("\n".join(json.dumps(r) for r in rows) + "\n")


if __name__ == "__main__":
    main()
