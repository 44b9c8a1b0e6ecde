#!/usr/bin/env python
"""N live recordings transcribed at once: the stream group (Model.stream_group) against N predict_stream_notes
generators stepped in turn, over the same 1 s audio blocks of 180 s synthetic clips, the two routes alternated in one
run (group, interleaved generators, group again).  Reports per N the wall time per push round (host clock around each
synchronous call), audio-seconds transcribed per second, kernel launches per push, the most frames held by one stream,
the note latency (frames from a note's end to the last frame committed by the push that returned it) and whether both
routes gave the same notes; and the card's name and power limit from the same run.  One JSON line per N (and --out).

--capture RATE,DTYPE,CHANNELS (e.g. 48000,int16,2) measures live PCM streams instead: the clips are rendered once at
22 050 Hz, resampled on the host to RATE and quantised to DTYPE (the channels are the clip and a delayed, quieter copy),
and pushed in 1 s blocks of that format through StreamGroup.open_pcm streams, alternated in one run with the float
route fed bp_load_pcm_host of each whole clip in 1 s blocks (PCM, float, PCM).  Per N: push median and max, audio-s/s,
launches per push, host-to-device bytes per push of each route, whether both give the same notes, and the stream
ingest kernel's time per push from torch.profiler in a separate run over a few pushes."""
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


def capture(clip, rate, dtype, channels):
    """The 22 050 Hz clip as a device would capture it: resampled to `rate`, quantised to `dtype`."""
    from math import gcd

    import scipy.signal

    g = gcd(rate, SR)
    y = scipy.signal.resample_poly(clip.astype(np.float64), rate // g, SR // g)
    y = np.stack([y if c == 0 else 0.6 * np.roll(y, 37 * c) for c in range(channels)], axis=1)
    dt = np.dtype(dtype)
    if dt == np.float32:
        q = y.astype(np.float32)
    elif dt == np.uint8:
        q = np.clip(np.round(y * 0.8 * 127 + 128), 0, 255).astype(np.uint8)
    else:
        top = float(np.iinfo(dt).max)
        q = np.clip(np.round(y * 0.8 * top), -top - 1, top).astype(dt)
    return q[:, 0].copy() if channels == 1 else q


def whole_ingest(model, pcm, rate):
    from basic_pitch_b200 import audio_io

    ch = 1 if pcm.ndim == 1 else pcm.shape[1]
    out = np.empty(int(model._lib.bp_resampled_length(len(pcm), rate)), np.float32)
    model._lib.bp_load_pcm_host(model.handle, pcm.ctypes.data, audio_io._PCM_FORMATS[pcm.dtype], len(pcm), ch, rate,
                                out.ctypes.data)
    return out


def run_pcm(model, pcms, rate, profile_pushes=0):
    """The PCM route: 1 s blocks of each stream's capture format.  profile_pushes > 0: only that many pushes, under
    torch.profiler, -> the stream ingest kernel's total CUDA time per push (ms)."""
    g = model.stream_group()
    ch = 1 if pcms[0].ndim == 1 else pcms[0].shape[1]
    ids = [g.open_pcm(rate, ch, p.dtype) for p in pcms]
    n_blocks = max(-(-len(p) // rate) for p in pcms)
    if profile_pushes:
        import torch
        from torch.profiler import ProfilerActivity, profile

        for k in range(2):  # warm
            g.push({i: p[k * rate : (k + 1) * rate] for i, p in zip(ids, pcms)})
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            for k in range(2, 2 + profile_pushes):
                g.push({i: p[k * rate : (k + 1) * rate] for i, p in zip(ids, pcms)})
            torch.cuda.synchronize()
        us = sum(e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                 for e in prof.key_averages() if "stream_ingest_kernel" in e.key)  # fmt: skip
        return us / 1e3 / profile_pushes
    notes = {i: [] for i in ids}
    push_s, launches = [], []
    t_all = time.perf_counter()
    for k in range(n_blocks + 1):
        l0 = model.launch_count
        t0 = time.perf_counter()
        ev = g.push({i: p[k * rate : (k + 1) * rate] for i, p in zip(ids, pcms)}) if k < n_blocks else g.end(ids)
        push_s.append(time.perf_counter() - t0)
        launches.append(model.launch_count - l0)
        for i in ids:
            notes[i] += ev[i]
    wall = time.perf_counter() - t_all
    return dict(wall=wall, push_s=push_s[:-1], launches=launches[:-1], notes=[list(map(key, notes[i])) for i in ids])


def main_capture(args, model, gpu):
    rate, dtype, channels = args.capture.split(",")
    rate, channels = int(rate), int(channels)
    base = [synth.melody_clip(args.seconds, seed=s) for s in range(args.clips)]
    pcm_base = [capture(c, rate, dtype, channels) for c in base]
    float_base = [whole_ingest(model, p, rate) for p in pcm_base]
    run_pcm(model, pcm_base[:2], rate)  # warm-up
    run_group(model, float_base[:2])
    rows = []
    for n in (int(x) for x in args.streams.split(",")):
        pcms = [pcm_base[i % len(pcm_base)] for i in range(n)]
        floats = [float_base[i % len(float_base)] for i in range(n)]
        a = run_pcm(model, pcms, rate)
        f = run_group(model, floats)
        b = run_pcm(model, pcms, rate)
        audio_s = n * args.seconds
        frame_bytes = channels * np.dtype(dtype).itemsize
        row = {
            "streams": n, "capture": args.capture, "seconds_per_stream": args.seconds, "pushes": len(a["push_s"]),
            "pcm_push_ms_median": round(1e3 * float(np.median(a["push_s"] + b["push_s"])), 3),
            "pcm_push_ms_max": round(1e3 * max(a["push_s"] + b["push_s"]), 3),
            "pcm_audio_s_per_s": [round(audio_s / a["wall"], 1), round(audio_s / b["wall"], 1)],
            "pcm_launches_per_push_median": float(np.median(a["launches"])),
            "pcm_launches_per_push_max": int(max(a["launches"])),
            # blocks as stored, each padded to 16 bytes, behind a 120-byte descriptor and an int per stream (one copy)
            "pcm_h2d_bytes_per_push": int(n * (-(-(rate * frame_bytes) // 16) * 16) + -(-(n * 124 + 4) // 16) * 16),
            "float_push_ms_median": round(1e3 * float(np.median(f["push_s"][:-1])), 3),
            "float_push_ms_max": round(1e3 * max(f["push_s"][:-1]), 3),
            "float_audio_s_per_s": round(audio_s / f["wall"], 1),
            "float_launches_per_push_median": float(np.median(f["launches"][:-1])),
            "float_h2d_bytes_per_push": int(n * SR * 4),
            "notes_equal_float_route": a["notes"] == f["notes"] and b["notes"] == f["notes"],
            "gpu": gpu,
        }  # fmt: skip
        row["ingest_kernel_ms_per_push"] = round(run_pcm(model, pcms, rate, profile_pushes=5), 4)
        print(json.dumps(row), flush=True)
        rows.append(row)
    return rows


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
    ap.add_argument("--capture", default=None, help="RATE,DTYPE,CHANNELS: live PCM streams of that format (see above)")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    model = Model(ICASSP_2022_MODEL_PATH)
    if args.capture:
        rows = main_capture(args, model, gpu)
        if args.out:
            args.out.parent.mkdir(parents=True, exist_ok=True)
            args.out.write_text("\n".join(json.dumps(r) for r in rows) + "\n")
        return
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
