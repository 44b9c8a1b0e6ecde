#!/usr/bin/env python
"""Several metric families of one batch under one settings grid, two routes in one process, alternating:

  separate  the existing calls, one per family: evaluate_grid, evaluate_transcription_grid, evaluate_velocity_grid,
            evaluate_frames_grid (pitch_bends False and True), evaluate_note_melody_grid (pitch_bends True and False),
            evaluate_salience_grid, evaluate_melody_grid — each loads the audio, runs the model and decodes the grid;
  all       one inference.evaluate_all call for the same families: one ingest, one model run, one decode per chunk.

Every family's counts and scores must be identical on both routes (asserted).  Workloads: (a) the 180 s line
synth.melody_clip(180 s, seed 1) with 1, 16 and 256 settings; (b) 1 250 10 s lines (seeds 3 + i) with 16 settings.
References: each clip's exact f0 at a 10 ms hop as an f0 track and as a multi-pitch series, and as reference notes the
notes of one fixed setting with random velocities.  Prints the card's name, power limit and maximum SM clock (read
only), then one JSON line per case with the median ms per call of each route over --repeats alternations."""
import argparse
import itertools
import json
import pathlib
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))

from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, inference, synth  # noqa: E402
from basic_pitch_b200 import note_creation as infer  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402

HOP = 0.01
SAL = [dict(threshold=0.3), dict(threshold=0.5)]
MEL = [dict(threshold=0.3), dict(threshold=0.5, guess_unvoiced=False)]


def settings_grid(n: int):
    """n distinct predict settings of onset x frame threshold x minimum note length x melodia (seeded order)."""
    all_ = [dict(onset_threshold=round(float(o), 3), frame_threshold=round(float(f), 3), minimum_note_length=m,
                 melodia_trick=mt)
            for o, f, m, mt in itertools.product(np.linspace(0.2, 0.8, 8), np.linspace(0.1, 0.5, 8), (58.0, 127.7),
                                                 (True, False))]
    order = np.random.default_rng(0).permutation(len(all_))
    return [all_[k] for k in order[:n]]


def references(model: Model, clips, f0s):
    outs = model.run_inference_arrays(clips)
    res = model.decode_grid([o["note"] for o in outs], [o["onset"] for o in outs], [o["contour"] for o in outs],
                            [dict(onset_thresh=0.6, frame_thresh=0.35)])[0]
    rng = np.random.default_rng(7)
    notes, mp, mel = [], [], []
    for o, r, f0 in zip(outs, res, f0s):
        t = infer.model_frames_to_time(o["note"].shape[0] + 1)
        iv = np.stack([t[r["start"]], t[r["end"]]], 1) if len(r["start"]) else np.zeros((0, 2))
        notes.append((iv, 440.0 * 2.0 ** ((r["pitch"] - 69) / 12.0), rng.uniform(0, 127, len(r["start"]))))
        tt = np.arange(0, o["note"].shape[0] * 256 / 22050, HOP)
        f = f0(tt)
        mel.append((tt, f))
        mp.append((tt, [np.array([x]) if x > 0 else np.zeros(0) for x in f]))
    return notes, mp, mel


def separate(model, clips, settings, notes, mp, mel):
    pitched = [(iv, hz) for iv, hz, _ in notes]
    return {
        "notes": inference.evaluate_grid(clips, pitched, settings, model),
        "transcription": inference.evaluate_transcription_grid(clips, pitched, settings, model),
        "velocity": inference.evaluate_velocity_grid(clips, notes, settings, model),
        "frames": inference.evaluate_frames_grid(clips, mp, settings, model),
        "bent_frames": inference.evaluate_frames_grid(clips, mp, settings, model, pitch_bends=True),
        "note_melody": inference.evaluate_note_melody_grid(clips, mel, settings, model),
        "flat_note_melody": inference.evaluate_note_melody_grid(clips, mel, settings, model, pitch_bends=False),
        "salience": inference.evaluate_salience_grid(clips, mp, SAL, model_or_model_path=model),
        "melody": inference.evaluate_melody_grid(clips, mel, MEL, model_or_model_path=model),
    }


def together(model, clips, settings, notes, mp, mel):
    return inference.evaluate_all(clips, settings, notes=notes, multipitch=mp, f0=mel, salience=dict(settings=SAL),
                                  melody=dict(settings=MEL), model_or_model_path=model)


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, tuple):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


def compare(model, label, clips, f0s, P, repeats):
    settings = settings_grid(P)
    notes, mp, mel = references(model, clips, f0s)
    res = {"all": together(model, clips, settings, notes, mp, mel)}  # warm-up
    times = {"separate": [], "all": []}
    for _ in range(repeats):
        for name, fn in (("separate", separate), ("all", together)):
            t0 = time.perf_counter()
            res[name] = fn(model, clips, settings, notes, mp, mel)  # both routes end with their outputs on the host
            times[name].append(time.perf_counter() - t0)
    identical = same(res["separate"], res["all"])
    row = {"case": label, "files": len(clips), "settings": P, "repeats": repeats, "outputs_identical": identical}
    for name in times:
        row[f"{name}_ms"] = round(1e3 * float(np.median(times[name])), 1)
    print(json.dumps(row), flush=True)
    assert identical, label


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--clips", type=int, default=1250, help="10 s clips of case (b)")
    ap.add_argument("--no-long", action="store_true", help="skip case (a)")
    ap.add_argument("--no-bench", action="store_true", help="skip case (b)")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": gpu[0] if gpu else "unknown"}), flush=True)
    model = Model(ICASSP_2022_MODEL_PATH)
    if not args.no_long:
        for P in (1, 16, 256):
            compare(model, "180s", [synth.melody_clip(180.0, seed=1)], [lambda t: synth.melody_f0(180.0, 1, t)], P,
                    args.repeats)
    if not args.no_bench:
        with ThreadPoolExecutor(8) as ex:
            clips = list(ex.map(lambda i: synth.melody_clip(10.0, seed=3 + i), range(args.clips)))
        f0s = [lambda t, i=i: synth.melody_f0(10.0, 3 + i, t) for i in range(args.clips)]
        compare(model, f"bench_{args.clips}x10s", clips, f0s, 16, args.repeats)


if __name__ == "__main__":
    main()
