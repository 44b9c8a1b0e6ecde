#!/usr/bin/env python
"""Scoring of the decoded notes with their pitch bends as a multi-f0 estimate (mir_eval.multipitch) and as a single-f0
track (mir_eval.melody) under a grid of note settings, two routes over the same host posteriorgrams in one process:

  host     Model.decode_grid (every note and bend comes to the host), evaluate.note_frames_to_multipitch /
           note_frames_to_melody for every (setting, file), then Model.score_multipitch / Model.score_melody on the
           series: the route a tuning loop has without the bent grid scorers;
  grid     Model.score_frames_grid(contours=...) (bp_score_bent_frames_grid_host) and Model.score_note_melody_grid
           (bp_score_note_melody_grid_host): the decode, the bends and the counts stay on the device.

Both routes' counts must be identical (asserted).  Workloads: (a) the 180 s monophonic line synth.melody_clip(180 s,
seed 1) with 1, 16 and 256 settings; (b) 1 250 10 s lines (seeds 3 + i) with 16 settings.  References: each clip's
exact f0 (synth.melody_f0) at a 10 ms hop, as a track and as a one-value-per-voiced-frame multi-pitch series.  Prints
the card's name, power limit and maximum SM clock, then one JSON line per case with the median ms per call of each
route over --repeats alternations (the host route runs --host-repeats times; on case (b) only with --bench-host)."""
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

from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, synth  # noqa: E402
from basic_pitch_b200.evaluate import note_frames_to_melody, note_frames_to_multipitch  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402

HOP = 0.01


def settings_grid(n: int):
    """n distinct note settings of onset x frame threshold x min_note_len x melodia x bends (seeded order)."""
    all_ = [dict(onset_thresh=round(float(o), 3), frame_thresh=round(float(f), 3), min_note_len=m, melodia_trick=mt,
                 include_pitch_bends=b)
            for o, f, m, mt, b in itertools.product(np.linspace(0.2, 0.8, 8), np.linspace(0.1, 0.5, 8), (5, 11),
                                                    (True, False), (True, False))]
    order = np.random.default_rng(0).permutation(len(all_))
    return [all_[k] for k in order[:n]]


class Case:
    def __init__(self, model: Model, outs, f0s):
        self.model = model
        self.notes, self.onsets, self.contours = ([o[k] for o in outs] for k in ("note", "onset", "contour"))
        self.n = len(outs)
        self.mel, self.mp = [], []
        for f0, g in zip(f0s, self.notes):
            t = np.arange(0, g.shape[0] * 256 / 22050, HOP)
            f = f0(t)
            self.mel.append((t, f))
            self.mp.append((t, [np.array([x]) if x > 0 else np.zeros(0) for x in f]))

    def host(self, settings):
        res = self.model.decode_grid(self.notes, self.onsets, self.contours, settings)
        mp_est, mel_est = [], []
        for per in res:
            for i, r in enumerate(per):
                bends = [r["bends"][r["bend_off"][j] : r["bend_off"][j + 1]] for j in range(len(r["start"]))]
                mp_est.append(note_frames_to_multipitch(r["start"], r["end"], r["pitch"], bends, self.notes[i].shape[0]))
                mel_est.append(note_frames_to_melody(r["start"], r["end"], r["pitch"], bends, self.notes[i]))
        P = len(settings)
        mp = self.model.score_multipitch(mp_est, self.mp * P).reshape(P, self.n, 7)
        mel = self.model.score_melody(mel_est, self.mel * P).reshape(P, self.n, 7)
        return mp, mel

    def grid(self, settings):
        mp = self.model.score_frames_grid(self.notes, self.onsets, settings, self.mp, contours=self.contours)
        mel = self.model.score_note_melody_grid(self.notes, self.onsets, self.contours, settings, self.mel)
        return mp, mel


def compare(case: Case, label: str, P: int, repeats: int, host_repeats: int):
    settings = settings_grid(P)
    res = {"grid": case.grid(settings)}  # warm-up
    times = {"host": [], "grid": []}
    for r in range(repeats):
        for name, fn in (("host", case.host), ("grid", case.grid)):
            if name == "host" and r >= host_repeats:
                continue
            t0 = time.perf_counter()
            res[name] = fn(settings)  # both routes end with their counts on the host
            times[name].append(time.perf_counter() - t0)
    mp, mel = res["grid"]
    row = {"case": label, "files": case.n, "settings": P, "ref_frames": int(mel[0, :, 0].sum()),
           "mp_tp": int(mp[..., 2].sum()), "mel_pitch_correct": int(mel[..., 4].sum()), "repeats": repeats,
           "host_repeats": len(times["host"])}
    for name in ("host", "grid"):
        row[f"{name}_ms"] = round(1e3 * float(np.median(times[name])), 2) if times[name] else None  # None: not measured
    if "host" in res:
        identical = all(np.array_equal(a, b) for a, b in zip(res["host"], res["grid"]))
        row["counts_identical"] = identical
        print(json.dumps(row), flush=True)
        assert identical, label
    else:
        row["counts_identical"] = None
        print(json.dumps(row), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--host-repeats", type=int, default=1)
    ap.add_argument("--clips", type=int, default=1250, help="10 s clips of case (b)")
    ap.add_argument("--no-long", action="store_true", help="skip case (a)")
    ap.add_argument("--no-bench", action="store_true", help="skip case (b)")
    ap.add_argument("--bench-host", action="store_true", help="also run the host route on case (b)")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": gpu[0] if gpu else "unknown"}), flush=True)
    model = Model(ICASSP_2022_MODEL_PATH)

    if not args.no_long:
        long_case = Case(model, model.run_inference_arrays([synth.melody_clip(180.0, seed=1)]),
                         [lambda t: synth.melody_f0(180.0, 1, t)])
        for P in (1, 16, 256):
            compare(long_case, "180s", P, args.repeats, args.host_repeats)
        del long_case

    if not args.no_bench:
        with ThreadPoolExecutor(8) as ex:
            clips = list(ex.map(lambda i: synth.melody_clip(10.0, seed=3 + i), range(args.clips)))
        f0s = [lambda t, i=i: synth.melody_f0(10.0, 3 + i, t) for i in range(args.clips)]
        compare(Case(model, model.run_inference_arrays(clips), f0s), f"bench_{args.clips}x10s", 16, args.repeats,
                args.host_repeats if args.bench_host else 0)


if __name__ == "__main__":
    main()
