#!/usr/bin/env python
"""Scoring a grid of note settings against annotated notes, three routes over the same host posteriorgrams, alternated in
one process:

  host     Model.decode_grid, then mir_eval's matching restated in NumPy / SciPy (oracle/transcription_ref.py) for every
           (setting, file) on the host — the route a tuning loop had before the library could score;
  notes    Model.decode_grid, then one Model.score_notes call (bp_score_notes_host) over every (setting, file);
  grid     Model.score_grid (bp_score_grid_host): decode and match on the device, four integers per pair come back.

Workloads: (a) the 180 s clip synth.random_notes_clip(180 s, seed 1) against its generating notes with 1, 8, 64 and 256
settings; (b) 1 250 annotated 10 s clips (seeds 3 + i) with 16 settings.  Prints the card's name and power limit, then one
JSON line per case (median ms per call over --repeats alternations, and whether the three routes' counts are identical),
then the device time per kernel (torch.profiler, a separate pass) of one grid call of the 180 s clip at 256 settings."""
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
from basic_pitch_b200.evaluate import EST_LOG2_HZ  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402
from basic_pitch_b200.note_creation import model_frames_to_time  # noqa: E402
from oracle import transcription_ref as tr  # noqa: E402

EST_HZ = 440.0 * 2.0 ** ((np.arange(128, dtype=np.float64) - 69.0) / 12.0)


def settings_grid(n: int):
    """n distinct settings of onset x frame threshold x minimum length x pitch range x inferred onsets (seeded order)."""
    all_ = [dict(onset_thresh=o, frame_thresh=f, min_note_len=m, min_pitch_idx=lo, max_pitch_idx=hi, infer_onsets=inf,
                 include_pitch_bends=False)
            for o, f, m, (lo, hi), inf in itertools.product((0.3, 0.4, 0.5, 0.6), (0.2, 0.25, 0.3, 0.35), (5, 8, 11, 17),
                                                             ((0, 88), (12, 76)), (True, False))]
    order = np.random.default_rng(0).permutation(len(all_))
    return [all_[k] for k in order[:n]]


class Case:
    def __init__(self, model: Model, outs, refs):
        self.model = model
        self.notes, self.onsets = [o["note"] for o in outs], [o["onset"] for o in outs]
        self.n = len(outs)
        self.refs = refs
        self.ref_l2 = [np.log2(hz) for _, hz in refs]
        self.times = model_frames_to_time(max(a.shape[0] for a in self.notes) + 1)

    def _estimates(self, arrs, P):
        noff = arrs["note_off"]
        n = int(noff[P * self.n])
        iv = np.stack([self.times[arrs["start"][:n]], self.times[arrs["end"][:n]]], 1)
        return noff, iv, arrs["pitch"][:n]

    def host(self, settings):
        P = len(settings)
        arrs = self.model.decode_grid(self.notes, self.onsets, None, settings, split_notes=False)
        noff, iv, pitch = self._estimates(arrs, P)
        out = np.zeros((P, self.n, 4), np.int64)
        for q in range(P * self.n):
            a, b = int(noff[q]), int(noff[q + 1])
            i = q % self.n
            n_ref, n_est = len(self.ref_l2[i]), b - a
            if n_ref and n_est:
                h0, h1 = tr.hit_matrices(self.refs[i][0], self.ref_l2[i], iv[a:b], EST_LOG2_HZ[pitch[a:b]])
                out[q // self.n, i] = (n_ref, n_est, tr.max_matching(h0), tr.max_matching(h1))
            else:
                out[q // self.n, i] = (n_ref, n_est, 0, 0)
        return out

    def notes_call(self, settings):
        P = len(settings)
        arrs = self.model.decode_grid(self.notes, self.onsets, None, settings, split_notes=False)
        noff, iv, pitch = self._estimates(arrs, P)
        hz = EST_HZ  # estimates go in as Hz; np.log2 of these is the table the grid route uses
        est = [(iv[noff[q] : noff[q + 1]], hz[pitch[noff[q] : noff[q + 1]]]) for q in range(P * self.n)]
        return self.model.score_notes(est, self.refs * P).reshape(P, self.n, 4)

    def grid(self, settings):
        return self.model.score_grid(self.notes, self.onsets, settings, self.refs)


def compare(case: Case, label: str, P: int, repeats: int):
    settings = settings_grid(P)
    routes = (("host", case.host), ("notes", case.notes_call), ("grid", case.grid))
    res = {name: fn(settings) for name, fn in routes}  # warm-up
    times = {name: [] for name, _ in routes}
    for _ in range(repeats):
        for name, fn in routes:
            t0 = time.perf_counter()
            res[name] = fn(settings)  # every route ends with its counts on the host
            times[name].append(time.perf_counter() - t0)
    row = {"case": label, "files": case.n, "settings": P, "refs": int(sum(len(x) for x in case.ref_l2)),
           "est_notes": int(res["grid"][..., 1].sum()), "matched": int(res["grid"][..., 3].sum()), "repeats": repeats}
    for name, _ in routes:
        row[f"{name}_ms"] = round(1e3 * float(np.median(times[name])), 2)
    row["counts_identical"] = bool(np.array_equal(res["host"], res["grid"]) and np.array_equal(res["notes"], res["grid"]))
    print(json.dumps(row), flush=True)


def kernel_times(case: Case, P: int):
    from torch.profiler import ProfilerActivity, profile

    settings = settings_grid(P)
    case.grid(settings)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        case.grid(settings)
    times = {}
    for ev in prof.key_averages():
        for short in ("decode_prep_kernel", "decode_cand_kernel", "decode_seq_kernel", "score_match_kernel"):
            if short in ev.key:
                us = getattr(ev, "device_time_total", None)
                times[short] = times.get(short, 0.0) + (us if us is not None else ev.cuda_time_total) / 1e3
    print(json.dumps({"case": f"kernel_ms_180s_grid_P{P}", **{k: round(v, 3) for k, v in times.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--clips", type=int, default=1250, help="10 s clips of case (b)")
    ap.add_argument("--no-bench", action="store_true", help="skip case (b)")
    args = ap.parse_args()
    assert np.array_equal(np.log2(EST_HZ), EST_LOG2_HZ)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": gpu[0] if gpu else "unknown"}), flush=True)
    model = Model(ICASSP_2022_MODEL_PATH)

    long_case = Case(model, model.run_inference_arrays([synth.random_notes_clip(180.0, seed=1)]),
                     [synth.random_notes_events(180.0, seed=1)])
    for P in (1, 8, 64, 256):
        compare(long_case, "180s", P, args.repeats)
    kernel_times(long_case, 256)
    del long_case

    if not args.no_bench:
        with ThreadPoolExecutor(8) as ex:
            clips = list(ex.map(lambda i: synth.random_notes_clip(10.0, seed=3 + i), range(args.clips)))
        refs = [synth.random_notes_events(10.0, seed=3 + i) for i in range(args.clips)]
        compare(Case(model, model.run_inference_arrays(clips), refs), f"bench_{args.clips}x10s", 16, args.repeats)


if __name__ == "__main__":
    main()
