#!/usr/bin/env python
"""Onset-only and offset-only scores of a grid of note settings against annotated notes, three routes over the same host
posteriorgrams, alternated in one process:

  host     Model.decode_grid, then mir_eval's match_note_onsets / match_note_offsets restated in NumPy
           (oracle/onset_offset_ref.py: dense hit matrices and the Hopcroft-Karp restatement) for every (setting, file);
  notes    Model.decode_grid, then one Model.score_onsets_offsets call (bp_score_onset_offset_notes_host) over every
           (setting, file);
  grid     Model.score_onset_offset_grid (bp_score_onset_offset_grid_host): decode and match on the device, four
           integers per pair come back.

Workloads are tools/score_grid_profile.py's: (a) the 180 s clip synth.random_notes_clip(180 s, seed 1) against its
generating notes with 1, 8, 64 and 256 settings; (b) 1 250 annotated 10 s clips (seeds 3 + i) with 16 settings.  Prints
the card's name and power limit, then one JSON line per case (median ms per call over --repeats alternations, the host
route over --host-repeats, and whether the three routes' counts are identical), then the device time per kernel
(torch.profiler, a separate pass) of one grid call of the 180 s clip at 256 settings."""
import argparse
import json
import pathlib
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))

from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, synth  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402
from basic_pitch_b200.note_creation import model_frames_to_time  # noqa: E402
from oracle import onset_offset_ref as oo  # noqa: E402
from tools.score_grid_profile import settings_grid  # noqa: E402


class Case:
    def __init__(self, model: Model, outs, refs):
        self.model = model
        self.notes, self.onsets = [o["note"] for o in outs], [o["onset"] for o in outs]
        self.n = len(outs)
        self.refs = [np.asarray(iv, np.float64).reshape(-1, 2) for iv, _ in refs]
        self.times = model_frames_to_time(max(a.shape[0] for a in self.notes) + 1)

    def _estimates(self, settings):
        P = len(settings)
        arrs = self.model.decode_grid(self.notes, self.onsets, None, settings, split_notes=False)
        noff = arrs["note_off"]
        n = int(noff[P * self.n])
        iv = np.stack([self.times[arrs["start"][:n]], self.times[arrs["end"][:n]]], 1)
        return [iv[noff[q] : noff[q + 1]] for q in range(P * self.n)]

    def host(self, settings):
        est = self._estimates(settings)
        out = np.array([oo.counts(self.refs[q % self.n], e) for q, e in enumerate(est)], np.int64)
        return out.reshape(len(settings), self.n, 4)

    def notes_call(self, settings):
        est = self._estimates(settings)
        return self.model.score_onsets_offsets(est, self.refs * len(settings)).reshape(len(settings), self.n, 4)

    def grid(self, settings):
        return self.model.score_onset_offset_grid(self.notes, self.onsets, settings, self.refs)


def compare(case: Case, label: str, P: int, repeats: int, host_repeats: int):
    settings = settings_grid(P)
    routes = (("notes", case.notes_call), ("grid", case.grid))
    res = {name: fn(settings) for name, fn in routes}  # warm-up
    times = {name: [] for name in ("host", "notes", "grid")}
    for r in range(repeats):
        for name, fn in ((("host", case.host),) if r < host_repeats else ()) + routes:
            t0 = time.perf_counter()
            res[name] = fn(settings)  # every route ends with its counts on the host
            times[name].append(time.perf_counter() - t0)
    g = res["grid"]
    row = {"case": label, "files": case.n, "settings": P, "refs": int(sum(len(x) for x in case.refs)),
           "est_notes": int(g[..., 1].sum()), "onsets_matched": int(g[..., 2].sum()),
           "offsets_matched": int(g[..., 3].sum()), "repeats": repeats, "host_repeats": len(times["host"])}
    for name in ("host", "notes", "grid"):
        if times[name]:
            row[f"{name}_ms"] = round(1e3 * float(np.median(times[name])), 2)
    same = np.array_equal(res["notes"], g) and ("host" not in res or np.array_equal(res["host"], g))
    row["counts_identical"] = bool(same)
    print(json.dumps(row), flush=True)


def kernel_times(case: Case, P: int):
    from torch.profiler import ProfilerActivity, profile

    settings = settings_grid(P)
    case.grid(settings)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        case.grid(settings)
    times = {}
    for ev in prof.key_averages():
        for short in ("decode_prep_kernel", "decode_cand_kernel", "decode_seq_kernel", "onset_offset_kernel"):
            if short in ev.key:
                us = getattr(ev, "device_time_total", None)
                times[short] = times.get(short, 0.0) + (us if us is not None else ev.cuda_time_total) / 1e3
    print(json.dumps({"case": f"kernel_ms_180s_grid_P{P}", **{k: round(v, 3) for k, v in times.items()}}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--host-repeats", type=int, default=1, help="alternations that include the (slow) host route")
    ap.add_argument("--clips", type=int, default=1250, help="10 s clips of case (b)")
    ap.add_argument("--no-bench", action="store_true", help="skip case (b)")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": gpu[0] if gpu else "unknown"}), flush=True)
    model = Model(ICASSP_2022_MODEL_PATH)

    long_case = Case(model, model.run_inference_arrays([synth.random_notes_clip(180.0, seed=1)]),
                     [synth.random_notes_events(180.0, seed=1)])
    for P in (1, 8, 64, 256):
        compare(long_case, "180s", P, args.repeats, args.host_repeats)
    kernel_times(long_case, 256)
    del long_case

    if not args.no_bench:
        with ThreadPoolExecutor(8) as ex:
            clips = list(ex.map(lambda i: synth.random_notes_clip(10.0, seed=3 + i), range(args.clips)))
        refs = [synth.random_notes_events(10.0, seed=3 + i) for i in range(args.clips)]
        compare(Case(model, model.run_inference_arrays(clips), refs), f"bench_{args.clips}x10s", 16, args.repeats,
                args.host_repeats)


if __name__ == "__main__":
    main()
