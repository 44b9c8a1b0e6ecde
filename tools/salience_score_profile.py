#!/usr/bin/env python
"""Frame-level scoring of the contour posteriorgram as a multi-f0 estimate under a grid of (threshold, peak picking,
frequency range) settings against annotated frames, two routes over the same host posteriorgrams in one process:

  host     evaluate.salience_to_multipitch, then mir_eval.multipitch restated in NumPy / SciPy
           (oracle/multipitch_ref.py) for every (setting, file) on the host: interp1d onto the reference times, one SciPy
           matching per frame and pass (memoised per distinct frame pair within a call, which only helps it) — the route
           a tuning loop has without the library;
  grid     Model.score_salience_grid (bp_score_salience_grid_host): the posteriorgrams go up once, estimates are read
           and matched on the device, seven integers per pair come back.

Workloads: (a) the 180 s clip synth.random_notes_clip(180 s, seed 1) with 1, 8, 64 and 256 settings; (b) 1 250 annotated
10 s clips (seeds 3 + i) with 16 settings.  References: each clip's generating notes at a 10 ms hop.  Prints the card's
name and power limit, then one JSON line per case: the median ms per call over --repeats alternations of the two routes
(the host route runs --host-repeats times; on case (b) only with --bench-host) and whether their counts are identical;
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
from basic_pitch_b200.evaluate import multipitch_values, notes_to_multipitch, salience_bins  # noqa: E402
from basic_pitch_b200.evaluate import salience_to_multipitch  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402
from oracle import multipitch_ref as mr  # noqa: E402

HOP = 0.01


def settings_grid(n: int):
    """n distinct settings of threshold x peak picking x frequency range (seeded order)."""
    hz = salience_bins("contour")[0]
    ranges = ((None, None), (55.0, 1760.0), (hz[36], hz[228]), (110.0, None))
    all_ = [dict(threshold=round(float(t), 4), peak_picking=p, minimum_frequency=a, maximum_frequency=b)
            for t, p, (a, b) in itertools.product(np.linspace(0.05, 0.95, 32), (True, False), ranges)]
    order = np.random.default_rng(0).permutation(len(all_))
    return [all_[k] for k in order[:n]]


class Case:
    def __init__(self, model: Model, outs, note_refs):
        self.model = model
        self.grams = [o["contour"] for o in outs]
        self.n = len(outs)
        self.lens = [a.shape[0] for a in self.grams]
        self.refs = []
        for (iv, hz), T in zip(note_refs, self.lens):
            t = np.arange(0, T * 256 / 22050, HOP)
            self.refs.append((t, notes_to_multipitch(iv, hz, t)))
        self.ref_vals = [[multipitch_values(f) for f in fr] for _, fr in self.refs]

    def host(self, settings):
        out = np.zeros((len(settings), self.n, 7), np.int64)
        memo = {}
        for k, s in enumerate(settings):
            for i, g in enumerate(self.grams):
                et, ef = salience_to_multipitch(g, **s)
                idx = mr.resample_index(et, self.refs[i][0])
                acc = np.zeros(7, np.int64)
                for j, (rm, rc) in enumerate(self.ref_vals[i]):
                    e = ef[idx[j]] if idx[j] >= 0 else np.zeros(0)
                    r, ne = len(rm), len(e)
                    tp = (0, 0)
                    if r and ne:
                        key = (rm.tobytes(), e.tobytes())
                        if key not in memo:
                            em, ec = multipitch_values(e)
                            memo[key] = (mr.max_matching(mr.hit_matrix(rm, em, 0.5, False)),
                                         mr.max_matching(mr.hit_matrix(rc, ec, 0.5, True)))
                        tp = memo[key]
                    acc += [r, ne, tp[0], tp[1], min(r, ne), max(r - ne, 0), max(ne - r, 0)]
                out[k, i] = acc
        return out

    def grid(self, settings):
        return self.model.score_salience_grid(self.grams, settings, self.refs)


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
    row = {"case": label, "files": case.n, "settings": P, "ref_frames": int(sum(len(t) for t, _ in case.refs)),
           "ref_values": int(res["grid"][0, :, 0].sum()), "est_values": int(res["grid"][..., 1].sum()),
           "tp": int(res["grid"][..., 2].sum()), "repeats": repeats, "host_repeats": len(times["host"])}
    for name in ("host", "grid"):
        row[f"{name}_ms"] = round(1e3 * float(np.median(times[name])), 2) if times[name] else None  # None: not measured
    row["counts_identical"] = bool(np.array_equal(res["host"], res["grid"])) if "host" in res else None
    print(json.dumps(row), flush=True)


def kernel_times(case: Case, P: int):
    from torch.profiler import ProfilerActivity, profile

    settings = settings_grid(P)
    case.grid(settings)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        case.grid(settings)
    times = {}
    for ev in prof.key_averages():
        for short in ("frame_match_kernel", "Memset", "Memcpy HtoD", "Memcpy DtoH"):
            if short in ev.key:
                us = getattr(ev, "device_time_total", None)
                times[short] = times.get(short, 0.0) + (us if us is not None else ev.cuda_time_total) / 1e3
    print(json.dumps({"case": f"kernel_ms_180s_grid_P{P}", **{k: round(v, 3) for k, v in times.items()}}), flush=True)


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
                args.host_repeats if args.bench_host else 0)


if __name__ == "__main__":
    main()
