#!/usr/bin/env python
"""Overlap and velocity scores of a grid of note settings against annotated notes with velocities, two routes over the
same host posteriorgrams:

  host     Model.decode_grid, then mir_eval's matching restated in plain Python (oracle/note_matching_ref.py) for every
           (setting, file, pass) on the host, then evaluate.matching_scores — the route a tuning loop has without the
           library's matchings;
  grid     Model.match_grid (bp_match_grid_host): decode and match on the device, the notes and the pairs come back, then
           evaluate.matching_scores.

Workloads: (a) the 180 s clip synth.random_notes_clip(180 s, seed 1) against its generating notes (seeded velocities)
with 1, 8, 64 and 256 settings; (b) 1 250 annotated 10 s clips (seeds 3 + i) with 16 settings.  Prints the card's name
and power limit, then one JSON line per case: the median ms of the grid route over --repeats calls, its share spent in
matching_scores on the host, the host route's ms (one call), and whether both routes give identical pairs and floats."""
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
from basic_pitch_b200.evaluate import EST_LOG2_HZ, matching_scores, note_velocities  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402
from basic_pitch_b200.note_creation import model_frames_to_time  # noqa: E402
from oracle import note_matching_ref as nm  # noqa: E402
from tools.score_grid_profile import settings_grid  # noqa: E402


class Case:
    def __init__(self, model: Model, outs, refs, seed: int):
        self.model = model
        self.notes, self.onsets = [o["note"] for o in outs], [o["onset"] for o in outs]
        self.n = len(outs)
        self.refs = refs
        self.ref_l2 = [np.log2(hz) for _, hz in refs]
        rng = np.random.default_rng(seed)
        self.ref_v = [rng.integers(20, 128, len(hz)) for _, hz in refs]
        self.times = model_frames_to_time(max(a.shape[0] for a in self.notes) + 1)

    def _scores(self, res, match):
        out = []
        for k, per in enumerate(res):
            for i, r in enumerate(per):
                est_iv = np.stack([self.times[r["start"]], self.times[r["end"]]], 1)
                out.append(matching_scores(self.refs[i][0], self.ref_v[i], est_iv, note_velocities(r["amp"]), match[k][i]))
        return out

    def host(self, settings):
        res = self.model.decode_grid(self.notes, self.onsets, None, settings)
        match = []
        for per in res:
            row = []
            for i, r in enumerate(per):
                est_iv = np.stack([self.times[r["start"]], self.times[r["end"]]], 1)
                est_l2 = EST_LOG2_HZ[np.asarray(r["pitch"], np.int64)]
                row.append(np.stack([nm.match_array(nm.match_notes(self.refs[i][0], self.ref_l2[i], est_iv, est_l2, w),
                                                    len(self.ref_l2[i])) for w in (False, True)]))
            match.append(row)
        return match, self._scores(res, match), 0.0

    def grid(self, settings):
        res, match = self.model.match_grid(self.notes, self.onsets, settings, self.refs)
        t0 = time.perf_counter()
        scores = self._scores(res, match)
        return match, scores, time.perf_counter() - t0


def _same(a, b):
    ma, sa, _ = a
    mb, sb, _ = b
    pairs = all(np.array_equal(x, y) for ra, rb in zip(ma, mb) for x, y in zip(ra, rb))
    floats = all(x.keys() == y.keys() and all(np.float64(x[k]).tobytes() == np.float64(y[k]).tobytes() for k in x)
                 for x, y in zip(sa, sb))
    return pairs and floats


def compare(case: Case, label: str, P: int, repeats: int):
    settings = settings_grid(P)
    case.grid(settings)  # warm-up
    times, host_scores = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        g = case.grid(settings)
        times.append(time.perf_counter() - t0)
        host_scores.append(g[2])
    t0 = time.perf_counter()
    h = case.host(settings)
    host_s = time.perf_counter() - t0
    row = {"case": label, "files": case.n, "settings": P, "refs": int(sum(len(x) for x in case.ref_l2)),
           "matched": int(sum((m[1] >= 0).sum() for per in g[0] for m in per)), "grid_repeats": repeats,
           "grid_ms": round(1e3 * float(np.median(times)), 1),
           "grid_matching_scores_ms": round(1e3 * float(np.median(host_scores)), 1),
           "host_ms": round(1e3 * host_s, 1), "identical": _same(g, h)}
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--clips", type=int, default=1250, help="10 s clips of case (b)")
    ap.add_argument("--no-bench", action="store_true", help="skip case (b)")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    rows = [{"gpu": gpu[0] if gpu else "unknown"}]
    print(json.dumps(rows[0]), flush=True)
    model = Model(ICASSP_2022_MODEL_PATH)

    long_case = Case(model, model.run_inference_arrays([synth.random_notes_clip(180.0, seed=1)]),
                     [synth.random_notes_events(180.0, seed=1)], seed=1)
    for P in (1, 8, 64, 256):
        rows.append(compare(long_case, "180s", P, args.repeats))
    del long_case

    if not args.no_bench:
        with ThreadPoolExecutor(8) as ex:
            clips = list(ex.map(lambda i: synth.random_notes_clip(10.0, seed=3 + i), range(args.clips)))
        refs = [synth.random_notes_events(10.0, seed=3 + i) for i in range(args.clips)]
        rows.append(compare(Case(model, model.run_inference_arrays(clips), refs, seed=2), f"bench_{args.clips}x10s", 16,
                            args.repeats))
    if args.out:
        pathlib.Path(args.out).parent.mkdir(parents=True, exist_ok=True)
        pathlib.Path(args.out).write_text("".join(json.dumps(r) + "\n" for r in rows))


if __name__ == "__main__":
    main()
