#!/usr/bin/env python
"""The grid decode (bp_decode_grid_device) against the same settings decoded one bp_decode_device call at a time, on
device-resident posteriorgrams, alternating the two in one process:

  (a) the 180 s BASELINE configs[1] clip (synth.random_notes_clip(180 s, seed 1)) with P = 1, 8, 64, 256 settings;
  (b) the bench workload, 1 250 x 10 s clips (synth.random_notes_clip(10 s, seed 3 + i)), with P = 16.

Prints one JSON line per case: median ms per call of each route over --repeats alternations, the chunk count, and
whether every (setting, file) of the grid equals its single decode bit for bit; then the device time per decode kernel
(torch.profiler, a separate pass) of one single-setting decode and one grid call of the 180 s clip, which breaks out
the sequential loop kernel; and the card's name and power limit."""
import argparse
import ctypes as C
import itertools
import json
import pathlib
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))

from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, _lib, synth  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402


def settings_grid(n: int):
    """n distinct settings of onset x frame threshold x minimum length x pitch range x inferred onsets (seeded order)."""
    all_ = [dict(onset_thresh=o, frame_thresh=f, min_note_len=m, min_pitch_idx=lo, max_pitch_idx=hi, infer_onsets=inf)
            for o, f, m, (lo, hi), inf in itertools.product((0.3, 0.4, 0.5, 0.6), (0.2, 0.25, 0.3, 0.35), (5, 8, 11, 17),
                                                             ((0, 88), (12, 76)), (True, False))]
    order = np.random.default_rng(0).permutation(len(all_))
    return [all_[k] for k in order[:n]]


class Case:
    """Posteriorgrams of a batch on the device and both decode routes over them."""

    def __init__(self, model: Model, outs):
        import torch

        self.model, self.lib = model, model._lib
        self.n = len(outs)
        self.foff = np.cumsum([0] + [o["note"].shape[0] for o in outs]).astype(np.int64)
        dev = f"cuda:{model.device}"
        self.d = [torch.from_numpy(np.ascontiguousarray(np.concatenate([o[k] for o in outs]))).to(dev)
                  for k in ("note", "onset", "contour")]
        self.stream = torch.cuda.Stream(device=dev)
        torch.cuda.synchronize(dev)
        self.total = int(self.foff[-1])

    def _ptrs(self):
        return self.d[0].data_ptr(), self.d[1].data_ptr(), self.d[2].data_ptr()

    def single(self, settings):
        """One bp_decode_device call per setting; the concatenated arrays of every call."""
        out = []
        for s in settings:
            p = self.model._params(**{**Model._DECODE_DEFAULTS, **s})
            nt, arrs = self.model._alloc_notes(self.n, 2 * self.total + 4096, 24 * self.total + 65536)
            self.lib.bp_decode_device(self.model.handle, *self._ptrs(), self.foff.ctypes.data, self.n, C.byref(p),
                                      C.byref(nt), self.stream.cuda_stream)
            out.append(arrs)
        return out

    def grid(self, settings):
        P = len(settings)
        ps = (_lib.DecodeParams * P)(*[self.model._params(**{**Model._DECODE_DEFAULTS, **s}) for s in settings])
        nt, arrs = self.model._alloc_notes(self.n * P, 2 * self.total * P + 4096, 24 * self.total * P + 65536)
        self.lib.bp_decode_grid_device(self.model.handle, *self._ptrs(), self.foff.ctypes.data, self.n, ps, P, C.byref(nt),
                                       self.stream.cuda_stream)
        return arrs

    def identical(self, single, grid) -> bool:
        flat = self.model._split_notes(grid, self.n * len(single))
        for k, arrs in enumerate(single):
            for i, r in enumerate(self.model._split_notes(arrs, self.n)):
                g = flat[k * self.n + i]
                for key in ("start", "end", "pitch", "bend_off", "bends"):
                    if not np.array_equal(np.asarray(g[key], np.int64), np.asarray(r[key], np.int64)):
                        return False
                if g["amp"].tobytes() != r["amp"].tobytes():
                    return False
        return True


def compare(case: Case, label: str, P: int, repeats: int):
    settings = settings_grid(P)
    case.single(settings)  # warm-up (workspace growth, module load)
    case.grid(settings)
    t_single, t_grid = [], []
    for _ in range(repeats):
        t0 = time.perf_counter()
        single = case.single(settings)  # every call synchronises its stream before returning
        t_single.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        grid = case.grid(settings)
        t_grid.append(time.perf_counter() - t0)
    chunk = int(case.lib.bp_decode_grid_chunk_params(case.total, case.n))
    n_notes = int(grid["note_off"][P * case.n])
    row = {"case": label, "files": case.n, "frames": case.total, "settings": P, "chunks": -(-P // chunk),
           "settings_per_chunk": chunk, "notes": n_notes, "repeats": repeats,
           "single_calls_ms": 1e3 * float(np.median(t_single)), "grid_call_ms": 1e3 * float(np.median(t_grid)),
           "notes_identical": case.identical(single, grid)}
    row["speedup"] = row["single_calls_ms"] / row["grid_call_ms"]
    print(json.dumps(row), flush=True)
    return row


def kernel_times(case: Case, P: int):
    """Device time per decode kernel (torch.profiler) of one single-setting call and one grid call of P settings."""
    from torch.profiler import ProfilerActivity, profile

    settings = settings_grid(P)
    out = {}
    for label, fn in (("single_default", lambda: case.single([{}])), (f"grid_P{P}", lambda: case.grid(settings))):
        fn()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        times = {}
        for ev in prof.key_averages():
            name = ev.key
            for short in ("decode_prep_kernel", "decode_cand_kernel", "decode_seq_kernel", "compact_notes_kernel",
                          "note_finish_kernel"):
                if short in name:
                    us = getattr(ev, "device_time_total", None)
                    if us is None:
                        us = ev.cuda_time_total
                    times[short] = times.get(short, 0.0) + us / 1e3
        out[label] = {k: round(v, 3) for k, v in times.items()}
    print(json.dumps({"case": "kernel_ms_180s", **out}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--clips", type=int, default=1250, help="10 s clips of case (b)")
    ap.add_argument("--no-bench", action="store_true", help="skip case (b)")
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    print(json.dumps({"gpu": gpu[0] if gpu else "unknown"}), flush=True)
    model = Model(ICASSP_2022_MODEL_PATH)

    clip = synth.random_notes_clip(180.0, seed=1)
    long_case = Case(model, model.run_inference_arrays([clip]))
    for P in (1, 8, 64, 256):
        compare(long_case, "180s", P, args.repeats)
    kernel_times(long_case, 64)
    del long_case

    if not args.no_bench:
        with ThreadPoolExecutor(8) as ex:
            clips = list(ex.map(lambda i: synth.random_notes_clip(10.0, seed=3 + i), range(args.clips)))
        bench_case = Case(model, model.run_inference_arrays(clips))
        compare(bench_case, f"bench_{args.clips}x10s", 16, args.repeats)


if __name__ == "__main__":
    main()
