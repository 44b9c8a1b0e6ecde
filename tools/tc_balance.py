"""How evenly one launch of each tensor-core conv kernel (conv_tc_kernel, 1 GPU) spreads its work over the SMs: builds
the library with -DBP_TC_CLOCKS into a temporary directory (or loads --lib), runs the forward pass on a batch of the
bench's full chunk and of its last, partial chunk, and prints per layer and batch as JSON the busy time of every CTA
(%globaltimer from its start to the end of its last MMA warp, bp_debug_tc_cta_busy): maximum, mean and minimum, and
the mean busy time of the CTAs grouped by blockIdx.x % k, k = the number of group ranges of the launch (a CTA walks the
items blockIdx.x, + grid, ...; under a uniform cut of every M-tile into k ranges it runs the same range in every item).
The launch lasts as long as its busiest CTA, so max / mean - 1 is the share of the launch the imbalance costs."""
import argparse
import ctypes as C
import json
import os
import sys
import tempfile
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

from tools.tc_clocks import build_clocks_lib  # noqa: E402

LAYERS = {0: "contour", 1: "onset", 2: "note"}
# (rows per window, frames an M-tile finishes, frequency groups) of the fused launches (tc_spec, tc_conv.cu)
GEOM = {0: (174, 60, 9), 1: (174, 62, 12), 2: (175, 58, 12)}


def uniform_split(n_windows, layer, n_sms):
    """the number of group runs per M-tile of the uniform decode (it / k, it % k) that launch_conv_tc used before it
    built a per-launch schedule: the least (waves x (groups per run + 0.5))"""
    rpw, ms, ng = GEOM[layer]
    n_mtiles = -(-n_windows * rpw // ms)
    best, split = 1e30, 1
    for s in range(1, ng + 1):
        cost = -(-n_mtiles * s // n_sms) * (-(-ng // s) + 0.5)
        if cost < best - 1e-9:
            best, split = cost, s
    return split


def n_ranges(lib, n_windows, layer, n_sms):
    """the launch's number of group ranges: the schedule's tail ranges where the library exports it"""
    if not hasattr(lib, "bp_debug_tc_schedule"):
        return uniform_split(n_windows, layer, n_sms), "uniform split"
    sizes = np.zeros(8, np.int32)
    lib.bp_debug_tc_schedule(layer, 1, n_windows, n_sms, sizes.ctypes.data, None, None)
    return int(sizes[4]), "tail ranges"


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1250, help="10 s clips of the bench step (sets the partial chunk)")
    ap.add_argument("--reps", type=int, default=5, help="timed forward passes per batch")
    ap.add_argument("--lib", help="an already built -DBP_TC_CLOCKS library (default: build one in a temporary directory)")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["BP_B200_LIB"] = a.lib or str(build_clocks_lib(Path(tmp)))
        import torch

        import bench
        from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
        from basic_pitch_b200.inference import Model

        model = Model(ICASSP_2022_MODEL_PATH)
        lib = model._lib
        n_sms = torch.cuda.get_device_properties(model.device).multi_processor_count
        chunk = int(lib.bp_model_chunk_windows(model.handle))
        step_windows = a.clips * int(lib.bp_num_windows(int(bench.CLIP_SECONDS * bench.SR)))
        batches = {"full_chunk": chunk, "partial_chunk": step_windows % chunk or chunk}
        rng = np.random.default_rng(0)
        busy = (C.c_uint64 * 256)()
        res = {"gpu": torch.cuda.get_device_name(0), "sms": n_sms, "reps": a.reps, "batches": {}}
        for label, n in batches.items():
            x = (0.1 * rng.standard_normal((n, 43844))).astype(np.float32)
            for _ in range(2):
                model.predict(x)
            for layer in LAYERS:
                lib.bp_debug_tc_cta_busy(model.handle, layer, busy, 0, 1)
            for _ in range(a.reps):
                model.predict(x)
            torch.cuda.synchronize()
            out = {"windows": n}
            for layer, name in LAYERS.items():
                lib.bp_debug_tc_cta_busy(model.handle, layer, busy, n_sms, 1)
                us = np.array(busy[:n_sms], np.float64) / a.reps / 1e3
                used = us[us > 0]
                k, kind = n_ranges(lib, n, layer, n_sms)
                out[name] = {
                    "max_us": round(float(used.max()), 1), "mean_us": round(float(us.mean()), 1),
                    "min_us": round(float(used.min()), 1), "max_over_mean": round(float(used.max() / us.mean()), 4),
                    "ctas": int(used.size), kind: k,
                    "mean_us_by_cta_mod_k": [round(float(us[np.arange(n_sms) % k == r].mean()), 1) for r in range(k)],
                }
            res["batches"][label] = out
        print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
