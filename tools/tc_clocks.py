"""Cycle accounting of the three tensor-core conv kernels (conv_tc_kernel, 1 GPU): builds the library with
-DBP_TC_CLOCKS into a temporary directory (or loads --lib), runs the bench workload and prints, per layer, where the
warps' SM cycles go as JSON: the consumer warpgroups (contour: waiting on a weight stage; onset / note: gathering the A
registers; then MMAs, epilogue, waiting on the data tile) and the producer warp (contour: waiting on a free stage; all:
waiting on the data tile to be released)."""
import argparse
import ctypes as C
import json
import os
import shutil
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

LAYERS = {0: "contour", 1: "onset", 2: "note"}
CONSUMER = ["wait_weight_stage", "mma", "epilogue", "wait_data_tile", "other"]
PRODUCER = ["wait_free_stage", "wait_data_release", "other"]
# the onset and note kernels gather their A operand and have no weight ring: the first consumer bucket is the gather
CONSUMER_GATHER = ["gather"] + CONSUMER[1:]


def build_clocks_lib(dst: Path) -> Path:
    """The library with -DBP_TC_CLOCKS, built from a copy of the sources under dst (the tree is not written)."""
    shutil.copytree(ROOT / "basic_pitch_b200" / "csrc", dst / "basic_pitch_b200" / "csrc",
                    ignore=shutil.ignore_patterns("*.o"))
    shutil.copytree(ROOT / "include", dst / "include")
    out = dst / "libbp_b200_clocks.so"
    jobs = str(max(1, min(8, os.cpu_count() or 1)))
    r = subprocess.run(["make", "-C", str(dst / "basic_pitch_b200" / "csrc"), "-j", jobs, "EXTRA=-DBP_TC_CLOCKS",
                        f"OUT={out}"], capture_output=True, text=True)
    if r.returncode != 0:
        sys.exit(f"building the -DBP_TC_CLOCKS library failed:\n{r.stdout}\n{r.stderr}")
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1250)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--lib", help="an already built -DBP_TC_CLOCKS library (default: build one in a temporary directory)")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        os.environ["BP_B200_LIB"] = a.lib or str(build_clocks_lib(Path(tmp)))
        import torch

        import bench
        from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, engine
        from basic_pitch_b200.inference import Model

        model = Model(ICASSP_2022_MODEL_PATH)
        lib = model._lib
        clips = bench.make_clips(a.clips, seed0=3)
        packed = engine.PackedAudio(clips, pinned=True)
        n_windows = sum(int(lib.bp_num_windows(len(c))) for c in clips)
        n_frames = sum(int(lib.bp_num_frames(len(c))) for c in clips)
        out = engine.NoteBuffers(a.clips, max(4096, 2 * n_frames), max(65536, 24 * n_frames))
        d_audio = packed.to_device(0)
        step = lambda: engine.transcribe_packed_device(model, d_audio, packed.offsets, out)  # noqa: E731
        for _ in range(3):
            step()
        cyc = (C.c_uint64 * 8)()
        for layer in LAYERS:
            lib.bp_debug_tc_clocks(model.handle, layer, cyc, 1)
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
        res = {"clips": a.clips, "windows": n_windows, "steps": a.steps,
               "gpu": torch.cuda.get_device_name(0), "layers": {}}
        for layer, name in LAYERS.items():
            lib.bp_debug_tc_clocks(model.handle, layer, cyc, 1)
            c = [int(v) for v in cyc]
            cons, prod = c[:5], c[5:]
            res["layers"][name] = {
                "consumer_share": {k: round(v / max(1, sum(cons)), 4)
                                   for k, v in zip(CONSUMER if layer == 0 else CONSUMER_GATHER, cons)},
                "producer_share": {k: round(v / max(1, sum(prod)), 4) for k, v in zip(PRODUCER, prod)},
                "consumer_warp_cycles_per_step": sum(cons) // a.steps,
            }
        print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
