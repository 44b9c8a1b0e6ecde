"""Per-stage device time of one bench step (1 GPU): runs the bench workload once per kernel family with the library's
event profiling (bp_model_profile) switched to that family and prints ms per step and us per window."""
import argparse
import ctypes as C
import json
import sys
import time
from pathlib import Path

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))

FAMILIES = {0: "contour conv (wgmma, fused conv2)", 1: "onset conv (wgmma)", 2: "CQT + log-normalise",
            3: "decimation chain", 4: "note conv + tap sums + contour tap sum", 5: "decode prep/cand/seq",
            6: "note finish (amplitude, bends)"}


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=1250)
    ap.add_argument("--steps", type=int, default=2)
    a = ap.parse_args()
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
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.steps):
        step()
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) * 1e3 / a.steps
    res = {"clips": a.clips, "windows": n_windows, "step_ms_wall": wall, "us_per_window": wall * 1e3 / n_windows, "families": {}}
    acc = 0.0
    for fam, name in FAMILIES.items():
        lib.bp_model_profile(model.handle, fam)
        for _ in range(a.steps):
            step()
        tot, nint, nwin = C.c_double(), C.c_int64(), C.c_int64()
        lib.bp_model_profile_read(model.handle, C.byref(tot), C.byref(nint), C.byref(nwin))
        lib.bp_model_profile(model.handle, -1)
        ms = tot.value / a.steps
        acc += ms
        res["families"][name] = {"ms_per_step": round(ms, 3), "us_per_window": round(ms * 1e3 / n_windows, 3)}
    res["sum_of_families_ms"] = round(acc, 3)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
