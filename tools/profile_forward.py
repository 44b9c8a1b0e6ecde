"""Runs the forward pass (HCQT + CNN) on one full internal chunk of windows a few times: a short, steady target for a
profiler (for instance `ncu --set full -k regex:<kernel> ... python tools/profile_forward.py`)."""
import argparse
import sys
from pathlib import Path

import numpy as np

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=0, help="0 = one full internal chunk")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--path", type=int, default=1)
    a = ap.parse_args()
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, synth
    from basic_pitch_b200.inference import Model

    m = Model(ICASSP_2022_MODEL_PATH)
    m.set_path(a.path)
    n = a.windows or int(m._lib.bp_model_chunk_windows(m.handle))
    x = synth.window_batch(n, seed=1)
    for _ in range(a.reps):
        out = m.predict(x)
    print(n, "windows", {k: float(np.abs(v).mean()) for k, v in out.items()})


if __name__ == "__main__":
    main()
