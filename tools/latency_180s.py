#!/usr/bin/env python
"""BASELINE configs[1]: one 180 s 22 050 Hz clip end to end on one GPU (audio in host memory -> note events),
with a per-stage breakdown and the event agreement against the oracle decode on the same posteriorgrams."""
import json
import sys
import time
import pathlib

import numpy as np

sys.path.insert(0, str(pathlib.Path(__file__).resolve().parent.parent))

from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, synth  # noqa: E402
from basic_pitch_b200.inference import Model  # noqa: E402


def main():
    import torch

    model = Model(ICASSP_2022_MODEL_PATH)
    clip = synth.random_notes_clip(180.0, seed=1)
    for _ in range(3):
        model.transcribe_arrays([clip], return_model_output=False)
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        outs, res, frames = model.transcribe_arrays([clip], return_model_output=False)
        ts.append(time.perf_counter() - t0)
    t_all = float(np.median(ts))
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        post = model.run_inference_arrays([clip])[0]
        ts.append(time.perf_counter() - t0)
    t_inf = float(np.median(ts))
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        dec = model.decode_arrays([post["note"]], [post["onset"]], [post["contour"]])[0]
        ts.append(time.perf_counter() - t0)
    t_dec = float(np.median(ts))
    out = {"clip_seconds": 180.0, "frames": int(frames[0]), "notes": int(len(res[0]["start"])),
           "transcribe_ms": 1e3 * t_all, "audio_s_per_s": 180.0 / t_all,
           "run_inference_ms_incl_posteriorgram_d2h": 1e3 * t_inf, "decode_ms_incl_posteriorgram_h2d": 1e3 * t_dec}
    if "--check" in sys.argv:
        from oracle import decode_ref

        with np.errstate(all="ignore"):
            wb, _ = decode_ref.model_output_to_note_events({k: np.array(v) for k, v in post.items()}, 0.5, 0.3)
        got = list(zip(dec["start"].tolist(), dec["end"].tolist(), dec["pitch"].tolist()))
        exp = [(a, b, p) for a, b, p, _a, _b in wb]
        out["events_identical_to_oracle_decode"] = got == exp
        out["bends_identical"] = [int(x) for x in dec["bends"]] == [int(v) for n in wb for v in n[4]]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
