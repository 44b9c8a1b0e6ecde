#!/usr/bin/env python
"""Throughput of the MIDI sonification (`--sonify-midi`): the bundled stand-in synthesiser file by file
(`note_events_to_midi(...).synthesize(fs)`, NumPy on the host) against the GPU render of the whole batch
(`note_creation.sonify_batch`, csrc/sonify.cu), each with and without writing the WAV files to a temporary directory.

Workload: 256 x 10 s `random_notes_clip` clips transcribed once (pitch bends included), rendered at 44.1 kHz.  Prints one
JSON line with audio-seconds per second, the note count and the device name and power limit read in the same run.

`--compare-with ROOT`: also times `predict_and_save` over 64 x 10 s WAV files with sonify_midi=True, the package under ROOT
(for example a built checkout of an earlier commit) against this tree, alternating the two in fresh processes."""
import argparse
import json
import os
import pathlib
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = pathlib.Path(__file__).resolve().parent.parent


def device_info():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"device": name, "power_limit": power}


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts))


def sonify_bench(n_clips, seconds, fs, reps):
    from scipy.io import wavfile

    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, synth
    from basic_pitch_b200 import note_creation as nc
    from basic_pitch_b200.inference import Model

    model = Model(ICASSP_2022_MODEL_PATH)
    clips = [synth.random_notes_clip(seconds, seed=1000 + i) for i in range(n_clips)]
    _outs, arrs, _frames = model.transcribe_arrays(clips, return_model_output=False, split_notes=False)
    events = nc.note_events_batch(arrs, n_clips)
    n_notes = int(sum(len(e) for e in events))
    with tempfile.TemporaryDirectory() as tmp:
        paths = [os.path.join(tmp, f"c{i}.wav") for i in range(n_clips)]

        def standin(write):
            for ev, p in zip(events, paths):
                y = nc.note_events_to_midi(ev.to_list(), False).synthesize(fs)
                if write:
                    wavfile.write(p, fs, y)

        def gpu(write):
            ys = nc.sonify_batch(events, fs, False, model)
            if write:
                for y, p in zip(ys, paths):
                    wavfile.write(p, fs, y)
            return ys

        audio_s = sum(len(y) for y in gpu(False)) / fs  # rendered seconds (each file is its notes' end + 1 s)
        for _ in range(2):
            gpu(True)
        t = {
            "standin": timed(lambda: standin(False), 1),
            "standin_wav": timed(lambda: standin(True), 1),
            "gpu": timed(lambda: gpu(False), reps),
            "gpu_wav": timed(lambda: gpu(True), reps),
        }
    out = {"clips": n_clips, "clip_seconds": seconds, "fs": fs, "notes": n_notes, "rendered_audio_s": audio_s}
    for k, v in t.items():
        out[f"{k}_ms"] = 1e3 * v
        out[f"{k}_audio_s_per_s"] = audio_s / v
    return out


def predict_and_save_once(wav_dir, reps):
    """One process: predict_and_save over the WAV files of wav_dir with sonify_midi=True (and MIDI / CSV), median of reps."""
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200 import inference as inf

    model = inf.Model(ICASSP_2022_MODEL_PATH)
    paths = sorted(pathlib.Path(wav_dir).glob("*.wav"))
    devnull = open(os.devnull, "w")

    def run():
        with tempfile.TemporaryDirectory() as out:
            stdout, sys.stdout = sys.stdout, devnull
            try:
                inf.predict_and_save(paths, out, True, True, False, True, model)
            finally:
                sys.stdout = stdout

    run()  # warm-up
    return timed(run, reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=10.0)
    ap.add_argument("--fs", type=int, default=44100)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--compare-with", default=None, help="root of another tree whose package to time against this one")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--pas-files", type=int, default=64)
    ap.add_argument("--_pas", default=None, help=argparse.SUPPRESS)  # child process: time predict_and_save on this dir
    args = ap.parse_args()
    if args._pas:
        print(json.dumps({"ms": 1e3 * predict_and_save_once(args._pas, 2)}))
        return
    sys.path.insert(0, str(HERE))
    out = device_info()
    out.update(sonify_bench(args.clips, args.seconds, args.fs, args.reps))
    if args.compare_with:
        from scipy.io import wavfile

        from basic_pitch_b200 import synth

        roots = {"parent": pathlib.Path(args.compare_with).resolve(), "this": HERE}
        times = {k: [] for k in roots}
        with tempfile.TemporaryDirectory() as wav_dir:
            for i in range(args.pas_files):
                clip = synth.random_notes_clip(args.seconds, seed=5000 + i)
                wavfile.write(os.path.join(wav_dir, f"f{i:03d}.wav"), 22050, (clip * 20000).astype(np.int16))
            for _ in range(args.rounds):
                for k, root in roots.items():
                    env = dict(os.environ, PYTHONPATH=str(root))
                    r = subprocess.run([sys.executable, str(pathlib.Path(__file__).resolve()), "--_pas", wav_dir],
                                       cwd=str(root), env=env, capture_output=True, text=True, check=True)
                    times[k].append(json.loads(r.stdout.strip().splitlines()[-1])["ms"])
        out["predict_and_save_sonify"] = {
            "files": args.pas_files, "clip_seconds": args.seconds,
            **{f"{k}_ms": v for k, v in times.items()},
            **{f"{k}_median_ms": float(np.median(v)) for k, v in times.items()},
        }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
