#!/usr/bin/env python
"""ORACLE tooling — generate tests/golden/*.npz by running the UNMODIFIED reference modules.

Runs only in the build container (needs /root/reference).  The reference's third-party imports are
satisfied by oracle/ref_shims (librosa / pretty_midi / mir_eval / resampy stand-ins, and an
`onnxruntime` stand-in whose arithmetic is oracle/model_ref.py), so every line of the reference's
`inference.py` host logic and `note_creation.py` decode executes as shipped.

    python oracle/make_golden.py                  # rewrites tests/golden/*.npz
    python oracle/make_golden.py decode_edges     # rewrites tests/golden/decode_edges.npz only (byte-reproducible)

Fixtures written (all small, committed):
  vocadito10_pcm44k.npz the same clip as stored in the reference's test resources (44.1 kHz int16 mono): ingest tests
  vocadito10.npz        reference golden posteriorgrams/events (tests/resources/vocadito_10/*.npz),
                        the 22 050 Hz audio they are checked with, and the events the reference
                        decode emits for the golden posteriorgrams under several parameter sets
  decode_cases.npz      posteriorgram inputs (uint16-quantised) + reference decode outputs
  host_cases.npz        window counts / unwrap lengths from the reference's windowing code
  predict_2s.npz        config-1 clip: int16 audio + reference predict() outputs (fake-ORT oracle model)
  decode_edges.npz      reference decode outputs on the adversarial posteriorgram sets of tests/postsets.py
"""
import hashlib
import io
import pathlib
import sys
import warnings

import numpy as np

ROOT = pathlib.Path(__file__).resolve().parent.parent
REF = pathlib.Path("/root/reference")
sys.path[:0] = [str(ROOT / "oracle" / "ref_shims"), str(REF), str(ROOT)]

import basic_pitch  # noqa: E402  (the reference package)

assert str(REF) in basic_pitch.__file__, basic_pitch.__file__
from basic_pitch import inference as ref_inf  # noqa: E402
from basic_pitch import note_creation as ref_nc  # noqa: E402

from basic_pitch_b200 import synth, weights  # noqa: E402
from oracle import model_ref, host_ref  # noqa: E402

GOLD = ROOT / "tests" / "golden"
ONNX = REF / "basic_pitch/saved_models/icassp_2022/nmp.onnx"
RES = REF / "tests/resources"


def quant(a: np.ndarray) -> np.ndarray:
    return np.clip(np.round(a.astype(np.float64) * 65535.0), 0, 65535).astype(np.uint16)


def dequant(q: np.ndarray) -> np.ndarray:
    return q.astype(np.float32) / np.float32(65535.0)


def pack_events(events):
    """events: list of (start, end, pitch, amp, bends|None) -> dict of arrays."""
    n = len(events)
    starts = np.array([e[0] for e in events], dtype=np.float64).reshape(n)
    ends = np.array([e[1] for e in events], dtype=np.float64).reshape(n)
    pitch = np.array([e[2] for e in events], dtype=np.int32).reshape(n)
    amp = np.array([e[3] for e in events], dtype=np.float32).reshape(n)
    off = [0]
    flat = []
    has = np.zeros(n, dtype=np.uint8)
    for i, e in enumerate(events):
        b = e[4] if len(e) > 4 else None
        if b is not None:
            has[i] = 1
            flat.extend(int(v) for v in b)
        off.append(len(flat))
    return {
        "start": starts,
        "end": ends,
        "pitch": pitch,
        "amp": amp,
        "bend_flat": np.array(flat, dtype=np.int32),
        "bend_off": np.array(off, dtype=np.int32),
        "bend_has": has,
    }


def ref_decode(post, **kw):
    """Run the reference decode on copies (it mutates its inputs in place)."""
    out = {k: np.array(v, copy=True) for k, v in post.items()}
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        frames_notes = ref_nc.output_to_notes_polyphonic(
            np.array(out["note"], copy=True),
            np.array(out["onset"], copy=True),
            onset_thresh=kw.get("onset_thresh", 0.5),
            frame_thresh=kw.get("frame_thresh", 0.3),
            infer_onsets=kw.get("infer_onsets", True),
            min_note_len=kw.get("min_note_len", 11),
            min_freq=kw.get("min_freq"),
            max_freq=kw.get("max_freq"),
            melodia_trick=kw.get("melodia_trick", True),
        )
        _midi, events = ref_nc.model_output_to_notes(
            out,
            onset_thresh=kw.get("onset_thresh", 0.5),
            frame_thresh=kw.get("frame_thresh", 0.3),
            infer_onsets=kw.get("infer_onsets", True),
            min_note_len=kw.get("min_note_len", 11),
            min_freq=kw.get("min_freq"),
            max_freq=kw.get("max_freq"),
            include_pitch_bends=True,
            multiple_pitch_bends=kw.get("multiple_pitch_bends", False),
            melodia_trick=kw.get("melodia_trick", True),
        )
    fr = np.array([[a, b, p] for a, b, p, _ in frames_notes], dtype=np.int32).reshape(-1, 3)
    return fr, events


PARAM_SETS = [
    dict(),
    dict(onset_thresh=0.3, frame_thresh=0.3, min_note_len=5),
    dict(onset_thresh=0.8, frame_thresh=0.1),
    dict(onset_thresh=0.5, frame_thresh=0.0),
    dict(onset_thresh=0.0, frame_thresh=0.5),
    dict(melodia_trick=False),
    dict(infer_onsets=False),
    dict(min_freq=110.0, max_freq=880.0),
    dict(onset_thresh=0.6, frame_thresh=0.4, min_note_len=20, melodia_trick=True, max_freq=2000.0),
]


def add_case(store, name, post, params):
    fr, events = ref_decode(post, **params)
    pe = pack_events(events)
    store[f"{name}/frames"] = fr
    for k, v in pe.items():
        store[f"{name}/{k}"] = v
    store[f"{name}/params"] = np.array(
        [
            params.get("onset_thresh", 0.5),
            params.get("frame_thresh", 0.3),
            params.get("min_note_len", 11),
            1.0 if params.get("infer_onsets", True) else 0.0,
            1.0 if params.get("melodia_trick", True) else 0.0,
            params["min_freq"] if params.get("min_freq") is not None else -1.0,
            params["max_freq"] if params.get("max_freq") is not None else -1.0,
        ],
        dtype=np.float64,
    )
    return len(events)


def smooth_fuzz(rng, n_t, n_f, density):
    """Blobby random activations in [0,1]: sparse impulses smoothed along time."""
    a = (rng.random((n_t + 40, n_f)) < density / 20.0).astype(np.float64) * rng.random((n_t + 40, n_f))
    k = np.exp(-np.arange(40) / rng.uniform(4, 12))
    out = np.zeros((n_t, n_f))
    for f in range(n_f):
        out[:, f] = np.convolve(a[:, f], k)[40 : 40 + n_t]
    out += 0.05 * rng.random((n_t, n_f))
    return np.clip(out, 0, 1).astype(np.float32)


def main() -> None:
    GOLD.mkdir(parents=True, exist_ok=True)
    w = weights.extract_from_onnx(ONNX)

    # ---------------------------------------------------------------- A. vocadito golden
    import librosa  # the shim

    wav = RES / "vocadito_10.wav"
    audio22k, _ = librosa.load(str(wav), sr=22050, mono=True)
    gold_out = np.load(RES / "vocadito_10/model_output.npz", allow_pickle=True)["arr_0"].item()
    gold_ev = np.load(RES / "vocadito_10/note_events.npz", allow_pickle=True)["arr_0"]
    model = ref_inf.Model(ONNX)
    assert model.model_type == ref_inf.Model.MODEL_TYPES.ONNX
    out, _midi, events = ref_inf.predict(str(wav), model)
    for k in ("note", "onset", "contour"):
        assert out[k].shape == gold_out[k].shape, (k, out[k].shape)
        print(f"reference predict() via oracle model vs golden {k}: max-abs {np.abs(out[k] - gold_out[k]).max():.3e}")
    print(f"events: reference-run {len(events)}  golden {len(gold_ev)}")
    store = {
        "audio22k": audio22k.astype(np.float32),
        "gold_note": gold_out["note"].astype(np.float32),
        "gold_onset": gold_out["onset"].astype(np.float32),
        "gold_contour": gold_out["contour"].astype(np.float32),
    }
    for k, v in pack_events([tuple(r) for r in gold_ev]).items():
        store[f"gold_events/{k}"] = v
    post = {k: gold_out[k] for k in ("note", "onset", "contour")}
    for i, p in enumerate(PARAM_SETS):
        n = add_case(store, f"decode{i}", post, p)
        print(f"  vocadito decode{i} {p}: {n} events")
    fr0 = store["decode0/frames"]
    assert len(fr0) == len(gold_ev)
    assert np.array_equal(store["decode0/pitch"], store["gold_events/pitch"])
    assert np.array_equal(store["decode0/bend_flat"], store["gold_events/bend_flat"])
    np.savez_compressed(GOLD / "vocadito10.npz", **store)
    # the clip as stored (44.1 kHz, 16-bit mono): input of the device ingest tests (csrc/ingest.cu)
    from scipy.io import wavfile

    sr44, pcm = wavfile.read(str(wav))
    assert sr44 == 44100 and pcm.dtype == np.int16 and pcm.ndim == 1
    np.savez_compressed(GOLD / "vocadito10_pcm44k.npz", pcm=pcm, sample_rate=np.int32(sr44))

    # ---------------------------------------------------------------- B. decode cases
    store = {}
    names = []
    rng = np.random.default_rng(1234)

    def add_post(name, post, param_sets):
        q = {k: quant(post[k]) for k in ("note", "onset", "contour")}
        dq = {k: dequant(v) for k, v in q.items()}
        for k, v in q.items():
            store[f"{name}/{k}_q"] = v
        for i, p in enumerate(param_sets):
            n = add_case(store, f"{name}/p{i}", dq, p)
            names.append(f"{name}/p{i}")
            print(f"  {name}/p{i} {p}: {n} events")

    clip = synth.random_notes_clip(10.0, seed=3)
    win = host_ref.window_audio(clip)
    o = model_ref.forward_batched(win, w)
    post = {k: host_ref.unwrap(o[k], len(clip)) for k in o}
    add_post("notes10s", post, PARAM_SETS)

    clip = synth.dense_chords_clip(4.0, seed=7)
    win = host_ref.window_audio(clip)
    o = model_ref.forward_batched(win, w)
    post = {k: host_ref.unwrap(o[k], len(clip)) for k in o}
    add_post("chords4s", post, PARAM_SETS[:4])

    for j, (n_t, dens) in enumerate([(300, 0.3), (257, 1.0), (64, 2.0)]):
        post = {
            "note": smooth_fuzz(rng, n_t, 88, dens),
            "onset": smooth_fuzz(rng, n_t, 88, dens * 0.5),
            "contour": smooth_fuzz(rng, n_t, 264, dens),
        }
        add_post(f"fuzz{j}", post, PARAM_SETS[:6])

    # silence-like: constant in time -> max(frame_diff) == 0 -> NaN path (SURVEY Appendix B.2)
    post = {
        "note": np.full((200, 88), 0.12, np.float32),
        "onset": np.full((200, 88), 0.05, np.float32),
        "contour": np.full((200, 264), 0.1, np.float32),
    }
    add_post("constant", post, [dict(), dict(onset_thresh=0.0, frame_thresh=0.1), dict(frame_thresh=0.1, infer_onsets=False)])

    for n_t in (1, 2, 3, 12, 13, 25):
        post = {
            "note": smooth_fuzz(rng, n_t, 88, 3.0),
            "onset": smooth_fuzz(rng, n_t, 88, 3.0),
            "contour": smooth_fuzz(rng, n_t, 264, 3.0),
        }
        add_post(f"tiny{n_t}", post, [dict(), dict(onset_thresh=0.0, frame_thresh=0.05, min_note_len=1)])
    store["names"] = np.array(names)
    np.savez_compressed(GOLD / "decode_cases.npz", **store)

    # ---------------------------------------------------------------- C. host logic
    lens = [1, 3840, 36163, 36164, 36165, 40004, 44100, 72328, 72329, 200607, 220500, 3969000]
    n_windows, n_frames = [], []
    hop = ref_inf.AUDIO_N_SAMPLES - 30 * ref_inf.FFT_HOP
    for n in lens:
        x = np.concatenate([np.zeros(3840, np.float32), np.zeros(n, np.float32)])
        nw = sum(1 for _ in ref_inf.window_audio_file(x, hop))
        fake = np.zeros((nw, 172, 2), np.float32)
        u = ref_inf.unwrap_output(fake, n, 30, hop)
        n_windows.append(nw)
        n_frames.append(u.shape[0])
    # content check on one ragged length
    x = np.arange(100000, dtype=np.float32) / 100000.0
    xw = np.concatenate([np.zeros(3840, np.float32), x])
    wins = np.concatenate([wd[None, :, 0] for wd, _ in ref_inf.window_audio_file(xw, hop)])
    np.savez_compressed(
        GOLD / "host_cases.npz",
        lens=np.array(lens),
        n_windows=np.array(n_windows),
        n_frames=np.array(n_frames),
        ramp_windows_sha=np.frombuffer(hashlib.sha256(wins.tobytes()).digest(), dtype=np.uint8),
        ramp_n_windows=np.array(wins.shape[0]),
    )
    print("host cases:", dict(zip(lens, zip(n_windows, n_frames))))

    # ---------------------------------------------------------------- D. config 1 through reference predict()
    from scipy.io import wavfile

    clip = synth.tones_clip(2.0, seed=0)
    pcm = np.clip(np.round(clip * 32767.0), -32768, 32767).astype(np.int16)
    tmp = pathlib.Path("/tmp/bp_cfg1.wav")
    wavfile.write(tmp, 22050, pcm)
    out, _midi, events = ref_inf.predict(str(tmp), model)
    store = {"pcm16": pcm, "note": out["note"], "onset": out["onset"], "contour": out["contour"]}
    for k, v in pack_events(events).items():
        store[f"events/{k}"] = v
    print(f"config-1 clip: {out['note'].shape[0]} frames, {len(events)} events")
    np.savez_compressed(GOLD / "predict_2s.npz", **store)

    decode_edges()
    for f in sorted(GOLD.glob("*.npz")):
        print(f"{f.name}: {f.stat().st_size} B")


def save_npz_reproducible(path: pathlib.Path, store) -> None:
    """np.savez_compressed with fixed member timestamps: the same arrays give the same bytes on every run."""
    import zipfile

    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for key in sorted(store):
            info = zipfile.ZipInfo(key + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(store[key]), allow_pickle=False)
            zf.writestr(info, buf.getvalue())


def column_range_as_freqs(lo: int, hi: int):
    """(min_freq, max_freq) that the reference's constrain_frequency turns into pitch columns [lo, hi)."""
    min_freq = None if lo == 0 else float(librosa_midi_to_hz(21 + lo))
    max_freq = None if hi == 88 else float(librosa_midi_to_hz(21 + hi))
    for f, col in ((min_freq, lo), (max_freq, hi)):
        assert f is None or int(np.round(ref_nc.librosa.hz_to_midi(f) - 21)) == col, (f, col)
    return min_freq, max_freq


def librosa_midi_to_hz(m):
    return ref_nc.librosa.midi_to_hz(m)


def decode_edges() -> None:
    """tests/golden/decode_edges.npz: the reference decode (`output_to_notes_polyphonic` with `energy_tol`,
    `get_pitch_bends`, `model_frames_to_time`) on every file and parameter set of tests/postsets.py.  The inputs are
    regenerated from tests/postsets.py (seeded) and identified by a SHA-256 per file; the outputs are stored per set and
    parameter set, concatenated over the files of the set (note_off[i] .. note_off[i + 1] are file i's notes), in the
    narrowest exact dtypes: start / end / pitch frames int16, bends int8 (|bend| <= 25), amplitudes float32.  Every note has end - start
    bends, so the bend offsets follow from the frames.  Frame times depend on the frame index only: one array for the
    longest file serves every file.

        python oracle/make_golden.py decode_edges     # this fixture only
    """
    from tests import postsets

    store = {}
    max_t = 0
    for name in postsets.NAMES:
        files, grid = postsets.get(name)
        store[f"{name}/sha"] = np.stack([np.frombuffer(postsets.file_sha(f), np.uint8) for f in files])
        store[f"{name}/T"] = np.array([f[0].shape[0] for f in files], np.int64)
        max_t = max([max_t] + [f[0].shape[0] for f in files])
        for j, p in enumerate(grid):
            min_freq, max_freq = column_range_as_freqs(p["lo_col"], p["hi_col"])
            frames, amp, flat, noff = [], [], [], [0]
            for note, onset, contour in postsets.get(name)[0]:
                notes = []
                if note.shape[0] > 0:  # the reference cannot take an empty file (np.max of nothing); it has no notes
                    with warnings.catch_warnings():
                        warnings.simplefilter("ignore")
                        notes = ref_nc.output_to_notes_polyphonic(
                            note, onset, onset_thresh=p["onset_thresh"], frame_thresh=p["frame_thresh"],
                            min_note_len=p["min_note_len"], infer_onsets=p["infer_onsets"], max_freq=max_freq,
                            min_freq=min_freq, melodia_trick=p["melodia_trick"], energy_tol=p["energy_tol"],
                        )
                        notes = ref_nc.get_pitch_bends(contour, notes)
                for a, b, pitch, am, bends in notes:
                    assert len(bends) == b - a
                    frames.append((a, b, pitch))
                    amp.append(am)
                    flat.extend(int(v) for v in bends)
                noff.append(len(frames))
            key = f"{name}/p{j}"
            store[f"{key}/params"] = np.array(
                [p["onset_thresh"], p["frame_thresh"], p["min_note_len"], p["energy_tol"], p["infer_onsets"],
                 p["melodia_trick"], p["lo_col"], p["hi_col"]], np.float64)  # fmt: skip
            fr = narrow(np.array(frames, np.int64).reshape(-1, 3), np.int16)
            for c, k in enumerate(("start", "end", "pitch")):  # one array per column: each compresses on its own
                store[f"{key}/{k}"] = np.ascontiguousarray(fr[:, c])
            store[f"{key}/amp"] = np.array(amp, np.float32)
            store[f"{key}/bend_flat"] = narrow(np.array(flat, np.int64), np.int8)
            store[f"{key}/note_off"] = np.array(noff, np.int32)
            print(f"  {key}: {np.diff(noff).tolist()} notes")
    store["times"] = np.asarray(ref_nc.model_frames_to_time(max_t), np.float64)
    # get_pitch_bends alone on the notes of pitch_edges (bp_pitch_bends_host)
    contour = postsets.get("pitch_edges")[0][0][2]
    wb = ref_nc.get_pitch_bends(contour, [(a, b, p, 0.5) for a, b, p in postsets.edge_notes()])
    store["pitch_edges/direct/bend_flat"] = narrow(np.array([int(v) for e in wb for v in e[4]], np.int64), np.int8)
    path = GOLD / "decode_edges.npz"
    save_npz_reproducible(path, store)
    print(f"{path.name}: {path.stat().st_size} B")


def narrow(a: np.ndarray, dtype) -> np.ndarray:
    """`a` in a narrower integer dtype, which must hold every value exactly."""
    out = a.astype(dtype)
    assert np.array_equal(out, a), dtype
    return out


if __name__ == "__main__":
    if sys.argv[1:] == ["decode_edges"]:
        decode_edges()
    else:
        main()
