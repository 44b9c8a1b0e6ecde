"""GPU: every metric family of a batch in one device pass (bp_evaluate_*, csrc/api.cu; Model.evaluate,
inference.evaluate_all).  Every count must equal, exactly, what the standalone grid call of its family returns for the
same posteriorgrams, settings and references."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_decode_edges import _set
from tests.test_gpu_decode_grid import _model_grid
from tests.test_gpu_note_f0 import _base_times, edges, model, model_case  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

FAMILIES = ("notes", "onset_offset", "pairs", "frames", "bent_frames", "note_melody", "flat_note_melody", "salience",
            "melody")
SAL = [dict(threshold=0.3), dict(threshold=0.5, peak_picking=False, minimum_frequency=100.0, maximum_frequency=900.0)]
MEL = [dict(threshold=0.3), dict(threshold=0.5, guess_unvoiced=False, minimum_frequency=100.0)]


def _note_refs(model, notes, onsets, contours):
    """Reference notes per file: the notes of one fixed setting, with file 1's set empty."""
    from basic_pitch_b200 import note_creation as infer

    res = model.decode_grid(notes, onsets, contours, [dict(onset_thresh=0.6, frame_thresh=0.35)])[0]
    refs = []
    for i, r in enumerate(res):
        t = infer.model_frames_to_time(notes[i].shape[0] + 1)
        iv = np.stack([t[r["start"]], t[r["end"]]], 1) if len(r["start"]) else np.zeros((0, 2))
        hz = 440.0 * 2.0 ** ((r["pitch"] - 69) / 12.0)
        refs.append((iv, hz) if i != 1 else (np.zeros((0, 2)), np.zeros(0)))
    return refs


def _standalone(model, notes, onsets, contours, settings, nrefs, mp, mel, fams=FAMILIES):
    flat = [{**s, "include_pitch_bends": False} for s in settings]
    out = {}
    if "notes" in fams:
        out["notes"] = model.score_grid(notes, onsets, settings, nrefs)
    if "onset_offset" in fams:
        out["onset_offset"] = model.score_onset_offset_grid(notes, onsets, settings, [r[0] for r in nrefs])
    if "pairs" in fams:
        out["pairs"] = model.match_grid(notes, onsets, settings, nrefs)
    if "frames" in fams:
        out["frames"] = model.score_frames_grid(notes, onsets, settings, mp)
    if "bent_frames" in fams:
        out["bent_frames"] = model.score_frames_grid(notes, onsets, settings, mp, contours=contours)
    if "note_melody" in fams:
        out["note_melody"] = model.score_note_melody_grid(notes, onsets, contours, settings, mel)
    if "flat_note_melody" in fams:
        out["flat_note_melody"] = model.score_note_melody_grid(notes, onsets, None, flat, mel)
    if "salience" in fams:
        out["salience"] = model.score_salience_grid(notes, SAL, mp, kind="note")
    if "melody" in fams:
        out["melody"] = model.score_melody_grid(contours, MEL, mel, kind="contour")
    return out


def _request(nrefs, mp, mel):
    return dict(note_refs=nrefs, multipitch_refs=mp, f0_refs=mel, salience=dict(settings=SAL, kind="note", references=mp),
                melody=dict(settings=MEL, kind="contour", references=mel))


def _assert_same(got, exp):
    for k, v in exp.items():
        if k == "pairs":
            res, match = got[k]
            for a, b in zip(res, v[0]):
                for x, y in zip(a, b):
                    for key in ("start", "end", "pitch", "amp", "bend_off"):
                        assert x[key].tobytes() == y[key].tobytes(), key
            for a, b in zip(match, v[1]):
                for x, y in zip(a, b):
                    np.testing.assert_array_equal(x, y)
        else:
            assert got[k].tobytes() == v.tobytes(), k


@pytest.fixture(scope="module")
def case(model, model_case):
    items, outs = model_case
    notes, onsets, contours = ([o[k] for o in outs] for k in ("note", "onset", "contour"))
    ts = [_base_times("hop58", a.shape[0], None) for a in notes]
    mp = [(t, f(t)) for t, (_, f, _) in zip(ts, items)]
    mel = [(t, f(t)) for t, (_, _, f) in zip(ts, items)]
    return notes, onsets, contours, _note_refs(model, notes, onsets, contours), mp, mel


def test_every_family_equals_its_standalone_call(model, case):
    """>= 48 settings (thresholds, min_note_len, melodia, ranges, bends) on the vocadito clip, synth clips, an empty
    clip and a file with empty references."""
    notes, onsets, contours, nrefs, mp, mel = case
    settings = _model_grid()
    assert len(settings) >= 48
    exp = _standalone(model, notes, onsets, contours, settings, nrefs, mp, mel)
    got = model.evaluate(FAMILIES, settings, grams=(notes, onsets, contours), **_request(nrefs, mp, mel))
    _assert_same(got, exp)
    assert exp["notes"][..., 3].sum() > 0 and exp["bent_frames"][..., 2].sum() > 0 and exp["melody"][..., 4].sum() > 0


def test_family_subsets(model, case):
    notes, onsets, contours, nrefs, mp, mel = case
    settings = _model_grid()[::6]
    exp = _standalone(model, notes, onsets, contours, settings, nrefs, mp, mel)
    for fams in [[f] for f in FAMILIES] + [[f for f in FAMILIES if f != g] for g in FAMILIES]:
        got = model.evaluate(fams, settings, grams=(notes, onsets, contours), **_request(nrefs, mp, mel))
        assert set(got) == set(fams)
        _assert_same(got, {k: exp[k] for k in fams})


def test_device_on_a_caller_stream_equals_host(model, case):
    import torch

    notes, onsets, contours, nrefs, mp, mel = case
    settings = _model_grid()[::5]
    dev = f"cuda:{model.device}"
    d = [torch.from_numpy(np.ascontiguousarray(np.concatenate(x), np.float32)).to(dev) for x in (notes, onsets, contours)]
    foff = np.cumsum([0] + [a.shape[0] for a in notes]).astype(np.int64)
    stream = torch.cuda.Stream(device=dev)
    torch.cuda.synchronize(dev)
    with torch.cuda.stream(stream):
        got = model.evaluate(FAMILIES, settings, grams=(*d, foff), stream=stream.cuda_stream, **_request(nrefs, mp, mel))
    exp = model.evaluate(FAMILIES, settings, grams=(notes, onsets, contours), **_request(nrefs, mp, mel))
    _assert_same(got, {k: v for k, v in exp.items()})


def test_forced_chunking_and_launch_count(model, edges):  # noqa: F811
    base = []
    for name in ("ties", "long_notes", "nan_file", "runs"):
        base += _set(edges, name)[0]
    files = []
    while sum(f[0].shape[0] for f in files) < 120_000:
        files += base
    notes, onsets, contours = ([f[k] for f in files] for k in range(3))
    lens = [a.shape[0] for a in notes]
    mp = [(np.arange(0, n * 256 / 22050, 0.01), None) for n in lens]
    mp = [(t, [np.array([261.63, 392.0])] * len(t)) for t, _ in mp]
    mel = [(t, np.where(np.arange(len(t)) % 7 == 0, 0.0, 261.63)) for t, _ in mp]
    nrefs = [(np.array([[0.1, 0.5]]), np.array([261.63]))] * len(files)
    fams = [f for f in FAMILIES if f != "pairs"]  # the matching's launches depend on the notes
    req = _request(nrefs, mp, mel)
    distinct = [dict(onset_thresh=0.5, frame_thresh=0.3), dict(frame_thresh=0.05, min_note_len=0, infer_onsets=False),
                dict(onset_thresh=0.95, min_note_len=1, energy_tol=64, include_pitch_bends=False),
                dict(onset_thresh=0.0, melodia_trick=False), dict(min_pitch_idx=20, max_pitch_idx=70)]
    chunk = model.evaluate_chunk_params(sum(lens), fams, distinct, **req)
    settings = [distinct[k % len(distinct)] for k in range(chunk + 3)]
    n_chunks = -(-len(settings) // chunk)
    assert n_chunks >= 2, chunk
    per_chunk = 3 + 1 + 1 + 3 + 3 + 4 + 4  # decode, notes, onset_offset, frames, bent_frames, two note melodies
    posterior = 1 + 3  # one salience chunk, one melody chunk
    before = model.launch_count
    got = model.evaluate(fams, settings, grams=(notes, onsets, contours), **req)
    assert model.launch_count - before == per_chunk * n_chunks + posterior
    standalone = 0
    for k0 in range(0, len(settings), chunk):
        part = settings[k0 : k0 + chunk]
        before = model.launch_count
        exp = _standalone(model, notes, onsets, contours, part, nrefs, mp, mel, fams)
        standalone += model.launch_count - before
        for f in fams:
            if f in ("salience", "melody"):
                assert got[f].tobytes() == exp[f].tobytes(), f
            else:
                assert got[f][k0 : k0 + chunk].tobytes() == exp[f].tobytes(), (f, k0)
    assert per_chunk * n_chunks + posterior < standalone


def test_invalid_requests_are_rejected_by_family_without_a_launch(model):
    from basic_pitch_b200 import _lib

    T = 6
    notes = [np.zeros((T, 88), np.float32)] * 3
    contours = [np.zeros((T, 264), np.float32)] * 3
    mp = [(np.array([0.0, 0.01]), [np.array([220.0]), np.zeros(0)])] * 3
    mel = [(np.array([0.0, 0.1]), np.array([220.0, 0.0]))] * 3
    nrefs = [(np.array([[0.1, 0.2]]), np.array([220.0]))] * 3
    good = _request(nrefs, mp, mel)
    before = model.launch_count

    def ev(settings=(dict(),), fams=FAMILIES, **kw):
        model.evaluate(fams, list(settings), grams=(notes, notes, contours), **{**good, **kw})

    bad_mp = [mp[0], mp[0], (np.array([0.0, -0.1]), [np.zeros(0)] * 2)]
    cases = [
        (lambda: ev(settings=[dict(), dict(energy_tol=0)]), r"bp_evaluate_host: decode params\[1\]: energy_tol"),
        (lambda: ev(note_refs=[nrefs[0], (np.array([[0.3, 0.2]]), np.array([220.0])), nrefs[0]]),
         "bp_evaluate_host: notes: references file 1 note 0: offset <= onset"),
        (lambda: ev(fams=["onset_offset"], note_refs=[nrefs[0], nrefs[0], (np.array([[-0.1, 0.2]]), np.array([1.0]))]),
         "bp_evaluate_host: onset_offset: references file 2 note 0: onset < 0"),
        (lambda: ev(fams=["frames"], multipitch_refs=bad_mp), "bp_evaluate_host: frames: references file 2 frame 1: time < 0"),
        (lambda: ev(fams=["bent_frames"], window=-1.0), "bp_evaluate_host: bent_frames: window must be finite"),
        (lambda: ev(fams=["note_melody"], cent_tolerance=0.0), "bp_evaluate_host: note_melody: cent_tolerance"),
        (lambda: ev(fams=["flat_note_melody"], f0_refs=[mel[0], (np.array([0.1, 0.05]), np.array([1.0, 1.0])), mel[0]]),
         "bp_evaluate_host: flat_note_melody: references file 1 frame 1: time decreases"),
        (lambda: ev(salience=dict(settings=[SAL[0], dict(threshold=-1.0)], references=mp)),
         r"bp_evaluate_host: salience: salience params\[1\]: threshold"),
        (lambda: ev(melody=dict(settings=[dict(threshold=np.inf)], references=mel)),
         r"bp_evaluate_host: melody: melody params\[0\]: threshold"),
    ]
    for call, msg in cases:
        with pytest.raises(_lib.BpError, match=msg) as e:
            call()
        assert e.value.code == _lib.BP_E_INVALID
    assert model.launch_count == before


def _wav_files(golden_dir, tmp_path):
    from scipy.io import wavfile

    zp = np.load(golden_dir / "vocadito10_pcm44k.npz")
    pcm = zp["pcm"]
    stereo = np.stack([pcm, pcm[::-1]], 1) if pcm.ndim == 1 else pcm
    paths = [tmp_path / "a.wav", tmp_path / "b.wav", tmp_path / "c.wav"]
    wavfile.write(paths[0], int(zp["sample_rate"]), stereo.astype(np.int16))  # int16 stereo 44.1 kHz
    mono = (pcm.reshape(len(pcm), -1).mean(axis=1) / 32768.0).astype(np.float32)
    wavfile.write(paths[1], 22050, mono[: len(mono) // 2])  # float32 mono 22.05 kHz
    wavfile.write(paths[2], 16000, (np.clip(mono[:80000] * 100 + 128, 0, 255)).astype(np.uint8))  # uint8
    return paths


def test_audio_entries_and_evaluate_all(model, golden_dir, tmp_path):
    """evaluate_all from WAV paths (stored-PCM pipeline) and from arrays (packed) equals each evaluate_* function; the
    returned posteriorgrams equal run_inference_arrays."""
    from basic_pitch_b200 import inference, synth
    from basic_pitch_b200.audio_io import load_audio_device

    paths = _wav_files(golden_dir, tmp_path)
    clip = synth.melody_clip(6.0, 51)
    arrays = [load_audio_device(p, model)[0] for p in paths] + [clip]
    outs = model.run_inference_arrays(arrays)
    notes, onsets, contours = ([o[k] for o in outs] for k in ("note", "onset", "contour"))
    ts = [np.arange(0.01, a.shape[0] * 256 / 22050, 0.01) for a in notes]
    mel = [(t, np.where(np.sin(7 * t) > 0, 261.63 * (1 + 0.3 * np.sin(t)), 0.0)) for t in ts]
    mp = [(t, [np.array([f]) if f > 0 else np.zeros(0) for f in f0]) for t, f0 in mel]
    nr = _note_refs(model, notes, onsets, contours)
    rng = np.random.default_rng(5)
    nrefs = [(iv, hz, rng.uniform(0, 127, len(hz))) for iv, hz in nr]
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2, minimum_note_length=58.0),
                dict(minimum_frequency=150.0, maximum_frequency=700.0), dict(melodia_trick=False)]
    sal = dict(settings=SAL, kind="contour")
    melo = dict(settings=MEL, kind="note")
    for src in (paths + [clip], arrays):
        got = inference.evaluate_all(src, settings, notes=nrefs, multipitch=mp, f0=mel, salience=sal, melody=melo,
                                     model_or_model_path=model, return_model_output=True)
        assert set(got) == set(inference.EVALUATE_FAMILIES) | {"model_output"}
        for o, e in zip(got["model_output"], outs):
            for k in ("note", "onset", "contour"):
                assert o[k].tobytes() == e[k].tobytes(), k
        pitched = [(iv, hz) for iv, hz, _ in nrefs]
        exp = {
            "notes": inference.evaluate_grid(src, pitched, settings, model),
            "transcription": inference.evaluate_transcription_grid(src, pitched, settings, model),
            "velocity": inference.evaluate_velocity_grid(src, nrefs, settings, model),
            "frames": inference.evaluate_frames_grid(src, mp, settings, model),
            "bent_frames": inference.evaluate_frames_grid(src, mp, settings, model, pitch_bends=True),
            "note_melody": inference.evaluate_note_melody_grid(src, mel, settings, model),
            "flat_note_melody": inference.evaluate_note_melody_grid(src, mel, settings, model, pitch_bends=False),
            "salience": inference.evaluate_salience_grid(src, mp, SAL, kind="contour", model_or_model_path=model),
            "melody": inference.evaluate_melody_grid(src, mel, MEL, kind="note", model_or_model_path=model),
        }
        for fam, (counts, scores) in exp.items():
            assert got[fam][0].tobytes() == counts.tobytes(), fam
            for k, v in scores.items():
                if k == "mean":
                    for kk, vv in v.items():
                        assert np.asarray(got[fam][1]["mean"][kk]).tobytes() == np.asarray(vv).tobytes(), (fam, kk)
                else:
                    assert np.asarray(got[fam][1][k]).tobytes() == np.asarray(v).tobytes(), (fam, k)
