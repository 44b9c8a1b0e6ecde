"""WAV files read by the library (`bp_probe_wav_files` + `bp_transcribe_pcm_sources_host` / `_evaluate_`, and through them
`predict_batch`, `predict_and_save` and `evaluate_all` on paths), and the two sample formats only whole WAV files bring to
the batched ingest: 4 packed 24-bit and 5 float64.

The contract is bit identity with the route every path took before: `read_pcm` on the host, then the stored-PCM pipeline
from memory.  That route is reached here by making the probe decline every file."""
import numpy as np
import pytest

from tests.test_gpu_ingest import RATES, assert_bits, make_pcm, write_wav24
from tests.test_gpu_pcm_batch import as_format, assert_same_notes, clip_batch, frames_for_outputs, interp_clip, shape_of


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH, device=0)


def decline_all(monkeypatch):
    """Today's route for every path: the probe declines, `read_pcm` reads."""
    from basic_pitch_b200 import inference

    monkeypatch.setattr(inference, "probe_wav", lambda paths: ([None] * len(paths), list(range(len(paths)))))


def count_calls(monkeypatch, lib, names):
    calls = {n: 0 for n in names}
    for n in names:
        real = getattr(lib, n)

        def wrapped(*a, _real=real, _n=n):
            calls[_n] += 1
            return _real(*a)

        monkeypatch.setattr(lib, n, wrapped)
    return calls


def write_wav(path, sr, pcm, fmt):
    """pcm as a WAV file of library format fmt (4: int32 values in [-2^23, 2^23) packed to 3 bytes)."""
    from scipy.io import wavfile

    if fmt == 4:
        write_wav24(path, sr, pcm if pcm.ndim == 2 else pcm[:, None])
    else:
        wavfile.write(path, sr, pcm)


def mixed_batch(model, tmp_path):
    """Paths of all six formats at several rates and channel counts (with an empty and a one-frame file), a file the
    probe declines (24-bit samples in 32-bit containers) and two arrays, spanning several sub-batches."""
    from basic_pitch_b200 import synth

    chunk = int(model._lib.bp_model_chunk_windows(model.handle))
    pcms, rates = clip_batch(12, 10.0 + 0.4 * chunk, seed=700)
    rng = np.random.default_rng(7)
    items, kinds = [], []
    for i, (x, sr) in enumerate(zip(pcms, rates)):
        fmt = {np.float32: 0, np.int16: 1, np.int32: 2, np.uint8: 3}[x.dtype.type]
        if i % 4 == 1 and x.dtype == np.int32:
            fmt, x = 4, x >> 8
        elif i % 4 == 3 and x.dtype == np.float32:
            fmt, x = 5, x.astype(np.float64) * 1.0000001
        p = tmp_path / f"f{i:02d}.wav"
        write_wav(p, sr, x, fmt)
        items.append(p)
        kinds.append(fmt)
    for fmt, sr, ch in ((4, 44100, 2), (5, 48000, 3), (4, 22050, 1), (5, 22050, 1)):
        n = 5 * sr + 11
        x = interp_clip(synth.random_notes_clip(6.0, seed=fmt + sr).astype(np.float64), n)
        x = as_format(x, np.int32 if fmt == 4 else np.float64, ch, rng)
        p = tmp_path / f"x{fmt}_{sr}_{ch}.wav"
        write_wav(p, sr, x >> 8 if fmt == 4 else x, fmt)
        items.append(p)
        kinds.append(fmt)
    dec = tmp_path / "declined.wav"  # 24-bit in a 4-byte container: scipy reads it, the probe declines it
    from tests.test_wav_probe_cpu import sample_bytes, wav_bytes

    x = as_format(interp_clip(synth.random_notes_clip(5.0, seed=9).astype(np.float64), 5 * 32000), np.int32, 2, rng)
    dec.write_bytes(wav_bytes(2, 2, 32000, sample_bytes(2, x & ~0xFF), bits=24, block=8))
    items.insert(3, dec)
    items.insert(1, synth.tones_clip(4.0, seed=3))
    items.insert(8, synth.random_notes_clip(7.0, seed=4).astype(np.float32))
    assert set(kinds) == set(range(6))
    return items, dec


@pytest.mark.gpu
def test_library_route_is_todays_route(model, tmp_path, monkeypatch):
    """predict_batch, predict_and_save and evaluate_all on a mixed batch: the same posteriorgrams, frame counts, notes,
    MIDI / CSV bytes and counts as when every path is read by `read_pcm`; one library call per batch, through the sources
    entry point."""
    from basic_pitch_b200 import audio_io, inference

    items, dec = mixed_batch(model, tmp_path)
    paths = [p for p in items if not isinstance(p, np.ndarray)]
    regions, declined = audio_io.probe_wav(paths)
    assert [paths[i] for i in declined] == [dec]
    lib = model._lib
    windows = sum(int(lib.bp_num_windows(int(lib.bp_resampled_length(r.n_frames, r.sample_rate)))) for r in regions if r)
    assert windows > 3 * int(lib.bp_model_chunk_windows(model.handle))  # several sub-batches

    names = ("bp_transcribe_pcm_sources_host", "bp_transcribe_pcm_files_host")
    with monkeypatch.context() as mp:
        calls = count_calls(mp, lib, names)
        got = inference.predict_batch(items, model, wav_in_library=True)
        assert calls == {names[0]: 1, names[1]: 0}
    with monkeypatch.context() as mp:
        calls = count_calls(mp, lib, names)
        want = inference.predict_batch(items, model)  # the default: every path through read_pcm
        assert calls == {names[0]: 0, names[1]: 1}
    assert len(got) == len(want) == len(items)
    for i, ((g_out, _gm, g_ev), (w_out, _wm, w_ev)) in enumerate(zip(got, want)):
        for k in ("note", "onset", "contour"):
            assert g_out[k].shape == w_out[k].shape, (i, k)
            assert np.array_equal(g_out[k].view(np.uint32), w_out[k].view(np.uint32)), (i, k)
        assert list(g_ev) == list(w_ev), i
    assert sum(len(list(ev)) for _o, _m, ev in want) > 0

    out = {}
    for route in ("library", "read_pcm"):
        d = tmp_path / route
        d.mkdir()
        with monkeypatch.context() as mp:
            if route == "read_pcm":
                decline_all(mp)
            inference.predict_and_save(paths, d, True, False, False, True, model)
        out[route] = {p.name: p.read_bytes() for p in sorted(d.iterdir())}
    assert len(out["library"]) == 2 * len(paths) and out["library"] == out["read_pcm"]

    refs = [(np.array([[0.5, 1.0], [1.5, 2.5]]), np.array([220.0, 440.0])) for _ in items]
    settings = [dict(), dict(onset_threshold=0.3, frame_threshold=0.2)]
    res = {}
    for route in ("library", "read_pcm"):
        with monkeypatch.context() as mp:
            if route == "read_pcm":
                decline_all(mp)
            res[route] = inference.evaluate_all(items, settings, notes=refs, model_or_model_path=model)
    assert np.array_equal(res["library"]["notes"][0], res["read_pcm"]["notes"][0])


def bytes_of(fmt, x):
    if fmt == 4:
        return np.ascontiguousarray(x.astype("<i4").reshape(-1).view(np.uint8).reshape(-1, 4)[:, :3]).reshape(-1)
    return x.reshape(-1)


@pytest.mark.gpu
def test_new_formats_are_their_wider_twins_bit_for_bit(model):
    """bp_load_pcm_sources_device: format 4 (packed 24-bit, 1-byte aligned) is format 2 of v << 8 and format 5
    (float64) is format 0 of float32(x), bit for bit, at 255 / 256 / 257 outputs and across many CTAs, at resampled
    and native rates and 1 / 2 / 7 channels, in one batch with their twins.  A source with a path is refused."""
    import torch

    lib = model._lib
    rng = np.random.default_rng(17)
    pcms, fmts, rates = [], [], []
    for sr in (22050, 44100, 48000, 8000, 96000):
        assert sr in RATES
        for n_out in (255, 256, 257, 3000):
            n = frames_for_outputs(sr, n_out) if sr >= 22050 else n_out * sr // 22050 + 1
            ch = (1, 2, 7)[(n_out + sr) % 3]
            v = make_pcm(np.int32, n, ch, "extremes" if n_out % 2 else "noise", sr, rng) >> 8
            x = rng.uniform(-1.5, 1.5, (n, ch) if ch > 1 else n) * np.exp2(rng.integers(-30, 3, (n, ch) if ch > 1 else n))
            x.reshape(-1)[:4] = (0.0, -0.0, 1e-40, 3.0000001)
            pcms += [v, v << 8, x, x.astype(np.float32)]
            fmts += [4, 2, 5, 0]
            rates += [sr] * 4
    dev = torch.device(f"cuda:{model.device}")
    blob = [torch.from_numpy(bytes_of(f, p).view(np.uint8).copy()).to(dev) for f, p in zip(fmts, pcms)]
    base = torch.zeros(sum(b.numel() for b in blob) + 16 * len(blob), dtype=torch.uint8, device=dev)
    ptrs, pos = [], 1  # every 24-bit file at an odd address
    for f, b in zip(fmts, blob):
        pos = pos + (-pos) % (8 if f in (0, 2, 5) else 1) + (1 if f == 4 and pos % 2 == 0 else 0)
        base[pos : pos + b.numel()] = b
        ptrs.append(base.data_ptr() + pos)
        pos += b.numel()
    from basic_pitch_b200 import _lib

    n = len(pcms)
    files = (_lib.PcmSource * n)()
    for s, x, k, sr, ptr in zip(files, pcms, fmts, rates, ptrs):
        f = s.pcm
        f.pcm, (f.n_frames, f.channels), f.sample_format, f.sample_rate = ptr, shape_of(x), k, sr
    off = np.zeros(n + 1, np.int64)
    total = sum(int(lib.bp_resampled_length(shape_of(p)[0], sr)) for p, sr in zip(pcms, rates))
    d_out = torch.zeros(total, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev)
    before = model.launch_count
    lib.bp_load_pcm_sources_device(model.handle, files, n, d_out.data_ptr(), off.ctypes.data, stream.cuda_stream)
    stream.synchronize()
    assert model.launch_count == before + 1
    got = d_out.cpu().numpy()
    files[3].path, files[3].data_offset = b"a.wav", 44  # a file on disk is not device memory
    before = model.launch_count
    with pytest.raises(_lib.BpError) as e:
        lib.bp_load_pcm_sources_device(model.handle, files, n, d_out.data_ptr(), off.ctypes.data, stream.cuda_stream)
    assert e.value.code == _lib.BP_E_INVALID and "file 3" in str(e.value) and model.launch_count == before
    assert {int(np.diff(off)[i]) for i in range(n)} >= {255, 256, 257, 3000}
    for i in range(0, n, 2):
        a, b = got[off[i] : off[i + 1]], got[off[i + 1] : off[i + 2]]
        assert len(a) == len(b) > 0
        assert_bits(a, b, (fmts[i], rates[i], shape_of(pcms[i])))


@pytest.mark.gpu
def test_file_truncated_after_the_probe(model, tmp_path):
    """A file that shrinks between the probe and the call raises OSError naming it; the model then gives the
    untouched batch's results bit for bit, and the sources of the same files in memory give them too."""
    from basic_pitch_b200 import audio_io

    pcms, rates = clip_batch(8, 20.0, seed=900)
    paths = []
    for i, (x, sr) in enumerate(zip(pcms, rates)):
        paths.append(tmp_path / f"t{i}.wav")
        write_wav(paths[-1], sr, x, {np.float32: 0, np.int16: 1, np.int32: 2, np.uint8: 3}[x.dtype.type])
    regions, declined = audio_io.probe_wav(paths)
    assert declined == []
    want_outs, want, _ = model.transcribe_pcm(list(zip(pcms, rates)), split_notes=False)
    want_outs = [{k: v.copy() for k, v in o.items()} for o in want_outs]
    got_outs, got, _ = model.transcribe_pcm(regions, split_notes=False)
    for g, w in zip(got_outs, want_outs):
        for k in w:
            assert np.array_equal(g[k].view(np.uint32), w[k].view(np.uint32)), k
    assert_same_notes(got, want, len(pcms), "before")
    k = max(range(len(regions)), key=lambda i: regions[i].n_frames)
    victim = paths[k]
    blob = victim.read_bytes()
    victim.write_bytes(blob[: len(blob) // 2])
    with pytest.raises(OSError) as e:
        model.transcribe_pcm(regions)
    assert str(victim) in str(e.value) and f"file {k}" in str(e.value)
    victim.write_bytes(blob)
    for what in ("after", "again"):
        got_outs, got, _ = model.transcribe_pcm(regions, split_notes=False)
        for g, w in zip(got_outs, want_outs):
            for k in w:
                assert np.array_equal(g[k].view(np.uint32), w[k].view(np.uint32)), (what, k)
        assert_same_notes(got, want, len(pcms), what)
    victim.unlink()
    with pytest.raises(OSError) as e:
        model.transcribe_pcm(regions)
    assert str(victim) in str(e.value)
