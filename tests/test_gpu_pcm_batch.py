"""The batched device ingest (csrc/ingest.cu: `ingest_batch_kernel` behind `bp_load_pcm_files_device`) and the whole
path that starts from stored PCM (`bp_transcribe_pcm_files_host`, `Model.transcribe_pcm`, `predict_batch` on paths).

What pins the arithmetic is one contract: file i of a batched ingest has exactly the bits `bp_load_pcm_host` gives for
file i alone, wherever it sits in the batch and whatever its neighbours are.  That single-file ingest is itself checked
against a float64 resampler in tests/test_gpu_ingest.py, whose generators are used here.  The whole path is then compared
with the two-step path it replaces: the ingest per file, then `bp_transcribe_files_host`."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_ingest import FORMATS, RATES, assert_bits, fmt_code, ingest, make_pcm, ratio, write_wav24

BYTES = (4, 2, 4, 1)  # per sample of format 0..3


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH, device=0)


def shape_of(pcm):
    return (pcm.shape[0], 1) if pcm.ndim == 1 else pcm.shape


def descriptors(pcms, rates, pointers=None):
    """A bp_pcm_file_t array over the arrays `pcms` (or over `pointers`, e.g. device addresses)."""
    from basic_pitch_b200 import _lib

    files = (_lib.PcmFile * max(len(pcms), 1))()
    for i, (f, x, sr) in enumerate(zip(files, pcms, rates)):
        f.pcm = pointers[i] if pointers is not None else (x.ctypes.data if x.size else None)
        (f.n_frames, f.channels), f.sample_format, f.sample_rate = shape_of(x), fmt_code(x), sr
    return files


def frames_for_outputs(sr, n_out):
    """The smallest frame count at rate sr (not above 22 050 Hz's output density) that resamples to n_out samples."""
    up, down = ratio(sr)
    assert down >= up
    n = (n_out - 1) * down // up + 1
    assert -(-n * up // down) == n_out, (sr, n_out)
    return n


def ingest_batch():
    """Files mixing every format, 1 / 2 / 6 / 130 channels, rates on both sides of 22 050 Hz, both signals, output
    lengths ending 0, 1, 255, 256 and 257 samples into a CTA, one frame, and nothing at all."""
    rng = np.random.default_rng(11)
    empty = lambda dt, ch: np.zeros((0, ch), dt) if ch > 1 else np.zeros(0, dt)  # noqa: E731
    spec = [("empty", np.int16, 2, 48000, None, 0)]
    ends = (512, 513, 255, 256, 257)
    rates = (44100, 44101, 1411200, 22050, 48000)  # 1 411 200 Hz: ratio 64, more than 48 KB staged per CTA
    for i, (n_out, sr) in enumerate(zip(ends, rates)):
        spec.append((f"end{n_out}", FORMATS[i % 4], (1, 2, 6, 130, 2)[i], sr, ("extremes", "noise")[i % 2],
                     frames_for_outputs(sr, n_out)))
    spec.append(("empty", np.float32, 1, 22050, None, 0))
    for i, sr in enumerate((4000, 8000, 11025, 16000, 24000, 32000, 96000, 192000)):
        assert sr in RATES
        spec.append((f"sr{sr}", FORMATS[(i + 1) % 4], (2, 1, 130, 6)[i % 4], sr, ("noise", "extremes")[i % 2],
                     1000 + 411 * i))
    spec.append(("one frame", np.uint8, 2, 44100, "noise", 1))
    spec.append(("long", np.int16, 2, 44100, "noise", 5 * 44100 + 3))
    spec.append(("empty", np.uint8, 6, 8000, None, 0))
    pcms = [empty(dt, ch) if n == 0 else make_pcm(dt, n, ch, signal, sr, rng) for _w, dt, ch, sr, signal, n in spec]
    return [s[0] for s in spec], pcms, [s[3] for s in spec]


@pytest.mark.gpu
def test_batched_ingest_is_the_single_file_ingest_bit_for_bit(model):
    """One bp_load_pcm_files_device call over `ingest_batch`, in both file orders: every slice is bp_load_pcm_host of
    that file alone, the offsets are bp_resampled_length, and the canaries before and behind the packed signals are
    intact."""
    import torch

    lib = model._lib
    names, pcms, rates = ingest_batch()
    assert {p.dtype.type for p in pcms} == set(FORMATS) and {shape_of(p)[1] for p in pcms} == {1, 2, 6, 130}
    assert min(rates) < 22050 < max(rates) and 44101 in rates
    alone = [ingest(model, p, sr) for p, sr in zip(pcms, rates)]
    assert {len(a) % 256 for a in alone} >= {0, 1, 255} and {256, 257, 1, 0} <= {len(a) for a in alone}
    dev = torch.device(f"cuda:{model.device}")
    d_pcm = [torch.from_numpy(p.reshape(-1).copy()).to(dev) for p in pcms]
    stream = torch.cuda.Stream(dev)
    stream.wait_stream(torch.cuda.current_stream(dev))
    pad = 300
    canary = np.float32(-123456.75)
    for order in (list(range(len(pcms))), list(reversed(range(len(pcms))))):
        files = descriptors([pcms[i] for i in order], [rates[i] for i in order], [d_pcm[i].data_ptr() for i in order])
        want_off = np.concatenate([[0], np.cumsum([len(alone[i]) for i in order])]).astype(np.int64)
        for i, o in zip(order, np.diff(want_off)):
            assert o == lib.bp_resampled_length(shape_of(pcms[i])[0], rates[i])
        total = int(want_off[-1])
        d_out = torch.full((pad + total + pad,), float(canary), dtype=torch.float32, device=dev)
        off = np.full(len(order) + 1, -1, np.int64)
        before = model.launch_count
        with torch.cuda.stream(stream):
            lib.bp_load_pcm_files_device(model.handle, files, len(order), d_out.data_ptr() + 4 * pad, off.ctypes.data,
                                         stream.cuda_stream)
        stream.synchronize()
        assert model.launch_count == before + 1  # one launch for the whole batch
        assert np.array_equal(off, want_off)
        got = d_out.cpu().numpy()
        assert np.all(got[:pad] == canary) and np.all(got[pad + total :] == canary)
        for j, i in enumerate(order):
            assert_bits(got[pad + off[j] : pad + off[j + 1]], alone[i], (names[i], j))


def interp_clip(clip, n):
    """`clip` stretched to n samples (float64)."""
    return np.interp(np.linspace(0, len(clip) - 1, n), np.arange(len(clip)), clip)


def as_format(x, dt, ch, rng):
    """Mono float64 x in [-1, 1] as (n,) / (n, ch) PCM of dtype dt, the channels slightly different from each other."""
    cols = np.stack([x * (1.0 - 0.1 * c) + 0.002 * rng.standard_normal(len(x)) for c in range(ch)], 1)
    if dt == np.uint8:
        pcm = np.round(cols * 100 + 128).astype(dt)
    elif np.dtype(dt).kind == "i":
        pcm = np.round(cols * 0.8 * np.iinfo(dt).max).astype(dt)
    else:
        pcm = cols.astype(dt)
    return np.ascontiguousarray(pcm[:, 0] if ch == 1 else pcm)


KINDS = ((np.float32, 1, 22050), (np.int16, 2, 44100), (np.int32, 1, 48000), (np.uint8, 2, 11025), (np.int16, 1, 16000),
         (np.float32, 2, 96000))  # fmt: skip


def clip_batch(n_files, seconds, seed, long_seconds=0.0):
    """-> (pcms, rates): n_files clips of `seconds` cycling through KINDS, with an empty and a one-frame file in the
    middle, and one int16 stereo 44.1 kHz file of long_seconds in front if asked for."""
    from basic_pitch_b200 import synth

    rng = np.random.default_rng(seed)
    base = [synth.random_notes_clip(10.0, seed=seed + i).astype(np.float64) for i in range(3)]
    pcms, rates = [], []
    if long_seconds:
        x = np.tile(interp_clip(base[0], 10 * 44100), int(np.ceil(long_seconds / 10)))[: int(long_seconds * 44100)]
        pcms.append(as_format(x, np.int16, 2, rng))
        rates.append(44100)
    for i in range(n_files):
        dt, ch, sr = KINDS[i % len(KINDS)]
        x = np.tile(interp_clip(base[i % 3], 10 * sr), int(np.ceil(seconds / 10)))[: int(seconds * sr) + 17 * i]
        pcms.append(as_format(x, dt, ch, rng))
        rates.append(sr)
        if i == n_files // 2:
            pcms += [np.zeros((0, 2), np.int16), np.full(1, 0.25, np.float32)]
            rates += [44100, 48000]
    return pcms, rates


NOTE_KEYS = ("note_off", "start", "end", "pitch", "amp", "bend_off", "bends")


def run_pcm(model, pcms, rates, posteriorgrams=True):
    """bp_transcribe_pcm_files_host -> (note, onset, contour | None, frame_off, sample_off, note arrays)."""
    from basic_pitch_b200 import _lib

    lib, n = model._lib, len(pcms)
    files = descriptors(pcms, rates)
    lens = [lib.bp_resampled_length(shape_of(p)[0], sr) for p, sr in zip(pcms, rates)]
    total = sum(lib.bp_num_frames(x) for x in lens)
    post = [np.full((total, w), np.nan, np.float32) if posteriorgrams else None for w in (88, 88, 264)]
    ptr = [None if a is None else a.ctypes.data for a in post]
    foff, soff = np.full(n + 1, -1, np.int64), np.full(n + 1, -1, np.int64)
    notes, arrs = model._alloc_notes(n, max(4096, 2 * total), max(65536, 24 * total))
    p = _lib.DecodeParams()
    lib.bp_default_decode_params(C.byref(p))
    lib.bp_transcribe_pcm_files_host(model.handle, files, n, C.byref(p), ptr[0], ptr[1], ptr[2], foff.ctypes.data,
                                     soff.ctypes.data, C.byref(notes))
    return post, foff, soff, arrs


def run_two_step(model, pcms, rates):
    """The path this replaces: the ingest file by file, then bp_transcribe_files_host on the 22 050 Hz signals."""
    from basic_pitch_b200 import _lib

    lib, n = model._lib, len(pcms)
    audios = [ingest(model, p, sr) for p, sr in zip(pcms, rates)]
    lens = np.array([len(a) for a in audios], np.int64)
    total = sum(lib.bp_num_frames(int(x)) for x in lens)
    post = [np.full((total, w), np.nan, np.float32) for w in (88, 88, 264)]
    foff = np.full(n + 1, -1, np.int64)
    notes, arrs = model._alloc_notes(n, max(4096, 2 * total), max(65536, 24 * total))
    p = _lib.DecodeParams()
    lib.bp_default_decode_params(C.byref(p))
    ptrs = (C.c_void_p * max(n, 1))(*[a.ctypes.data for a in audios])
    lib.bp_transcribe_files_host(model.handle, ptrs, lens.ctypes.data, n, C.byref(p), post[0].ctypes.data,
                                 post[1].ctypes.data, post[2].ctypes.data, foff.ctypes.data, C.byref(notes))
    return post, foff, np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), arrs


def assert_same_notes(got, want, n_files, what):
    n_notes = int(want["note_off"][n_files])
    assert n_notes > 0, what
    n_bends = int(want["bend_off"][n_notes])
    sizes = {"note_off": n_files + 1, "bend_off": n_notes + 1, "bends": n_bends}
    for k in NOTE_KEYS:
        m = sizes.get(k, n_notes)
        assert np.array_equal(got[k][:m].view(np.int32), want[k][:m].view(np.int32)), (what, k)


@pytest.mark.gpu
def test_whole_path_is_the_two_step_path(model):
    """Mixed formats over several sub-batches (more than four chunks of windows, one file longer than a chunk, an empty
    and a one-frame file): posteriorgrams, offsets and every note field are those of the ingest per file followed by
    bp_transcribe_files_host; also without posteriorgram outputs, and on a second call that reuses the buffers."""
    lib = model._lib
    chunk = int(lib.bp_model_chunk_windows(model.handle))
    pcms, rates = clip_batch(24, 40.0, seed=100, long_seconds=1.75 * chunk)
    want_post, want_foff, want_soff, want = run_two_step(model, pcms, rates)
    windows = [lib.bp_num_windows(int(x)) for x in np.diff(want_soff)]
    assert sum(windows) > 4 * chunk and windows[0] > chunk
    for call in range(2):
        post, foff, soff, arrs = run_pcm(model, pcms, rates)
        assert np.array_equal(foff, want_foff) and np.array_equal(soff, want_soff), call
        for got, exp, k in zip(post, want_post, ("note", "onset", "contour")):
            assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)), (call, k)
        assert_same_notes(arrs, want, len(pcms), call)
    _post, foff, soff, arrs = run_pcm(model, pcms, rates, posteriorgrams=False)
    assert np.array_equal(foff, want_foff) and np.array_equal(soff, want_soff)
    assert_same_notes(arrs, want, len(pcms), "no posteriorgram outputs")


@pytest.mark.gpu
def test_predict_batch_on_paths_and_arrays(model, tmp_path):
    """predict_batch over WAV files (int16 stereo 44.1 kHz, 24-bit, float64, 8-bit) mixed with arrays: the results of
    predict_batch over the load_audio_device signals of the same files, which never touches the PCM entry point."""
    from scipy.io import wavfile

    from basic_pitch_b200 import audio_io, synth
    from basic_pitch_b200.inference import predict_batch

    rng = np.random.default_rng(21)
    clips = [synth.random_notes_clip(6.0 + i, seed=300 + i).astype(np.float64) for i in range(5)]
    paths = {k: tmp_path / f"{k}.wav" for k in ("s16", "s24", "f64", "u8")}
    wavfile.write(paths["s16"], 44100, as_format(interp_clip(clips[0], 6 * 44100), np.int16, 2, rng))
    write_wav24(paths["s24"], 48000, as_format(interp_clip(clips[1], 7 * 48000), np.int32, 2, rng) >> 8)
    wavfile.write(paths["f64"], 44101, np.stack([interp_clip(clips[2], 8 * 44101)] * 3, 1) * 1.2)
    wavfile.write(paths["u8"], 22050, as_format(clips[3][: 9 * 22050], np.uint8, 1, rng))
    arrays = [clips[4].astype(np.float32), synth.tones_clip(3.0, seed=2)]
    mixed = [paths["s16"], arrays[0], paths["s24"], paths["f64"], arrays[1], paths["u8"]]
    two_step = [a if isinstance(a, np.ndarray) else audio_io.load_audio_device(a, model)[0] for a in mixed]

    calls = []
    real = model._lib.bp_transcribe_pcm_files_host
    model._lib.bp_transcribe_pcm_files_host = lambda *a: (calls.append(1), real(*a))[1]
    try:
        want = predict_batch(two_step, model)
        assert not calls  # arrays only: the float32 entry point, as before
        got = predict_batch(mixed, model)
        assert len(calls) == 1
    finally:
        model._lib.bp_transcribe_pcm_files_host = real
    assert len(got) == len(want) == len(mixed)
    for i, ((g_out, g_midi, g_ev), (w_out, w_midi, w_ev)) in enumerate(zip(got, want)):
        for k in ("note", "onset", "contour"):
            assert g_out[k].shape == w_out[k].shape and g_out[k].shape[0] > 0
            assert np.array_equal(g_out[k].view(np.uint32), w_out[k].view(np.uint32)), (i, k)
        assert len(w_ev) > 0 and list(g_ev) == list(w_ev), i
        assert len(g_midi.instruments[0].notes) == len(w_midi.instruments[0].notes)
    with pytest.raises(ValueError):
        predict_batch([paths["s16"], np.zeros((10, 2), np.float32)], model)


BAD_FIELDS = (("sample_format", -1), ("sample_format", 4), ("channels", 0), ("sample_rate", 0), ("sample_rate", -5),
              ("n_frames", -1), ("pcm", None), ("sample_rate", 2822400))  # fmt: skip


@pytest.mark.gpu
def test_invalid_file_in_the_middle(model):
    """Each invalid field in file 2 of 5: BP_E_INVALID naming the file from both entry points before anything is
    launched, and the model still gives the same results afterwards.  An empty batch succeeds."""
    import torch

    from basic_pitch_b200 import _lib

    lib = model._lib
    pcms, rates = clip_batch(5, 3.0, seed=400)
    pcms, rates = pcms[:5], rates[:5]
    _post, want_foff, want_soff, want = run_pcm(model, pcms, rates)
    dev = torch.device(f"cuda:{model.device}")
    d_pcm = [torch.from_numpy(p.reshape(-1).copy()).to(dev) for p in pcms]
    d_out = torch.zeros(int(want_soff[-1]) + 1, dtype=torch.float32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    off = np.zeros(6, np.int64)
    p = _lib.DecodeParams()
    lib.bp_default_decode_params(C.byref(p))
    notes, _arrs = model._alloc_notes(5, 4096, 65536)
    for on_device in (False, True):
        cases = BAD_FIELDS + ((("pcm", d_pcm[1].data_ptr() + 1),) if on_device else ())  # file 2 is int32: misaligned
        for field, value in cases:
            files = descriptors(pcms, rates, [t.data_ptr() for t in d_pcm] if on_device else None)
            setattr(files[2], field, value)
            before = model.launch_count
            with pytest.raises(_lib.BpError) as e:
                if on_device:
                    lib.bp_load_pcm_files_device(model.handle, files, 5, d_out.data_ptr(), off.ctypes.data, stream)
                else:
                    lib.bp_transcribe_pcm_files_host(model.handle, files, 5, C.byref(p), None, None, None,
                                                     off.ctypes.data, None, C.byref(notes))
            assert e.value.code == _lib.BP_E_INVALID and "file 2" in str(e.value), (on_device, field, str(e.value))
            assert model.launch_count == before, (on_device, field)
    _post, foff, soff, arrs = run_pcm(model, pcms, rates)
    assert np.array_equal(foff, want_foff) and np.array_equal(soff, want_soff)
    assert_same_notes(arrs, want, 5, "after the rejected calls")
    before = model.launch_count
    lib.bp_load_pcm_files_device(model.handle, None, 0, None, off.ctypes.data, stream)
    assert off[0] == 0 and model.launch_count == before
    _post, foff, soff, arrs = run_pcm(model, [], [])
    assert foff.tolist() == [0] and soff.tolist() == [0] and arrs["note_off"].tolist() == [0]


@pytest.mark.gpu
def test_two_models_side_by_side(model):
    """Two models on one device, batches of different sizes (one sub-batch, several), calls interleaved: each call gives
    what that batch gives on a model of its own."""
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    other = Model(ICASSP_2022_MODEL_PATH, device=0)
    chunk = int(model._lib.bp_model_chunk_windows(model.handle))
    small = clip_batch(4, 5.0, seed=500)
    large = clip_batch(12, 0.25 * chunk, seed=600)
    want = {"small": run_pcm(model, *small), "large": run_pcm(model, *large)}
    batches = {"small": small, "large": large}
    for m, name in ((model, "large"), (other, "small"), (other, "large"), (model, "small"), (other, "small"), (model, "large")):
        post, foff, soff, arrs = run_pcm(m, *batches[name])
        w_post, w_foff, w_soff, w_arrs = want[name]
        assert np.array_equal(foff, w_foff) and np.array_equal(soff, w_soff), name
        for got, exp in zip(post, w_post):
            assert np.array_equal(got.view(np.uint32), exp.view(np.uint32)), name
        assert_same_notes(arrs, w_arrs, len(batches[name][0]), name)


def test_descriptors_and_packing_layout():
    """CPU: `audio_io.pcm_descriptors` describes (n,) and (n, channels) arrays of every format as they are stored, and
    the library packs such files with every start on a 16-byte boundary and resampled lengths of
    ceil(n * 22050 / rate) — restated here in NumPy; invalid files are rejected by index without a device."""
    from basic_pitch_b200 import _lib, audio_io

    lib = _lib.load()
    rng = np.random.default_rng(0)
    shapes = [(7,), (5, 2), (0,), (33, 3), (1,), (0, 6), (1000, 1), (19, 130)]
    rates = [22050, 44100, 48000, 8000, 44101, 96000, 11025, 1411200]
    items = []
    for i, (shape, sr) in enumerate(zip(shapes, rates)):
        dt = FORMATS[i % 4]
        items.append(((rng.uniform(0, 100, shape)).astype(dt), sr))
    strided = rng.integers(-9, 9, (40, 4)).astype(np.int16)[::2, ::2]  # not contiguous: described through a copy
    items.append((strided, 32000))
    files, keep = audio_io.pcm_descriptors(items)
    n = len(items)
    assert len(keep) == n and np.array_equal(keep[-1], strided) and keep[-1].flags.c_contiguous
    byte_off, sample_off = np.full(n + 1, -1, np.int64), np.full(n + 1, -1, np.int64)
    lib.bp_debug_pcm_layout(files, n, byte_off.ctypes.data, sample_off.ctypes.data)
    pos = samples = 0
    for i, ((x, sr), f, k) in enumerate(zip(items, files, keep)):
        frames, ch = shape_of(x)
        assert (f.n_frames, f.channels, f.sample_rate, f.sample_format) == (frames, ch, sr, FORMATS.index(x.dtype.type)), i
        assert f.pcm == (k.ctypes.data if k.size else None), i
        assert byte_off[i] == pos and pos % 16 == 0 and sample_off[i] == samples, i
        nbytes = frames * ch * BYTES[f.sample_format]
        assert nbytes == k.nbytes
        pos += -(-nbytes // 16) * 16
        samples += -(-frames * 22050 // sr)
        assert lib.bp_resampled_length(frames, sr) == -(-frames * 22050 // sr)
    assert byte_off[n] == pos and sample_off[n] == samples
    for bad in (np.zeros(4, np.float64), np.zeros(4, np.int64), np.zeros((2, 2, 2), np.int16)):
        with pytest.raises(ValueError):
            audio_io.pcm_descriptors([(bad, 22050)])
    for field, value in BAD_FIELDS:
        files, keep = audio_io.pcm_descriptors(items)
        setattr(files[1], field, value)
        with pytest.raises(_lib.BpError) as e:
            lib.bp_debug_pcm_layout(files, n, byte_off.ctypes.data, sample_off.ctypes.data)
        assert e.value.code == _lib.BP_E_INVALID and "file 1" in str(e.value), (field, str(e.value))
    lib.bp_debug_pcm_layout(None, 0, byte_off.ctypes.data, sample_off.ctypes.data)
    assert byte_off[0] == 0 and sample_off[0] == 0
