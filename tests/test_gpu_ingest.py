"""The device audio ingest (csrc/ingest.cu: `bp_load_pcm_host` / `bp_load_pcm_device`, `audio_io.load_audio_device`)
against the host loader `audio_io.load_audio` and a float64 resampler.

At 22 050 Hz nothing is resampled and the device output is the host loader's float32 down-mix bit for bit (the kernel
sums the channels in NumPy's pairwise order).  Elsewhere each output is checked against scipy.signal.resample_poly of
the same float32 down-mix in float64, within the per-element bound of `reference`; the CPU tests at the end check the
down-mix order the kernel implements and which plausible faults that bound can see."""
import struct
from math import gcd

import numpy as np
import pytest

U = 2.0**-24
RATES = (4000, 8000, 11025, 16000, 22050, 24000, 32000, 44100, 44101, 48000, 88200, 96000, 192000, 352800, 705600,
         1411200)  # fmt: skip
RESAMPLED = tuple(sr for sr in RATES if sr != 22050)
FORMATS = (np.float32, np.int16, np.int32, np.uint8)  # sample_format 0..3
SIGNALS = ("extremes", "noise", "pass", "stop")
GOLD_TOL = 5e-4  # vs the reference's golden file (44.1 kHz source, resampler differs; see tests/golden/README.md)


def ratio(sr):
    g = gcd(22050, sr)
    return 22050 // g, sr // g


def design(sr):
    """-> (up, down, h, taps per phase T, half) of the resampler from sr to 22 050 Hz."""
    from basic_pitch_b200 import audio_io

    up, down = ratio(sr)
    h = audio_io._resample_filter(up, down)
    return up, down, h, -(-len(h) // up), (len(h) - 1) // 2


def gamma(k, u):
    return k * u / (1.0 - k * u)


def reference(x32, sr):
    """-> (float64 resample_poly of the float32 signal x32, per-element bound of the kernel's error, magnitude A).

    The kernel sums T = ceil(len(h) / up) products per output in float32 with four FMA accumulators; a0 also takes the
    T % 4 remainder taps and the two final adds come after, so the longest chain has n = T // 4 + T % 4 + 2 roundings.
    With A = resample_poly(|x|, window=|h|) = sum of up |h| |x| per output:
      |got - ref| <= (gamma_n (1 + u) + u) A + gamma64_T A + n 2^-149 + 2 up T d max|x|,
    u A for the polyphase table rounded to float32 (the accumulation then acts on taps up to (1 + u) up |h|),
    gamma64_T A for the float64 reference itself, n 2^-149 for products in the float32 denormal range, and the last
    term for the library's own design of the taps, within d = 1e-12 max|h| of audio_io's
    (test_ingest_filter_and_length_match_scipy), T of them per output (the 2 covers their rounding and accumulation)."""
    import scipy.signal

    up, down, h, T, _half = design(sr)
    x = np.asarray(x32, np.float64)
    ref = scipy.signal.resample_poly(x, up, down, window=h)
    a = scipy.signal.resample_poly(np.abs(x), up, down, window=np.abs(h))
    n = T // 4 + T % 4 + 2
    taps = 2.0 * up * T * 1e-12 * np.abs(h).max() * (np.abs(x).max() if len(x) else 0.0)
    return ref, (gamma(n, U) * (1 + U) + U) * a + gamma(T, 2.0**-53) * a + n * 2.0**-149 + taps, a


def host_mono(pcm):
    """load_audio's conversion and down-mix of the stored samples ((n,) or (n, channels))."""
    from basic_pitch_b200 import audio_io

    x = audio_io._to_float32(pcm)
    return x.mean(axis=1, dtype=np.float32) if x.ndim == 2 else x


def make_pcm(dt, n, ch, signal, sr, rng):
    """(n,) for one channel, else (n, ch) samples of format dt.  extremes: runs of each format's limits (float: +-1,
    +-4.0 overshoots, denormals ~1e-40, frames of -0.0 in every channel); noise: uniform over the format's range;
    pass: a sine at 0.9 x the resampler's pass edge; stop: one in its stop band (or near the input's Nyquist rate when
    the input is the lower rate)."""
    dt = np.dtype(dt)
    k = np.arange(n)[:, None] + np.zeros((1, ch), np.int64)
    c = np.arange(ch)[None, :]
    seg = k // 37
    if dt.kind in "iu":
        lo, hi = (0, 255) if dt == np.uint8 else (int(np.iinfo(dt).min), int(np.iinfo(dt).max))
    if signal == "extremes":
        if dt.kind in "iu":
            hi_mask = [seg % 4 == 0, seg % 4 == 2, (seg % 4 == 1) & (c % 2 == 0), (seg % 4 == 3) & (k % 2 == 1)]
            pcm = np.where(hi_mask[0] | hi_mask[2] | hi_mask[3], hi, lo)
            pcm = np.where(seg % 8 == 6, (lo + hi + 1) // 2, pcm)  # a run of the format's zero
        else:
            s = seg % 6
            sign = np.where((c + k) % 2 == 0, 1.0, -1.0)
            pcm = np.select(
                [s == 0, s == 1, s == 2, s == 3, s == 4],
                [np.where(c % 2 == 0, 1.0, -1.0), np.where(c % 2 == 0, -1.0, 1.0), 4.0 * sign,
                 sign * rng.uniform(0.5, 1.5, k.shape) * 1e-40, np.full(k.shape, -0.0)],
                0.0,
            )  # fmt: skip
        pcm = pcm.astype(dt)
    elif signal == "noise":
        pcm = rng.uniform(-1.0, 1.0, k.shape).astype(dt) if dt.kind == "f" else rng.integers(lo, hi, k.shape, endpoint=True).astype(dt)
    else:
        nyq_low = min(sr, 22050) / 2
        f = 0.9 * 0.913 * nyq_low if signal == "pass" else min(1.1 * nyq_low, 0.95 * sr / 2)
        v = 0.9 * np.sin(2 * np.pi * f * k / sr + 0.7 * c)
        if dt == np.uint8:
            pcm = np.round(v * 127 + 128).astype(dt)
        elif dt.kind == "i":
            pcm = np.round(v * hi).astype(dt)
        else:
            pcm = v.astype(dt)
    return np.ascontiguousarray(pcm[:, 0] if ch == 1 else pcm)


def fmt_code(pcm):
    return FORMATS.index(pcm.dtype.type)


def ingest(model, pcm, sr):
    """bp_load_pcm_host; unwritten outputs stay NaN."""
    n, ch = (pcm.shape[0], 1) if pcm.ndim == 1 else pcm.shape
    lib = model._lib
    out = np.full(int(lib.bp_resampled_length(n, sr)), np.nan, np.float32)
    lib.bp_load_pcm_host(model.handle, pcm.ctypes.data, fmt_code(pcm), n, ch, sr, out.ctypes.data)
    return out


def assert_bits(got, want, what):
    assert got.dtype == want.dtype == np.float32 and got.shape == want.shape, (what, got.shape, want.shape)
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert bad.size == 0, (what, f"{bad.size} of {want.size} differ", int(bad[0]), float(got[bad[0]]), float(want[bad[0]]))


def assert_within(got, x32, sr, what):
    """Element-wise against `reference`.  -> max err/bound."""
    ref, bound, _a = reference(x32, sr)
    assert got.dtype == np.float32 and got.shape == ref.shape, (what, got.shape, ref.shape)
    err = np.abs(got.astype(np.float64) - ref)
    bad = np.flatnonzero(~(err <= bound))  # NaN (an output never written) fails too
    assert bad.size == 0, (what, int(bad[0]), float(got[bad[0]]), float(ref[bad[0]]), float(bound[bad[0]]))
    return float((err / bound).max()) if len(err) else 0.0


def short_lengths(sr):
    """Frame counts whose output lengths are the first of >= 1, 255, 256, 257 and 1025 (CTA boundaries: 256 outputs per
    CTA), and one below T / 2 for which every output's taps reach past both ends of the signal."""
    up, down, _h, T, half = design(sr)
    ns = [(t - 1) * down // up + 1 for t in (1, 255, 256, 257, 1025)]
    n = max(1, T // 3)
    n_out = -(-n * up // down)
    assert (0 * down + half) // up >= n and ((n_out - 1) * down + half) // up - (T - 1) < 0, sr
    return ns + [n]


@pytest.fixture(scope="module")
def model():
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    return Model(ICASSP_2022_MODEL_PATH, device=0)


@pytest.mark.gpu
@pytest.mark.parametrize("channels", [1, 2, 3, 7, 8, 9, 16, 130])
def test_native_rate_is_the_host_downmix_bit_for_bit(model, channels):
    """At 22 050 Hz: conversion and down-mix only, bit-identical to load_audio's (NumPy's pairwise float32 mean from
    +0, so a frame of -0.0 in every channel gives +0.0), for every format and signal and at CTA boundaries."""
    rng = np.random.default_rng(channels)
    lengths = (1, 255, 256, 257, 4099)
    for fi, dt in enumerate(FORMATS):
        for si, signal in enumerate(SIGNALS):
            # extremes: 1025 frames hold every run of make_pcm's cycle (222 frames); the other signals take the lengths
            n = 1025 if signal == "extremes" else lengths[(3 * fi + si) % len(lengths)]
            pcm = make_pcm(dt, n, channels, signal, 22050, rng)
            want = host_mono(pcm)
            if signal == "extremes" and dt == np.float32:  # the frames of -0.0 and of denormals are there
                frames = pcm.reshape(n, channels)
                neg0 = np.all((frames == 0) & np.signbit(frames), axis=1)
                assert neg0.sum() >= 37 and np.any((frames != 0) & (np.abs(frames) < 1.1754944e-38))
                assert np.all(np.signbit(want[neg0]) == (channels == 1))  # a mean from +0: -0.0 only when not averaged
            assert_bits(ingest(model, pcm, 22050), want, (np.dtype(dt).name, signal, pcm.shape))


@pytest.mark.gpu
def test_downmix_of_a_huge_channel_count(model):
    """2^24 + 3 channels (any int count is accepted): the pairwise split 17 levels deep and a count that float32 cannot
    hold, which NumPy divides by in float64; bit-identical to load_audio's down-mix."""
    rng = np.random.default_rng(4)
    pcm = rng.integers(-32768, 32767, (2, (1 << 24) + 3), endpoint=True).astype(np.int16)
    assert_bits(ingest(model, pcm, 22050), host_mono(pcm), pcm.shape)


@pytest.mark.gpu
@pytest.mark.parametrize("sr", RESAMPLED)
def test_resampled_rate_within_the_bound(model, sr):
    """Every format, channels 1 / 2 / 8, every signal, output lengths at CTA boundaries, an input shorter than the
    filter, and a 30 s input; 705 600 and 1 411 200 Hz stage more than 48 KB per CTA (opt-in shared memory)."""
    r = RESAMPLED.index(sr)
    rng = np.random.default_rng(sr)
    worst = 0.0
    for i, n in enumerate(short_lengths(sr)):
        pcm = make_pcm(FORMATS[(i + r) % 4], n, (1, 2, 8)[i % 3], SIGNALS[(3 * i + r) % 4], sr, rng)
        worst = max(worst, assert_within(ingest(model, pcm, sr), host_mono(pcm), sr, (sr, pcm.dtype.name, pcm.shape)))
    pcm = make_pcm(FORMATS[r % 4], 30 * sr, 1, "noise", sr, rng)
    worst = max(worst, assert_within(ingest(model, pcm, sr), host_mono(pcm), sr, (sr, pcm.dtype.name, pcm.shape)))
    print(f"{sr} Hz (up {ratio(sr)[0]}, down {ratio(sr)[1]}, T {design(sr)[3]}): max err/bound {worst:.3f}")


@pytest.mark.gpu
def test_device_ingest_vocadito_44k_vs_golden(model, golden_dir):
    """The reference's 44.1 kHz test clip through the device ingest and the model against the reference's golden
    posteriorgrams (reference: tests/test_inference.py:43-70; tolerance = the resampler residual, tests/golden/README.md)."""
    z = np.load(golden_dir / "vocadito10_pcm44k.npz")
    pcm, sr = z["pcm"], int(z["sample_rate"])
    lib = model._lib
    audio = np.empty(int(lib.bp_resampled_length(len(pcm), sr)), np.float32)
    lib.bp_load_pcm_host(model.handle, pcm.ctypes.data, 1, len(pcm), 1, sr, audio.ctypes.data)
    gold = np.load(golden_dir / "vocadito10.npz")
    assert np.abs(audio - gold["audio22k"]).max() < 3e-6  # the host resampler of the fixture
    out = model.run_inference_arrays([audio])[0]
    for k in ("note", "onset", "contour"):
        assert out[k].shape == gold[f"gold_{k}"].shape
        assert float(np.abs(out[k] - gold[f"gold_{k}"]).max()) < GOLD_TOL, k


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [44100, 48000, 8000, 44101])
def test_outputs_do_not_depend_on_their_cta(model, sr):
    """down * c leading zero frames move every output by up * c (not a multiple of the 256 outputs of a CTA): output
    k + up * c is output k bit for bit, since each output sums its taps in a fixed order."""
    up, down = ratio(sr)
    c = 3
    assert up * c % 256 != 0
    rng = np.random.default_rng(7)
    pcm = make_pcm(np.int16, 3 * 1025 * down // up + 11, 2, "noise", sr, rng)
    out = ingest(model, pcm, sr)
    moved = ingest(model, np.concatenate([np.zeros((down * c, 2), np.int16), pcm]), sr)
    assert len(moved) == len(out) + up * c and len(out) > 3 * 256
    assert_bits(moved[up * c :], out, sr)


@pytest.mark.gpu
def test_device_entry_point(model):
    """bp_load_pcm_device on torch tensors on a non-default stream, from an int16 pointer at an odd element offset: the
    bits of bp_load_pcm_host, twice, and its output, fed on the same stream to bp_transcribe_device, gives the notes of
    the same samples through bp_transcribe_host."""
    import torch

    from basic_pitch_b200 import engine, synth

    sr = 44100
    clip = np.repeat(synth.tones_clip(4.0, seed=5), 2).astype(np.float64)
    rng = np.random.default_rng(3)
    pcm = np.round(np.stack([clip, 0.5 * clip + 0.01 * rng.standard_normal(len(clip))], 1) * 20000).astype(np.int16)
    host = ingest(model, pcm, sr)
    n, n_out = pcm.shape[0], len(host)
    dev = torch.device(f"cuda:{model.device}")
    src = torch.zeros(pcm.size + 1, dtype=torch.int16, device=dev)
    src[1:].copy_(torch.from_numpy(pcm.reshape(-1)))
    view = src[1:]
    assert view.data_ptr() % 4 == 2
    outs = [torch.full((n_out,), float("nan"), dtype=torch.float32, device=dev) for _ in range(2)]
    stream = torch.cuda.Stream(dev)
    stream.wait_stream(torch.cuda.current_stream(dev))
    offsets = np.array([0, n_out], np.int64)
    out_d = engine.NoteBuffers(1, 4096, 65536)
    with torch.cuda.stream(stream):
        for out in outs:
            model._lib.bp_load_pcm_device(model.handle, view.data_ptr(), 1, n, 2, sr, out.data_ptr(), stream.cuda_stream)
        n_dev = engine.transcribe_packed_device(model, outs[0], offsets, out_d, stream=stream.cuda_stream)
    stream.synchronize()
    for out in outs:
        assert_bits(out.cpu().numpy(), host, "bp_load_pcm_device")
    out_h = engine.NoteBuffers(1, 4096, 65536)
    assert engine.transcribe_packed_host(model, engine.PackedAudio([host]), out_h) == n_dev > 3
    got, want = engine.split_results(out_d)[0], engine.split_results(out_h)[0]
    for key in want:
        np.testing.assert_array_equal(got[key], want[key], err_msg=key)


@pytest.mark.gpu
def test_filter_cache_across_models(model):
    """The designed filters are cached per device and shared by its models: rates A and B interleaved over two models
    give, on every call, the bits of the first call at that rate."""
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH
    from basic_pitch_b200.inference import Model

    other = Model(ICASSP_2022_MODEL_PATH, device=0)
    rng = np.random.default_rng(9)
    pcm = {sr: make_pcm(np.int16, 20000, 2, "noise", sr, rng) for sr in (37800, 50000)}  # rates no other test uses
    first = {}
    for m, sr in ((model, 37800), (other, 50000), (other, 37800), (model, 50000), (model, 37800), (other, 50000)):
        got = ingest(m, pcm[sr], sr)
        if sr not in first:
            first[sr] = got
            assert_within(got, host_mono(pcm[sr]), sr, sr)
        assert_bits(got, first[sr], sr)


@pytest.mark.gpu
def test_invalid_arguments(model):
    """Unsupported format, channel count or sample rate (2 822 400 Hz stages 221 KB per CTA, over the 200 KB limit)
    return BP_E_INVALID from both entry points; n_frames = 0 succeeds and writes nothing; after each, a valid call
    still gives the same bits."""
    import torch

    from basic_pitch_b200 import _lib

    lib = model._lib
    rng = np.random.default_rng(1)
    pcm = make_pcm(np.int16, 4000, 2, "noise", 48000, rng)
    want = ingest(model, pcm, 48000)
    dev = torch.device(f"cuda:{model.device}")
    d_pcm = torch.from_numpy(pcm.reshape(-1)).to(dev)
    d_out = torch.full((1 << 16,), 7.0, dtype=torch.float32, device=dev)
    h_out = np.full(1 << 16, 7.0, np.float32)
    stream = torch.cuda.current_stream(dev).cuda_stream
    for fmt, n, ch, sr in ((-1, 4000, 2, 48000), (4, 4000, 2, 48000), (1, 4000, 0, 48000), (1, 4000, 2, 0),
                           (1, 4000, 2, -1), (1, 2000, 2, 2822400)):  # fmt: skip
        for name, call in (("host", lambda: lib.bp_load_pcm_host(model.handle, pcm.ctypes.data, fmt, n, ch, sr, h_out.ctypes.data)),
                           ("device", lambda: lib.bp_load_pcm_device(model.handle, d_pcm.data_ptr(), fmt, n, ch, sr, d_out.data_ptr(), stream))):  # fmt: skip
            with pytest.raises(_lib.BpError) as e:
                call()
            assert e.value.code == _lib.BP_E_INVALID, (name, fmt, n, ch, sr)
            assert_bits(ingest(model, pcm, 48000), want, (name, fmt, n, ch, sr))
    lib.bp_load_pcm_host(model.handle, pcm.ctypes.data, 1, 0, 2, 48000, h_out.ctypes.data)
    lib.bp_load_pcm_device(model.handle, d_pcm.data_ptr(), 1, 0, 2, 48000, d_out.data_ptr(), stream)
    torch.cuda.synchronize(dev)
    assert np.all(h_out == 7.0) and bool((d_out == 7.0).all())
    assert_bits(ingest(model, pcm, 48000), want, "after n_frames = 0")


def write_wav24(path, sr, pcm):
    """A 24-bit PCM WAV of int32 samples (n, channels) in [-2^23, 2^23) (scipy.io.wavfile cannot write one)."""
    data = pcm.astype("<i4").reshape(-1).view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    ch = pcm.shape[1]
    fmt = struct.pack("<HHIIHH", 1, ch, sr, sr * ch * 3, ch * 3, 24)
    body = b"WAVE" + b"fmt " + struct.pack("<I", len(fmt)) + fmt + b"data" + struct.pack("<I", len(data)) + data
    path.write_bytes(b"RIFF" + struct.pack("<I", len(body)) + body + b"\0" * (len(data) % 2))


@pytest.mark.gpu
@pytest.mark.parametrize("sr", [22050, 48000, 44101])
def test_wav_files_through_load_audio_device(model, tmp_path, sr):
    """load_audio_device against load_audio on a 24-bit WAV (read as left-justified int32), a float64 WAV (converted to
    float32 before the ingest) and an 8-bit WAV: bits at 22 050 Hz, the bound elsewhere (plus u A: load_audio rounds
    its float64 result to float32)."""
    from scipy.io import wavfile

    from basic_pitch_b200 import audio_io

    rng = np.random.default_rng(sr)
    n = 3 * sr // 2 + 1
    s24 = np.clip(np.round(make_pcm(np.float64, n, 2, "pass", sr, rng) * 2**23), -(2**23), 2**23 - 1).astype(np.int32)
    s24[: n // 3] = rng.integers(-(2**23), 2**23, (n // 3, 2))
    files = {"s24": tmp_path / "s24.wav", "f64": tmp_path / "f64.wav", "u8": tmp_path / "u8.wav"}
    write_wav24(files["s24"], sr, s24)
    wavfile.write(files["f64"], sr, make_pcm(np.float64, n, 3, "noise", sr, rng) * 1.5)
    wavfile.write(files["u8"], sr, make_pcm(np.uint8, n, 1, "extremes", sr, rng))
    stored, _ = audio_io.read_pcm(files["s24"])
    assert stored.dtype == np.int32 and np.array_equal(stored, s24 << 8)
    for name, path in files.items():
        got, sr_out = audio_io.load_audio_device(path, model)
        want, _ = audio_io.load_audio(path)
        assert sr_out == 22050
        if sr == 22050:
            assert_bits(got, want, name)
        else:
            x, _ = audio_io.read_audio(path)
            assert_within(got, host_mono(x), sr, name)
            _ref, bound, a = reference(host_mono(x), sr)
            assert np.all(np.abs(got.astype(np.float64) - want) <= bound + U * a), name


def numpy_pairwise_sum(x):
    """NumPy's pairwise float32 sum of each row of x (rows, n) (numpy/_core/src/umath/loops_utils.h.src): below 8 a
    sequential sum from 0, up to 128 eight interleaved accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7))
    then the tail, above 128 the sums of the halves split at n2 = n/2 - (n/2) % 8."""
    n = x.shape[1]
    f = np.float32
    if n < 8:
        s = np.zeros(x.shape[0], f)
        for i in range(n):
            s = s + x[:, i]
        return s
    if n <= 128:
        r = x[:, :8].copy()
        i = 8
        while i + 8 <= n:
            r = r + x[:, i : i + 8]
            i += 8
        s = ((r[:, 0] + r[:, 1]) + (r[:, 2] + r[:, 3])) + ((r[:, 4] + r[:, 5]) + (r[:, 6] + r[:, 7]))
        for j in range(i, n):
            s = s + x[:, j]
        return s
    n2 = n // 2 - (n // 2) % 8
    return numpy_pairwise_sum(x[:, :n2]) + numpy_pairwise_sum(x[:, n2:])


def test_downmix_order_is_numpys():
    """CPU: the order csrc/ingest.cu's mono_sample implements, +0 + pairwise_sum then / channels in float64 rounded to
    float32, is x.mean(axis=1, dtype=float32) bit for bit for 1..300 channels, frames of -0.0 included (-> +0.0), and
    for counts whose split goes deep or that float32 cannot hold; a sequential sum is not, from 8 channels on."""
    rng = np.random.default_rng(0)

    def emulated(x):
        return ((np.float32(0) + numpy_pairwise_sum(x)).astype(np.float64) / x.shape[1]).astype(np.float32)

    for ch in range(1, 301):
        x = (rng.standard_normal((64, ch)) * 10.0 ** rng.uniform(-3, 3, (64, ch))).astype(np.float32)
        x[0] = -0.0
        x[1, ::2] = -0.0
        x[2] = 1e-40
        want = x.mean(axis=1, dtype=np.float32)
        assert np.array_equal(emulated(x).view(np.uint32), want.view(np.uint32)), ch
        assert want[0] == 0 and not np.signbit(want[0])
        if ch >= 8:
            seq = x[:, 0].copy()
            for i in range(1, ch):
                seq = seq + x[:, i]
            assert not np.array_equal(seq / np.float32(ch), want), ch
    for ch in (65535, 100003, (1 << 24) + 3):
        x = (rng.standard_normal((2, ch)) * 10.0 ** rng.uniform(-3, 3, (2, ch))).astype(np.float32)
        want = x.mean(axis=1, dtype=np.float32)
        assert np.array_equal(emulated(x).view(np.uint32), want.view(np.uint32)), ch


def polyphase(x, g, up, down, off, n_out):
    """float64 y[k] = sum_i x[i] g[k * down + off - i * up] for k < n_out (g zero outside): the kernel's sum with the
    filter g = up * h and off = half; faults are other g or off."""
    import scipy.signal

    pre = (-off) % down
    q0 = (off + pre) // down
    z = scipy.signal.upfirdn(np.concatenate([np.zeros(pre), g]), x, up, down)[q0 : q0 + n_out]
    return np.concatenate([z, np.zeros(n_out - len(z))])


def faults(pcm, sr):
    """-> {fault: float64 output} of plausible kernel faults on int16 PCM (n, channels)."""
    up, down, h, T, half = design(sr)
    x = host_mono(pcm).astype(np.float64)
    n_out = -(-len(x) * up // down)
    g = up * h
    p = (np.arange(n_out) * down + half) % up
    out = {
        # phase (p + 1) % up with the same newest input (no fault for up = 1: one phase)
        "phase + 1": np.where(p == up - 1, polyphase(x, g, up, down, half - (up - 1), n_out),
                              polyphase(x, g, up, down, half + 1, n_out)),
        "half + 1": polyphase(x, g, up, down, half + 1, n_out),
        "output shifted": polyphase(x, g, up, down, half + down, n_out),
        "newest tap dropped": polyphase(x, np.where(np.arange(len(g)) < up, 0.0, g), up, down, half, n_out),
        "int16 / 32767": polyphase(pcm.astype(np.float64).mean(axis=1) / 32767.0, g, up, down, half, n_out),
        "channel dropped": polyphase(pcm[:, :-1].astype(np.float64).sum(axis=1) / 32768.0 / pcm.shape[1], g, up, down,
                                     half, n_out),
        "last frame dropped": polyphase(np.where(np.arange(len(x)) < len(x) - 1, x, 0.0), g, up, down, half, n_out),
        "oldest tap dropped": polyphase(x, np.where(np.arange(len(g)) >= (T - 1) * up, 0.0, g), up, down, half, n_out),
    }  # fmt: skip
    return x, out


@pytest.mark.parametrize("sr", RESAMPLED)
def test_the_bound_sees_plausible_faults(sr):
    """CPU: which faults of the kernel the GPU tests' bound can see, on 2-channel int16 noise with 1025 outputs.  At
    44 100 and 48 000 Hz every fault must exceed the bound somewhere (the phase fault is no fault where up = 1: there
    is one phase); at the other rates the bound loosens with the tap count (gamma_n ~ 9e-5 at 705 600 Hz, where a
    3e-5 scale error passes) and the result is reported.  So is a dropped newest or oldest tap: both are taps at the
    edges of the Kaiser window (h[p] and h[p + (T - 1) up]), at most 1.6e-7 of the centre tap, and stay below the bound at every
    rate; a dropped last input frame is the newest-end fault the bound does see."""
    up, down, _h, _T, half = design(sr)
    rng = np.random.default_rng(5)
    pcm = rng.integers(-32768, 32767, (1024 * down // up + 1, 2), endpoint=True).astype(np.int16)
    x, out = faults(pcm, sr)
    ref, bound, a = reference(x.astype(np.float32), sr)
    exact = polyphase(x, up * design(sr)[2], up, down, half, len(ref))
    assert np.all(np.abs(exact - ref) <= 1e-12 * a)  # the emulation is the kernel's sum
    seen = {k: float((np.abs(v - ref) / bound).max()) for k, v in out.items()}
    print(f"{sr} Hz: max err/bound " + ", ".join(f"{k} {v:.3g}" for k, v in seen.items()))
    if sr in (44100, 48000):
        for k, v in seen.items():
            if k in ("newest tap dropped", "oldest tap dropped") or (k == "phase + 1" and up == 1):
                continue
            assert v > 1.0, (sr, k, v)
