"""CPU: the WAV header probe (`bp_probe_wav_files`, `audio_io.probe_wav`), the packing of the two formats only whole WAV
files bring (4 packed 24-bit, 5 float64) and the routing of a batch of paths and arrays (`inference._pcm_items`).

The probe's claim is agreement with scipy.io.wavfile.read on every file it accepts: the same dtype (24-bit: scipy's
int32 is the packed value << 8), channels, rate and frame count, and the same sample bytes at the reported offset.  A file
it declines goes to `read_pcm`, which gives it the result or the exception it always did."""
import ctypes as C
import os
import struct
import warnings

import numpy as np
import pytest

from tests.test_gpu_pcm_batch import shape_of

DTYPES = {0: np.dtype("<f4"), 1: np.dtype("<i2"), 2: np.dtype("<i4"), 3: np.dtype("u1"), 4: None, 5: np.dtype("<f8")}
BITS = {0: 32, 1: 16, 2: 32, 3: 8, 4: 24, 5: 64}
BYTES6 = (4, 2, 4, 1, 3, 8)  # per sample of format 0..5
GUID_TAIL = b"\x00\x00\x10\x00\x80\x00\x00\xaa\x00\x38\x9b\x71"


def chunk(cid, body, pad=True):
    return cid + struct.pack("<I", len(body)) + body + (b"\0" if pad and len(body) % 2 else b"")


def fmt_body(fmt, ch, sr, extensible=False, tag=None, bits=None, block=None, rate=None, cb=22):
    bits = BITS[fmt] if bits is None else bits
    tag = (3 if fmt in (0, 5) else 1) if tag is None else tag
    block = ch * bits // 8 if block is None else block
    rate = sr * block if rate is None else rate
    if not extensible:
        return struct.pack("<HHIIHH", tag, ch, sr, rate, block, bits)
    return struct.pack("<HHIIHH", 0xFFFE, ch, sr, rate, block, bits) + struct.pack("<HHI", cb, bits, 0) + \
        struct.pack("<I", tag) + GUID_TAIL


def sample_bytes(fmt, x):
    """Interleaved little-endian bytes of samples x (format 4: int32 values in [-2^23, 2^23))."""
    if fmt == 4:
        return x.astype("<i4").reshape(-1).view(np.uint8).reshape(-1, 4)[:, :3].tobytes()
    return np.ascontiguousarray(x, DTYPES[fmt]).tobytes()


def make_samples(fmt, n, ch, rng):
    shape = (n, ch) if ch > 1 else (n,)
    if fmt in (0, 5):
        return rng.uniform(-1.5, 1.5, shape).astype(DTYPES[fmt])
    if fmt == 4:
        return rng.integers(-(1 << 23), 1 << 23, shape).astype(np.int32)
    info = np.iinfo(DTYPES[fmt])
    return rng.integers(info.min, info.max, shape, endpoint=True).astype(DTYPES[fmt])


def wav_bytes(fmt, ch, sr, data, before=(), after=(), extensible=False, riff=b"RIFF", riff_size=None, **kw):
    body = b"WAVE" + b"".join(before) + chunk(b"fmt ", fmt_body(fmt, ch, sr, extensible, **kw)) + \
        chunk(b"data", data) + b"".join(after)
    return riff + struct.pack("<I", len(body) if riff_size is None else riff_size) + body


def assert_agrees_with_scipy(path, region):
    from scipy.io import wavfile

    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        sr, x = wavfile.read(path)
    n, ch = shape_of(x)
    assert (region.sample_rate, region.n_frames, region.channels) == (sr, n, ch), path
    fmt = region.sample_format
    if fmt == 4:
        assert x.dtype == np.int32 and np.all((x & 0xFF) == 0)
        want = sample_bytes(4, x >> 8)
    else:
        assert x.dtype.newbyteorder("<") == DTYPES[fmt], (path, x.dtype, fmt)
        want = np.ascontiguousarray(x, DTYPES[fmt]).tobytes()
    with open(path, "rb") as f:
        f.seek(region.data_offset)
        got = f.read(len(want))
    assert got == want, path


def test_accepted_files_agree_with_scipy(tmp_path):
    """Every format, 1 / 2 / 6 / 9 channels, five rates, 0 / 1 / 37 frames (odd data sizes with their pad byte), written
    by scipy where it can (uint8, int16, int32, float32, float64) and by hand for 24-bit."""
    from scipy.io import wavfile

    from basic_pitch_b200 import audio_io

    rng = np.random.default_rng(0)
    paths, expect = [], []
    for fmt in range(6):
        for ch in (1, 2, 6, 9):
            for sr in (8000, 22050, 44100, 48000, 96000):
                for n in (0, 1, 37):
                    x = make_samples(fmt, n, ch, rng)
                    p = tmp_path / f"f{fmt}_c{ch}_r{sr}_n{n}.wav"
                    if fmt == 4:
                        p.write_bytes(wav_bytes(4, ch, sr, sample_bytes(4, x)))
                    else:
                        wavfile.write(p, sr, x)
                    paths.append(p)
                    expect.append((fmt, ch, sr, n))
    regions, declined = audio_io.probe_wav(paths)
    assert declined == []
    for p, r, (fmt, ch, sr, n) in zip(paths, regions, expect):
        assert (r.sample_format, r.channels, r.sample_rate, r.n_frames) == (fmt, ch, sr, n), p
        assert r.path == str(p)
        assert_agrees_with_scipy(str(p), r)


def test_chunk_layouts_and_extensible(tmp_path):
    """LIST / fact / unknown chunks before and after `data`, odd-sized chunks with their pad byte, EXTENSIBLE with the
    PCM and the IEEE-float sub-formats, a RIFF size that ends at the data chunk's odd end without its pad byte."""
    from basic_pitch_b200 import audio_io

    rng = np.random.default_rng(1)
    odd = chunk(b"LIST", b"INFOabc")  # 7 bytes + pad
    fact = chunk(b"fact", struct.pack("<I", 5))
    junk = chunk(b"abcd", b"x" * 13)
    cases = []
    for fmt in range(6):
        for ch in (1, 3):
            x = make_samples(fmt, 5, ch, rng)
            data = sample_bytes(fmt, x)
            cases.append((f"pre{fmt}{ch}", wav_bytes(fmt, ch, 44100, data, before=(odd, fact)), (fmt, ch, 5)))
            cases.append((f"post{fmt}{ch}", wav_bytes(fmt, ch, 48000, data, after=(junk, odd, fact)), (fmt, ch, 5)))
            cases.append((f"both{fmt}{ch}", wav_bytes(fmt, ch, 22050, data, before=(junk,), after=(odd,)), (fmt, ch, 5)))
            cases.append((f"ext{fmt}{ch}", wav_bytes(fmt, ch, 96000, data, extensible=True, before=(fact,)),
                          (fmt, ch, 5)))
    x = make_samples(1, 3, 1, rng)  # 6 bytes of data + an odd fmt chunk: 18-byte fmt (cbSize 0) is even; use 17 + pad
    body = b"WAVE" + chunk(b"fmt ", fmt_body(1, 1, 8000) + b"\0") + chunk(b"data", sample_bytes(1, x))
    cases.append(("oddfmt", b"RIFF" + struct.pack("<I", len(body)) + body, (1, 1, 3)))
    x = make_samples(3, 3, 1, rng)  # odd data, RIFF size without the pad byte, no pad byte in the file
    body = b"WAVE" + chunk(b"fmt ", fmt_body(3, 1, 8000)) + chunk(b"data", sample_bytes(3, x), pad=False)
    cases.append(("nopad", b"RIFF" + struct.pack("<I", len(body)) + body, (3, 1, 3)))
    paths = []
    for name, blob, _ in cases:
        paths.append(tmp_path / f"{name}.wav")
        paths[-1].write_bytes(blob)
    regions, declined = audio_io.probe_wav(paths)
    assert declined == [], [cases[i][0] for i in declined]
    for p, r, (name, _blob, (fmt, ch, n)) in zip(paths, regions, cases):
        assert (r.sample_format, r.channels, r.n_frames) == (fmt, ch, n), name
        assert_agrees_with_scipy(str(p), r)


def declined_cases(tmp_path):
    """name -> path of every kind of file the probe must decline."""
    rng = np.random.default_rng(2)
    x16 = make_samples(1, 6, 2, rng)
    d16 = sample_bytes(1, x16)
    blobs = {
        "rifx": b"RIFX" + struct.pack(">I", 4 + 24 + 8 + len(d16)) + b"WAVE" + b"fmt " +
                struct.pack(">IHHIIHH", 16, 1, 2, 44100, 44100 * 4, 4, 16) + b"data" + struct.pack(">I", len(d16)) +
                np.ascontiguousarray(x16, ">i2").tobytes(),
        "rf64": wav_bytes(1, 2, 44100, d16, riff=b"RF64"),
        "w64": b"riff" + b"\0" * 60,
        "mulaw": wav_bytes(3, 1, 8000, bytes(6), tag=7),
        "alaw": wav_bytes(3, 1, 8000, bytes(6), tag=6),
        "adpcm": wav_bytes(1, 1, 8000, bytes(8), tag=2, bits=4, block=256),
        "int64": wav_bytes(5, 1, 8000, bytes(16), tag=1),
        "float16": wav_bytes(1, 1, 8000, bytes(8), tag=3),
        "24in32": wav_bytes(2, 2, 44100, sample_bytes(2, make_samples(2, 3, 2, rng) & ~0xFF), bits=24, block=8),
        "block_align": wav_bytes(1, 2, 44100, d16, block=6),
        "byte_rate": wav_bytes(1, 2, 44100, d16, rate=12345),
        "ext_guid": wav_bytes(1, 2, 44100, d16, extensible=True, tag=2),
        "ext_cbsize": wav_bytes(1, 2, 44100, d16, extensible=True, cb=0),
        "ext_bad_tail": wav_bytes(1, 2, 44100, d16, extensible=True).replace(GUID_TAIL, b"\x01" * 12),
        "no_fmt": b"RIFF" + struct.pack("<I", 4 + 8 + len(d16)) + b"WAVE" + chunk(b"data", d16),
        "no_data": b"RIFF" + struct.pack("<I", 4 + 24) + b"WAVE" + chunk(b"fmt ", fmt_body(1, 2, 44100)),
        "two_fmt": wav_bytes(1, 2, 44100, d16, before=(chunk(b"fmt ", fmt_body(1, 2, 44100)),)),
        "two_data": wav_bytes(1, 2, 44100, d16, after=(chunk(b"data", d16),)),
        "data_first": b"RIFF" + struct.pack("<I", 4 + 8 + len(d16) + 24) + b"WAVE" + chunk(b"data", d16) +
                      chunk(b"fmt ", fmt_body(1, 2, 44100)),
        "ragged": wav_bytes(1, 2, 44100, d16 + b"\0\0"),
        "truncated": wav_bytes(1, 2, 44100, d16)[:-3],
        "riff_short": wav_bytes(1, 2, 44100, d16, riff_size=4 + 24),  # data beyond what the RIFF size covers
        "riff_zero": wav_bytes(1, 2, 44100, d16, riff_size=0),
        "partial_header": wav_bytes(1, 2, 44100, d16, riff_size=4 + 24 + 8 + len(d16) + 8) + b"LIS",
        "rate_zero": wav_bytes(1, 1, 0, bytes(4)),
        "rate_too_high": wav_bytes(1, 1, 2822400, bytes(4)),
        "channels_zero": wav_bytes(1, 0, 8000, b"", block=0),
        "empty": b"",
        "not_wave": b"RIFF" + struct.pack("<I", 4) + b"AVI ",
        "text": b"hello, world\n",
    }
    paths = {}
    for name, blob in blobs.items():
        paths[name] = tmp_path / f"{name}.wav"
        paths[name].write_bytes(blob)
    paths["missing"] = tmp_path / "does-not-exist.wav"
    paths["directory"] = tmp_path / "adir.wav"
    paths["directory"].mkdir()
    return paths


def outcome(fn):
    try:
        return "ok", fn()
    except Exception as e:  # noqa: BLE001 - the exception itself is the result compared
        return "raise", (type(e), str(e))


def test_declined_files_take_read_pcm(tmp_path):
    """Every kind of file the rules exclude is declined, and the batch routing gives it exactly `read_pcm`'s result or
    exception; files scipy reads (RIFX, 24-bit in a 32-bit container, a repeated data chunk) still work."""
    from basic_pitch_b200 import audio_io, inference

    paths = declined_cases(tmp_path)
    names = list(paths)
    regions, declined = audio_io.probe_wav([paths[k] for k in names])
    assert declined == list(range(len(names))), [names[i] for i in range(len(names)) if i not in declined]
    assert all(r is None for r in regions)
    readable = 0
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        for k in names:
            want = outcome(lambda: audio_io.read_pcm(paths[k]))
            got = outcome(lambda: inference._pcm_items([paths[k]])[0])
            assert got[0] == want[0], k
            if want[0] == "ok":
                readable += 1
                (gx, gsr), (wx, wsr) = got[1], want[1]
                assert gsr == wsr and gx.dtype == wx.dtype and np.array_equal(gx, wx), k
            else:
                assert got[1] == want[1], k
    assert readable >= 3


def test_unreadable_file_is_declined(tmp_path):
    from basic_pitch_b200 import audio_io

    if os.geteuid() == 0:
        pytest.skip("root reads files without read permission")
    p = tmp_path / "locked.wav"
    p.write_bytes(wav_bytes(1, 1, 8000, bytes(4)))
    p.chmod(0)
    try:
        assert audio_io.probe_wav([p]) == ([None], [0])
    finally:
        p.chmod(0o600)


def test_probe_arguments():
    from basic_pitch_b200 import _lib, audio_io

    lib = _lib.load()
    assert audio_io.probe_wav([]) == ([], [])
    lib.bp_probe_wav_files(None, 0, None, None)
    out = (_lib.PcmSource * 2)()
    acc = np.zeros(2, np.int32)
    with pytest.raises(_lib.BpError) as e:
        lib.bp_probe_wav_files((C.c_char_p * 2)(b"a.wav", None), 2, out, acc.ctypes.data)
    assert e.value.code == _lib.BP_E_INVALID and "path 1" in str(e.value)
    with pytest.raises(_lib.BpError):
        lib.bp_probe_wav_files(None, 1, out, acc.ctypes.data)


def test_layout_of_24_bit_and_float64():
    """bp_debug_pcm_sources_layout packs format 4 at 3 and format 5 at 8 bytes per sample, every file on a 16-byte
    boundary, among the other formats, for memory and file sources alike; a bp_pcm_file_t still takes only 0..3, and a
    source format beyond 5 or a negative data offset is refused by index."""
    from basic_pitch_b200 import _lib

    lib = _lib.load()
    spec = [(4, 1, 1), (5, 3, 7), (4, 5, 2), (0, 2, 3), (4, 0, 6), (5, 1, 1), (3, 7, 1), (4, 11, 9), (5, 2, 130)]
    n = len(spec)
    sources = (_lib.PcmSource * n)()
    buf = np.zeros(1 << 16, np.uint8)
    for i, (s, (fmt, frames, ch)) in enumerate(zip(sources, spec)):
        s.pcm.pcm, s.pcm.n_frames, s.pcm.sample_format, s.pcm.channels, s.pcm.sample_rate = buf.ctypes.data, frames, \
            fmt, ch, 44100
        if i % 2:
            s.path, s.data_offset, s.pcm.pcm = b"/nonexistent/only-described.wav", 44 + i, None
    byte_off, sample_off = np.zeros(n + 1, np.int64), np.zeros(n + 1, np.int64)
    lib.bp_debug_pcm_sources_layout(sources, n, byte_off.ctypes.data, sample_off.ctypes.data)
    pos = 0
    for i, (fmt, frames, ch) in enumerate(spec):
        assert byte_off[i] == pos and pos % 16 == 0, i
        pos += -(-frames * ch * BYTES6[fmt] // 16) * 16
        assert sample_off[i + 1] - sample_off[i] == -(-frames * 22050 // 44100)
    assert byte_off[n] == pos
    files = (_lib.PcmFile * 1)(sources[0].pcm)
    with pytest.raises(_lib.BpError) as e:
        lib.bp_debug_pcm_layout(files, 1, byte_off.ctypes.data, sample_off.ctypes.data)
    assert e.value.code == _lib.BP_E_INVALID and "file 0" in str(e.value)
    for field, value in (("sample_format", 6), ("sample_format", -1), ("data_offset", -1)):
        bad = (_lib.PcmSource * n).from_buffer_copy(sources)
        if field == "data_offset":
            bad[3].data_offset = value
        else:
            bad[3].pcm.sample_format = value
        with pytest.raises(_lib.BpError) as e:
            lib.bp_debug_pcm_sources_layout(bad, n, byte_off.ctypes.data, sample_off.ctypes.data)
        assert e.value.code == _lib.BP_E_INVALID and "file 3" in str(e.value), field


def test_routing_splits_a_mixed_batch(tmp_path):
    """`_pcm_items`: arrays stay (float32 mono at 22 050 Hz), accepted WAV files become their probe regions, declined
    files `read_pcm`'s (samples, rate), all in input order; a non-mono array is still a ValueError."""
    from scipy.io import wavfile

    from basic_pitch_b200 import audio_io, inference

    rng = np.random.default_rng(3)
    a16 = tmp_path / "a16.wav"
    wavfile.write(a16, 44100, make_samples(1, 50, 2, rng))
    a24 = tmp_path / "a24.wav"
    a24.write_bytes(wav_bytes(4, 1, 48000, sample_bytes(4, make_samples(4, 40, 1, rng))))
    dec = tmp_path / "dec.wav"  # 24-bit samples in 32-bit containers: scipy reads them, the probe declines
    dec.write_bytes(wav_bytes(2, 2, 44100, sample_bytes(2, make_samples(2, 9, 2, rng) & ~0xFF), bits=24, block=8))
    arr = [np.linspace(-1, 1, 100), np.zeros(7, np.float32)]
    items = inference._pcm_items([arr[0], str(a16), dec, a24, arr[1]])
    assert isinstance(items[0], tuple) and items[0][0].dtype == np.float32 and items[0][1] == 22050
    assert np.array_equal(items[0][0], arr[0].astype(np.float32))
    assert items[1] == audio_io.probe_wav([a16])[0][0] and isinstance(items[1], audio_io.WavRegion)
    x, sr = audio_io.read_pcm(dec)
    assert isinstance(items[2], tuple) and items[2][1] == sr and np.array_equal(items[2][0], x)
    assert items[3].sample_format == 4 and items[3].n_frames == 40
    assert items[4][0] is not arr[1] or items[4][0].dtype == np.float32
    with pytest.raises(ValueError):
        inference._pcm_items([a16, np.zeros((4, 2), np.float32)])
    plain = inference._pcm_items([arr[0], str(a16), dec, a24, arr[1]], wav_in_library=False)  # every path by read_pcm
    for got, path in zip(plain[1:4], (a16, dec, a24)):
        x, sr = audio_io.read_pcm(path)
        assert isinstance(got, tuple) and got[1] == sr and got[0].dtype == x.dtype and np.array_equal(got[0], x)
    sources, keep = audio_io.pcm_sources(items)
    assert sources[1].path == os.fsencode(str(a16)) and sources[1].data_offset == items[1].data_offset
    assert sources[0].path is None and sources[0].pcm.n_frames == 100 and sources[2].pcm.sample_format == 2
