"""Live PCM streams of a stream group (bp_stream_group_open_pcm / push_pcm_host, StreamGroup.open_pcm,
predict_streams_notes(sample_rates=...)) against the whole-file ingest bp_load_pcm_host and the single-stream routes,
bit for bit: whatever the block schedule, a stream's 22 050 Hz signal is the whole recording's, its frames are
run_inference_stream's on that signal and its notes predict_stream_notes'."""
import ctypes as C

import numpy as np
import pytest

from tests.test_gpu_ingest import FORMATS, RATES, make_pcm
from tests.test_gpu_stream_decode import ev_key, model  # noqa: F401  (fixture)
from tests.test_gpu_stream_group import single
from tests.test_stream_pcm_cpu import schedules

pytestmark = pytest.mark.gpu


def load_whole(model, pcm, sr):
    """bp_load_pcm_host of the whole recording ((n,) or (n, channels))."""
    from basic_pitch_b200 import audio_io

    x = np.ascontiguousarray(pcm)
    n = x.shape[0]
    ch = 1 if x.ndim == 1 else x.shape[1]
    out = np.empty(int(model._lib.bp_resampled_length(n, sr)), np.float32)
    model._lib.bp_load_pcm_host(model.handle, x.ctypes.data if n else None, audio_io._PCM_FORMATS[x.dtype], n, ch, sr,
                                out.ctypes.data)
    return out


def cut(pcm, frames):
    at = np.cumsum([0] + list(frames))
    return [pcm[at[i] : at[i + 1]] for i in range(len(frames))]


def final_count(lib, fmt, ch, sr, frames):
    """Per push, the samples the stream holds as final (bp_debug_pcm_stream_plan's out_hi)."""
    fr = np.ascontiguousarray(frames, np.int64)
    o = [np.zeros(len(fr) + 1, np.int64) for _ in range(4)]
    lib.bp_debug_pcm_stream_plan(fmt, ch, sr, len(fr), fr.ctypes.data if len(fr) else None, 1, *[x.ctypes.data for x in o])
    return o[1]


def bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


def run_signal_group(model, streams, ending=False):
    """streams: [(sr, pcm, frames)], all opened in one group and pushed together step by step.  Returns per stream the
    22 050 Hz signal stitched from debug_tail after every push, the sample count after every push, and the group."""
    g = model.stream_group()
    ids = [g.open_pcm(sr, 1 if p.ndim == 1 else p.shape[1], p.dtype) for sr, p, _ in streams]
    blocks = [cut(p, fr) for _, p, fr in streams]
    sig = [np.full(400_000, np.nan, np.float32) for _ in streams]
    counts = [[] for _ in streams]
    for step in range(max(len(b) for b in blocks)):
        push = {ids[i]: b[step] for i, b in enumerate(blocks) if step < len(b)}
        g.push(push)
        for i, sid in enumerate(ids):
            first, tail = g.debug_tail(sid)
            sig[i][first : first + len(tail)] = tail
            if sid in push:
                counts[i].append(first + len(tail))
    return sig, counts, g, ids


def capped(sr, frames):
    """The schedule cut short so that the recording stays below a window (no window runs before the end, so the whole
    signal stays in the tail) and its PCM stays small."""
    cap = min(int(1.4 * sr), 150_000)
    out, t = [], 0
    for f in frames:
        f = min(f, cap - t)
        out.append(f)
        t += f
    return out


@pytest.mark.parametrize("sr", RATES)
def test_signal_is_the_whole_file_ingest(model, sr):
    """Every format, channels 1..3 and every schedule of the CPU plan test, all as streams of one group: after each push
    the stream holds exactly F(n) samples, and the samples stitched from its tail are bp_load_pcm_host(whole) bit for
    bit."""
    rng = np.random.default_rng(sr + 1)
    streams = []
    for fmt, dt in enumerate(FORMATS):
        for ch in (1, 2, 3):
            for frames in schedules(sr, rng):
                frames = capped(sr, frames)
                sig = "noise" if (fmt + ch + len(frames)) % 2 else "extremes"
                streams.append((sr, make_pcm(dt, sum(frames), ch, sig, sr, rng), frames, fmt, ch))
    sig, counts, _, _ = run_signal_group(model, [s[:3] for s in streams])
    for i, (_, pcm, frames, fmt, ch) in enumerate(streams):
        exp_counts = final_count(model._lib, fmt, ch, sr, frames)
        assert counts[i] == list(exp_counts[: len(frames)]), (fmt, ch, frames)
        n_final = int(exp_counts[len(frames) - 1]) if frames else 0
        whole = load_whole(model, pcm, sr)
        assert np.array_equal(bits(sig[i][:n_final]), bits(whole[:n_final])), (fmt, ch, frames)


def test_signal_130_channels(model):
    """A 130-channel int16 stream (the pairwise sum splits above 128 channels)."""
    rng = np.random.default_rng(130)
    frames = [0, 1, 300, 4, 20_000, 7, 10_001]
    pcm = make_pcm(np.int16, sum(frames), 130, "noise", 44100, rng)
    sig, counts, _, _ = run_signal_group(model, [(44100, pcm, frames)])
    exp_counts = final_count(model._lib, 1, 130, 44100, frames)
    assert counts[0] == list(exp_counts[:-1])
    n = int(exp_counts[-2])
    assert np.array_equal(bits(sig[0][:n]), bits(load_whole(model, pcm, 44100)[:n]))


def test_region_moves_keep_the_signal(model):
    """Twenty streams with doubling blocks outgrow their audio regions push after push; every move shows as one copy
    launch besides the ingest, and the signal stays bit-exact."""
    rng = np.random.default_rng(7)
    streams = []
    for i in range(20):
        sr = (48000, 16000, 44100, 8000)[i % 4]
        frames = [0] + [min(2**k + i, 12_000) for k in range(15)]
        frames = capped(sr, frames)
        streams.append((sr, make_pcm((np.int16, np.float32)[i % 2], sum(frames), 1 + i % 2, "noise", sr, rng), frames))
    g = model.stream_group()
    ids = [g.open_pcm(sr, 1 if p.ndim == 1 else p.shape[1], p.dtype) for sr, p, _ in streams]
    blocks = [cut(p, fr) for _, p, fr in streams]
    sig = [np.full(400_000, np.nan, np.float32) for _ in streams]
    moves = 0
    for step in range(len(blocks[0])):
        before = model.launch_count
        g.push({ids[i]: b[step] for i, b in enumerate(blocks)})
        moves += max(0, model.launch_count - before - 1)  # the ingest, then any region move
        for i, sid in enumerate(ids):
            first, tail = g.debug_tail(sid)
            sig[i][first : first + len(tail)] = tail
    assert moves >= 5
    for i, (sr, pcm, frames) in enumerate(streams):
        n = int(final_count(model._lib, 1, 1, sr, frames)[len(frames) - 1])
        assert np.array_equal(bits(sig[i][:n]), bits(load_whole(model, pcm, sr)[:n])), i


def odd_blocks(pcm, rng, sizes):
    out, t = [], 0
    while t < len(pcm):
        n = int(rng.choice(sizes))
        out.append(pcm[t : t + n])
        t += n
    return out


def stereo_48k(seconds=20.0):
    """A 48 kHz int16 stereo clip: a synth melody rendered at 22 050 Hz, resampled and quantised."""
    import scipy.signal

    from basic_pitch_b200 import synth

    x = synth.melody_clip(seconds, seed=11).astype(np.float64)
    y = scipy.signal.resample_poly(x, 320, 147)
    lr = np.stack([y, 0.6 * np.roll(y, 37)], axis=1)
    return np.clip(np.round(lr * 0.8 * 32767), -32768, 32767).astype(np.int16)


def test_end_to_end_equals_the_whole_file(model, golden_dir):
    """vocadito10 as stored (int16, 44.1 kHz) and a 48 kHz int16 stereo clip, pushed in odd blocks: the committed
    posteriorgrams are run_inference_stream's on bp_load_pcm_host(whole) bit for bit and the events
    predict_stream_notes' on that signal, through StreamGroup and through predict_streams_notes(sample_rates=...)."""
    from basic_pitch_b200.inference import predict_streams_notes

    z = np.load(golden_dir / "vocadito10_pcm44k.npz")
    recs = [(z["pcm"], int(z["sample_rate"])), (stereo_48k(), 48000)]
    rng = np.random.default_rng(3)
    for pcm, sr in recs:
        whole = load_whole(model, pcm, sr)
        exp_ev, exp_parts = single(model, [whole[i : i + 30_000] for i in range(0, len(whole), 30_000)])
        blocks = odd_blocks(pcm, rng, [0, 1, 333, 4_410, 48_000, 100_003])
        g = model.stream_group()
        sid = g.open_pcm(sr, 1 if pcm.ndim == 1 else pcm.shape[1], pcm.dtype)
        ev, parts = [], []
        for b in blocks + [None]:
            e, p = g.push({sid: b}, with_posteriorgrams=True) if b is not None else g.end([sid], with_posteriorgrams=True)
            ev += list(map(ev_key, e[sid]))
            parts.append(p[sid])
        for k in ("note", "onset", "contour"):
            got = np.concatenate([p[k] for p in parts])
            assert np.array_equal(bits(got), bits(exp_parts[k])), (sr, k)
        assert ev == exp_ev, sr
        got_ev = []
        for step in predict_streams_notes([iter(blocks)], model, sample_rates=[sr]):
            got_ev += list(map(ev_key, step.get(0, [])))
        assert got_ev == exp_ev, sr


def test_predict_streams_notes_mixes_rates_and_refuses_a_changed_format(model):
    """Recordings with and without a rate (and an empty one with a rate) in one call; a block whose dtype or channel
    count differs from the recording's first raises ValueError."""
    from basic_pitch_b200 import synth
    from basic_pitch_b200.inference import predict_streams_notes

    clip = synth.tones_clip(5.0, seed=4)
    pcm = stereo_48k(6.0)
    streams = [[clip[i : i + 22050] for i in range(0, len(clip), 22050)], [pcm[i : i + 48000] for i in range(0, len(pcm), 48000)], []]
    got = {0: [], 1: [], 2: []}
    for step in predict_streams_notes([iter(s) for s in streams], model, sample_rates=[None, 48000, 16000]):
        for k, ev in step.items():
            got[k] += list(map(ev_key, ev))
    assert got[0] == single(model, streams[0])[0]
    assert got[1] == single(model, [load_whole(model, pcm, 48000)])[0]
    assert got[2] == []
    for bad in (pcm[:100].astype(np.int32), pcm[:100, :1]):
        with pytest.raises(ValueError):
            for _ in predict_streams_notes([iter([pcm[:48000], bad])], model, sample_rates=[48000]):
                pass


def test_mixed_group_each_stream_as_alone(model):
    """Plain float streams, PCM streams at different rates and formats, and a posteriorgram stream in one group; the
    audio ones in the same push calls.  Each equals its own single-stream result, and a plain stream's frames are those
    it gets through push_host."""
    from basic_pitch_b200 import synth

    rng = np.random.default_rng(5)
    plain = [synth.melody_clip(8.0, seed=21), synth.dense_chords_clip(6.0)]
    pcms = [(stereo_48k(7.0), 48000),
            ((synth.random_notes_clip(7.0, seed=22) * 127 + 128).astype(np.uint8), 22050),
            (np.repeat((synth.tones_clip(6.0, seed=23) * 2**30).astype(np.int32)[::2, None], 3, axis=1), 11025),
            (synth.melody_clip(9.0, seed=24)[::7].copy(), 3150)]  # fmt: skip
    g = model.stream_group()
    ids_plain = [g.open() for _ in plain]
    ids_pcm = [g.open_pcm(sr, 1 if p.ndim == 1 else p.shape[1], p.dtype) for p, sr in pcms]
    id_post = g.open()
    pb = [odd_blocks(a, rng, [0, 777, 22050, 40_000]) for a in plain]
    cb = [odd_blocks(p, rng, [0, 1, 999, sr // 2 + 3]) for p, sr in pcms]
    _, frames = single(model, [synth.tones_clip(4.0, seed=25)])  # the posteriorgram stream's input, in three parts
    post = [{k: v[a:b] for k, v in frames.items()} for a, b in ((0, 100), (100, 101), (101, None))]
    post_ev = []
    ev = {i: [] for i in ids_plain + ids_pcm}
    parts = {i: [] for i in ids_plain + ids_pcm}
    steps = max(len(b) for b in pb + cb)
    for step in range(steps + 1):
        push = {}
        for sid, b in zip(ids_plain + ids_pcm, pb + cb):
            if step < len(b):
                push[sid] = b[step]
        end = [sid for sid, b in zip(ids_plain + ids_pcm, pb + cb) if step == len(b)]
        if push:
            e, p = g.push(push, with_posteriorgrams=True)
            for sid in push:
                ev[sid] += list(map(ev_key, e[sid]))
                parts[sid].append(p[sid])
        if end:
            e, p = g.end(end, with_posteriorgrams=True)
            for sid in end:
                ev[sid] += list(map(ev_key, e[sid]))
                parts[sid].append(p[sid])
        if step < 3:
            post_ev += list(map(ev_key, g.push_frames({id_post: tuple(post[step][k] for k in ("note", "onset", "contour"))})[id_post]))
    post_ev += list(map(ev_key, g.end([id_post])[id_post]))
    alone = model.note_stream()
    exp_post = []
    for x in post:
        exp_post += list(map(ev_key, alone.push(x["note"], x["onset"], x["contour"])))
    exp_post += list(map(ev_key, alone.end()))
    assert post_ev == exp_post
    for sid, blocks in zip(ids_plain, pb):
        exp_ev, exp_parts = single(model, blocks)
        assert ev[sid] == exp_ev
        for k in ("note", "onset", "contour"):
            assert np.array_equal(bits(np.concatenate([x[k] for x in parts[sid]])), bits(exp_parts[k]))
    for sid, (p, sr) in zip(ids_pcm, pcms):
        exp_ev, exp_parts = single(model, [load_whole(model, p, sr)])
        assert ev[sid] == exp_ev, sr
        for k in ("note", "onset", "contour"):
            assert np.array_equal(bits(np.concatenate([x[k] for x in parts[sid]])), bits(exp_parts[k])), (sr, k)


def test_launch_counts(model):
    """N = 1 and N = 40 identical PCM streams make the same launches push by push; a PCM push makes the launches of a
    float push of the samples it produces, the ingest launch in place of the append copy (and one launch when the block
    only adds to the history)."""
    pcm = stereo_48k(12.0)
    frames = [0, 1, 5, 48_000, 0, 100_000, 70_001, 3, 200_000]
    frames.append(len(pcm) - sum(frames))
    blocks = cut(pcm, frames)
    produced = np.diff(np.concatenate([[0], final_count(model._lib, 1, 2, 48000, frames)]))
    whole = load_whole(model, pcm, 48000)
    at = np.concatenate([[0], np.cumsum(produced)])

    def counts(n_streams, pcm_route):
        g = model.stream_group()
        ids = [g.open_pcm(48000, 2, np.int16) if pcm_route else g.open() for _ in range(n_streams)]
        out = []
        for p in range(len(frames) + 1):
            before = model.launch_count
            if p == len(frames):
                g.end(ids)
            elif pcm_route:
                g.push({i: blocks[p] for i in ids})
            else:
                g.push({i: whole[at[p] : at[p + 1]] for i in ids})
            out.append(model.launch_count - before)
        return out

    one, forty, flt = counts(1, True), counts(40, True), counts(1, False)
    assert one == forty
    for p in range(len(frames)):
        assert one[p] == flt[p] + (1 if produced[p] == 0 and frames[p] > 0 else 0), (p, one, flt)


def test_validation_leaves_the_group_usable(model):
    from basic_pitch_b200 import _lib

    lib = model._lib
    g = model.stream_group()
    sid = C.c_int32(0)
    for fmt, ch, sr in ((4, 1, 48000), (1, 0, 48000), (1, 1, 0), (1, 2, 2_822_400)):
        with pytest.raises(_lib.BpError) as e:
            lib.bp_stream_group_open_pcm(g._h, fmt, ch, sr, C.byref(sid))
        assert e.value.code == _lib.BP_E_INVALID
    a = g.open_pcm(48000, 2, np.int16)
    post = g.open()
    g.push_frames({post: (np.zeros((5, 88), np.float32), np.zeros((5, 88), np.float32), np.zeros((5, 264), np.float32))})
    ids = np.array([a], np.int32)
    block = np.zeros((100, 2), np.int16)
    ptrs = (C.c_void_p * 1)(block.ctypes.data)
    null = (C.c_void_p * 1)(None)

    def refused(call, *args):
        with pytest.raises(_lib.BpError) as e:
            call(g._h, *args)
        assert e.value.code == _lib.BP_E_INVALID

    refused(lib.bp_stream_group_push_host, 1, ids.ctypes.data, ptrs, np.array([100], np.int64).ctypes.data, None, None, None, None)
    refused(lib.bp_stream_group_push_pcm_host, 1, np.array([post], np.int32).ctypes.data, ptrs,
            np.array([100], np.int64).ctypes.data, None, None, None, None)
    refused(lib.bp_stream_group_push_pcm_host, 1, ids.ctypes.data, null, np.array([100], np.int64).ctypes.data, None, None, None, None)
    refused(lib.bp_stream_group_push_pcm_host, 1, ids.ctypes.data, ptrs, np.array([-1], np.int64).ctypes.data, None, None, None, None)
    refused(lib.bp_stream_group_push_pcm_host, 1, ids.ctypes.data, ptrs, np.array([2**61], np.int64).ctypes.data, None, None, None, None)
    before = model.launch_count
    first, tail = g.debug_tail(a)
    assert (first, len(tail)) == (0, 0) and model.launch_count == before  # nothing was enqueued
    pcm = make_pcm(np.int16, 96_000, 2, "noise", 48000, np.random.default_rng(1))
    g.push({a: pcm[:50_000]})
    g.push({a: pcm[50_000:]})
    first, tail = g.debug_tail(a)
    n = first + len(tail)
    assert n == int(final_count(lib, 1, 2, 48000, [50_000, 46_000])[1])
    assert np.array_equal(bits(tail), bits(load_whole(model, pcm, 48000)[first:n]))
    g.end([a, post])
