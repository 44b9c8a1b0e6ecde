"""The stream group (bp_stream_group_*, Model.stream_group, inference.predict_streams_notes) against the single note
stream and its oracle (oracle/stream_ref.py), never against itself: every stream of a group must give, bit for bit, what
it gives alone, whatever the other streams do."""
import ctypes as C

import numpy as np
import pytest

from oracle import stream_ref
from tests import postsets, streamsets
from tests.golden_util import dequant
from tests.test_gpu_stream_decode import ev_key, model  # noqa: F401  (fixture)
from tests.test_gpu_stream_edges import Oracle, prm
from tests.test_stream_edges_cpu import schedules

pytestmark = pytest.mark.gpu

SR = 22050


def blocks_of(audio, rng, sizes):
    """`audio` cut into blocks whose lengths are drawn from `sizes` (0-length blocks included)."""
    out, t = [], 0
    while t < len(audio):
        n = int(rng.choice(sizes))
        out.append(audio[t : t + n])
        t += n
    return out


def single(model, blocks, **kw):
    """predict_stream_notes on one recording: its events and its concatenated posteriorgram parts."""
    from basic_pitch_b200.inference import predict_stream_notes

    ev, parts = [], []
    for part, e in predict_stream_notes(iter(blocks), model, **kw):
        ev += e
        parts.append(part)
    return list(map(ev_key, ev)), {k: np.concatenate([p[k] for p in parts]) for k in ("note", "onset", "contour")}


def run_group(model, plans, with_posteriorgrams=True, **kw):
    """plans[i] = (step the stream opens at, its blocks); a stream ends at the step after its last block.  Returns per
    stream the event keys and the concatenated posteriorgram parts."""
    from basic_pitch_b200 import inference as I

    min_note_len = int(np.round(kw.get("minimum_note_length", I.DEFAULT_MINIMUM_NOTE_LENGTH_MS) / 1000 * (SR / 256)))
    max_seg = kw.get("max_segment_seconds")
    max_seg = None if max_seg is None else max(1, int(np.round(max_seg * SR / 256)))
    g = model.stream_group(kw.get("onset_threshold", I.DEFAULT_ONSET_THRESHOLD),
                           kw.get("frame_threshold", I.DEFAULT_FRAME_THRESHOLD), min_note_len,
                           kw.get("minimum_frequency"), kw.get("maximum_frequency"), kw.get("melodia_trick", True), True,
                           max_seg)  # fmt: skip
    ids, ev, parts = {}, {i: [] for i in range(len(plans))}, {i: [] for i in range(len(plans))}
    step, done = 0, set()
    while len(done) < len(plans):
        for i, (open_at, _) in enumerate(plans):
            if open_at == step:
                ids[i] = g.open()
        push, end = {}, []
        for i, (open_at, blocks) in enumerate(plans):
            if i in ids and i not in done:
                k = step - open_at
                if k < len(blocks):
                    push[ids[i]] = blocks[k]
                else:
                    end.append(ids[i])
        back = {v: k for k, v in ids.items()}
        for call, arg in ((g.push, push), (g.end, end)):
            if not arg:
                continue
            res = call(arg, with_posteriorgrams=with_posteriorgrams)
            e, p = res if with_posteriorgrams else (res, {})
            for sid, x in e.items():
                ev[back[sid]] += list(map(ev_key, x))
            for sid, x in p.items():
                parts[back[sid]].append(x)
        for sid in end:
            done.add(back[sid])
            assert g.held_frames(sid) == 0
        step += 1
    cat = {i: {k: np.concatenate([x[k] for x in ps]) if ps else None for k in ("note", "onset", "contour")}
           for i, ps in parts.items()}  # fmt: skip
    return ev, cat


def clips():
    from basic_pitch_b200 import synth

    return [synth.melody_clip(12.0, seed=1), synth.random_notes_clip(9.0, seed=2), synth.dense_chords_clip(10.0),
            synth.tones_clip(6.0, seed=3)]


def vocadito(golden_dir):
    a = np.load(golden_dir / "vocadito10.npz")["audio22k"]
    return dequant(a) if a.dtype.kind in "ui" else np.asarray(a, np.float32)


@pytest.mark.parametrize("n_streams", [1, 2, 7, 40])
def test_audio_streams_equal_the_single_stream(model, golden_dir, n_streams):
    """Random block sizes per stream (0-length, shorter than a hop, several windows), streams opening late and ending
    at different steps, one empty recording and one shorter than a window: every stream's events and posteriorgram
    parts equal predict_stream_notes' on its blocks alone."""
    rng = np.random.default_rng(n_streams)
    sources = clips()
    sources.append(vocadito(golden_dir))
    plans = []
    for i in range(n_streams):
        if i == 1:
            audio = np.zeros(0, np.float32)
        elif i == 2:
            audio = sources[0][: 30_000]
        else:
            audio = sources[i % len(sources)]
        sizes = [0, 500, 22050, 36_164, 90_000] if i % 2 else [22050]
        plans.append((int(rng.integers(0, 4)) if i else 0, blocks_of(audio, rng, sizes)))
    ev, parts = run_group(model, plans)
    for i, (_, blocks) in enumerate(plans):
        exp_ev, exp_parts = single(model, blocks)
        assert ev[i] == exp_ev, i
        for k in ("note", "onset", "contour"):
            if exp_parts[k].shape[0] == 0:
                assert parts[i][k] is None or parts[i][k].shape[0] == 0, (i, k)
            else:
                assert np.array_equal(parts[i][k], exp_parts[k]), (i, k)


def test_push_spanning_forward_chunks_and_settings(model):
    """One push whose windows span more than one forward chunk, and melodia off / a pitch range / a forced cut."""
    from basic_pitch_b200 import synth

    chunk = int(model._lib.bp_model_chunk_windows(model.handle))
    long = np.tile(synth.random_notes_clip(30.0, seed=5), (chunk * 36_164) // (30 * SR) + 2)
    rng = np.random.default_rng(0)
    plans = [(0, [long]), (0, blocks_of(synth.melody_clip(8.0, seed=4), rng, [7000, 40_000]))]
    ev, _ = run_group(model, plans, with_posteriorgrams=False)
    for i, (_, blocks) in enumerate(plans):
        assert ev[i] == single(model, blocks)[0], i
    dense = synth.dense_chords_clip(10.0)
    for kw in (dict(melodia_trick=False), dict(minimum_frequency=200.0, maximum_frequency=900.0),
               dict(max_segment_seconds=1.5)):
        plans = [(0, blocks_of(dense, rng, [SR, 3000])), (1, blocks_of(synth.melody_clip(10.0, seed=6), rng, [SR]))]
        ev, _ = run_group(model, plans, with_posteriorgrams=False, **kw)
        for i, (_, blocks) in enumerate(plans):
            assert ev[i] == single(model, blocks, **kw)[0], (kw, i)


def test_predict_streams_notes(model):
    """The generator: each recording's events, concatenated over the steps, equal predict_stream_notes'."""
    from basic_pitch_b200 import synth
    from basic_pitch_b200.inference import predict_streams_notes

    rng = np.random.default_rng(3)
    recs = [blocks_of(c, rng, [SR, 5000]) for c in (synth.melody_clip(6.0, seed=8), synth.tones_clip(3.0, seed=1))]
    recs.append([])
    got = {i: [] for i in range(len(recs))}
    for step in predict_streams_notes([iter(r) for r in recs], model):
        for i, e in step.items():
            got[i] += list(map(ev_key, e))
    for i, r in enumerate(recs):
        assert got[i] == single(model, r)[0], i


def group_frames_case(model, cases, p, keys, max_seg=0):
    """Carved inputs of one setting spread across one group, stream i pushed under schedule keys[i % len(keys)]: each
    push's events and held frames equal the oracle's, which test_gpu_stream_edges checks bp_stream against."""
    params = model._params(p["onset_thresh"], p["frame_thresh"], p["min_note_len"], p["energy_tol"], p["infer_onsets"],
                           p["melodia_trick"], p["bends"], p["lo"], p["hi"])  # fmt: skip
    from basic_pitch_b200.inference import StreamGroup

    g = StreamGroup(model, params, max_seg)
    refs = [Oracle(out, p, max_seg) for out in cases]
    ends = [schedules(r.n, r.confirming())[keys[i % len(keys)]] for i, r in enumerate(refs)]
    ids = [g.open() for _ in cases]
    got = [[[] for _ in range(len(e) + 1)] for e in ends]
    held = [[] for _ in cases]
    pos = [0] * len(cases)
    for step in range(max(len(e) for e in ends) + 1):
        push, fin = {}, []
        for i, out in enumerate(cases):
            if step < len(ends[i]):
                t, u = pos[i], ends[i][step]
                push[ids[i]] = (out["note"][t:u], out["onset"][t:u], out["contour"][t:u] if p["bends"] else None)
                pos[i] = u
            elif step == len(ends[i]):
                fin.append(ids[i])
        for sid, e in (g.push_frames(push) if push else {}).items():
            i = ids.index(sid)
            got[i][step] = list(map(ev_key, e))
            held[i].append(g.held_frames(sid))
        for sid, e in (g.end(fin) if fin else {}).items():
            got[ids.index(sid)][-1] = list(map(ev_key, e))
    for i, ref in enumerate(refs):
        closed_by, exp_held = stream_ref.push_schedule(ref.plan, p["energy_tol"], ends[i])
        exp = [[] for _ in range(len(ends[i]) + 1)]
        for k, ks in enumerate(ref.keys):
            exp[closed_by[k]] += ks
        assert got[i] == exp, i
        assert held[i] == exp_held, i


@pytest.mark.parametrize("name", postsets.NAMES)
def test_carved_sets_across_a_group(model, name):
    """Every carved file of a set under each setting of its grid, the files of one setting in one group, each under
    its own push schedule (one frame, 7 / 8 / 9, 255 / 256 / 257 / 31, up to each confirmation and one past it, whole):
    several cuts of one stream in one push go through several rounds."""
    files, grid = postsets.get(name)
    keys = ["one", "7-8-9", "255-256-257-31", "to t", "to t + 1", "whole"]
    for j, q in enumerate(grid):
        cases = [streamsets.carved(f, q, 100 * i + j, ("all", "range")[(i + j) % 2])
                 for i, f in enumerate(files) if f[0].shape[0]]
        group_frames_case(model, cases, prm(q), keys[j % len(keys):] + keys[: j % len(keys)])


def test_forced_cuts_and_slot_retry_across_a_group(model):
    """Forced cuts next to quiet ones (streamsets.precedence) and the crowded segments that overflow the first slot
    allowance, several streams per group."""
    for max_seg, tol in ((40, 11), (25, 5)):
        cases = [streamsets.precedence(max_seg, tol, d) for d in (-2, -1, 0, 1)]
        group_frames_case(model, cases, prm(postsets.params(energy_tol=tol)), ["one", "7-8-9", "whole", "to t"], max_seg)
    files, grid = postsets.get("crowded")
    for j, q in enumerate(grid):
        group_frames_case(model, [streamsets.carved(files[1], q, 40 + j)] * 3, prm(q), ["one", "7-8-9", "whole"])


def test_launches_do_not_grow_with_streams(model):
    """N identical streams pushed identical blocks make the same cuts and rounds: the launches of every push are those
    of one stream."""
    from basic_pitch_b200 import synth

    audio = synth.melody_clip(8.0, seed=9)
    blocks = [audio[t : t + SR] for t in range(0, len(audio), SR)]

    def launches(n):
        g = model.stream_group()
        ids = [g.open() for _ in range(n)]
        out = []
        for b in blocks:
            l0 = model.launch_count
            g.push({i: b for i in ids})
            out.append(model.launch_count - l0)
        l0 = model.launch_count
        g.end(ids)
        return out + [model.launch_count - l0]

    one = launches(1)
    assert launches(40) == one
    assert sum(one) > 0


def test_interleaved_with_other_entry_points(model):
    """A group, a NoteStream and whole-file transcriptions alternate on one model: each gives its standalone result."""
    from basic_pitch_b200 import synth

    a, b = synth.melody_clip(6.0, seed=11), synth.random_notes_clip(6.0, seed=12)
    ba, bb = [a[t : t + SR] for t in range(0, len(a), SR)], [b[t : t + 15_000] for t in range(0, len(b), 15_000)]
    exp_a, exp_b = single(model, ba)[0], single(model, bb)[0]
    out = model.run_inference_arrays([b])[0]
    cuts = list(range(0, out["note"].shape[0], 150)) + [out["note"].shape[0]]

    def note_stream(between=None):
        s, ev = model.note_stream(), []
        for k in range(len(cuts) - 1):
            t, u = cuts[k], cuts[k + 1]
            ev += s.push(out["note"][t:u], out["onset"][t:u], out["contour"][t:u])
            if between:
                between(k)
        return list(map(ev_key, ev + s.end()))

    alone_ns = note_stream()
    alone_tr = model.transcribe_arrays([a])[1][0]
    g = model.stream_group()
    ia, ib = g.open(), g.open()
    got = {ia: [], ib: []}

    def step(k):
        push = {i: bl[k] for i, bl in ((ia, ba), (ib, bb)) if k < len(bl)}
        for sid, e in (g.push(push) if push else {}).items():
            got[sid] += list(map(ev_key, e))
        tr = model.transcribe_arrays([a])[1][0]
        assert all(np.array_equal(tr[k2], alone_tr[k2]) for k2 in ("start", "end", "pitch", "amp"))

    assert note_stream(step) == alone_ns
    for k in range(len(cuts) - 1, max(len(ba), len(bb))):
        step(k)
    for sid, e in g.end([ia, ib]).items():
        got[sid] += list(map(ev_key, e))
    assert got[ia] == exp_a and got[ib] == exp_b


def test_errors_and_capacity(model):
    from basic_pitch_b200 import _lib

    lib = model._lib
    g = model.stream_group()
    a, f = g.open(), g.open()
    g.push({a: np.zeros(1000, np.float32)})
    n = np.random.default_rng(0).random((50, 88), dtype=np.float32)
    g.push_frames({f: (n, n, np.zeros((50, 264), np.float32))})

    def invalid(fn):
        with pytest.raises(_lib.BpError) as e:
            fn()
        assert e.value.code == _lib.BP_E_INVALID

    invalid(lambda: g.push({99: np.zeros(10, np.float32)}))  # unknown id
    invalid(lambda: g.push({f: np.zeros(10, np.float32)}))  # mixed kinds
    invalid(lambda: g.push_frames({a: (n, n, np.zeros((50, 264), np.float32))}))
    ids = (C.c_int32 * 1)(a)
    neg = (C.c_int64 * 1)(-1)
    ptrs = (C.c_void_p * 1)(None)
    invalid(lambda: lib.bp_stream_group_push_host(g._h, 1, ids, ptrs, neg, None, None, None, None))
    ten = (C.c_int64 * 1)(10)
    invalid(lambda: lib.bp_stream_group_push_host(g._h, 1, ids, ptrs, ten, None, None, None, None))
    g.end([a])
    invalid(lambda: g.push({a: np.zeros(10, np.float32)}))  # ended
    invalid(lambda: g.end([a]))
    # take capacity: notes stay queued and bp_last_required says how many
    from basic_pitch_b200 import synth

    clip = synth.random_notes_clip(6.0, seed=4)
    c = g.open()
    g2 = model.stream_group()
    c2 = g2.open()
    want = g2.push({c2: clip})
    want.update(g2.end([c2]))
    lib.bp_stream_group_push_host(g._h, 1, (C.c_int32 * 1)(c), (C.c_void_p * 1)(clip.ctypes.data),
                                  (C.c_int64 * 1)(len(clip)), None, None, None, None)
    lib.bp_stream_group_end(g._h, 1, (C.c_int32 * 1)(c), None, None, None, None)
    exp = len(want[c2])
    assert exp > 1
    notes, arrs = model._alloc_notes(1, exp - 1, 1 << 16)
    with pytest.raises(_lib.BpError) as e:
        lib.bp_stream_group_take(g._h, 1, (C.c_int32 * 1)(c), C.byref(notes))
    assert e.value.code == _lib.BP_E_CAPACITY
    need_n, need_b = C.c_int64(0), C.c_int64(0)
    lib.bp_last_required(C.byref(need_n), C.byref(need_b))
    assert need_n.value == exp
    got = g._take(np.array([c], np.int32))[c]
    assert list(map(ev_key, got)) == list(map(ev_key, want[c2]))
