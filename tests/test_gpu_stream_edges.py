"""The note stream on the device (bp_stream_*, csrc/stream.cu, api.cu) on adversarial posteriorgrams, bit for bit: every
decode edge set of tests/postsets.py with quiet runs carved into it, under every setting of its grid and push schedules
that end on, after and around every confirming frame; the corners of the quiet scan (chunk and warp edges, runs longer
than a chunk, more rows in one push than one grid of CTAs covers); forced cuts next to quiet ones; the slot-allowance
retry; degenerate settings; two streams and the other entry points interleaved on one model; the take's capacity
check; and predict_stream_notes end to end.

Every push is checked against oracle/stream_ref.py: the notes of exactly the segments whose cuts it confirms (events in
order, amplitude and pitch-bend bytes), the frames held after it, and the kernel launches it makes.  Run with -s to see
the counts of cases, cuts, pushes and scan offsets reached."""
import ctypes as C
import time

import numpy as np
import pytest

from oracle import stream_ref
from tests import postsets, streamsets
from tests.test_gpu_stream_decode import ev_key, model  # noqa: F401  (fixture)
from tests.test_stream_edges_cpu import scan_starts, schedules

pytestmark = pytest.mark.gpu

STATS = dict(cases=0, cuts=0, forced=0, pushes=0, retried=0, largest_push=0)
OFFSETS = set()


def prm(q, bends=True):
    """A tests/postsets.py setting as the stream takes it."""
    return dict(onset_thresh=q["onset_thresh"], frame_thresh=q["frame_thresh"], min_note_len=q["min_note_len"],
                energy_tol=q["energy_tol"], infer_onsets=q["infer_onsets"], melodia_trick=q["melodia_trick"],
                bends=bends, lo=q["lo_col"], hi=q["hi_col"])


class Oracle:
    """The stream's expected output for one (input, setting, max_segment_frames), computed once and checked against any
    push schedule: per segment its event keys, the notes its decode range yields before the start filter, and the
    plan."""

    def __init__(self, out, p, max_seg=0):
        self.p, self.max_seg, self.n = p, max_seg, out["note"].shape[0]
        decoded = []
        segs, self.plan = stream_ref.stream_notes(
            out, p["onset_thresh"], p["frame_thresh"], p["infer_onsets"], p["min_note_len"], p["melodia_trick"],
            p["energy_tol"], p["lo"], p["hi"], p["bends"], max_seg, decoded=decoded)  # fmt: skip
        self.decoded = decoded
        self.kept = [len(s) for s in segs]
        ev = stream_ref.events([x for s in segs for x in s], self.n)
        keys, k = list(map(ev_key, ev)), 0
        self.keys = []
        for s in segs:
            self.keys.append(keys[k : k + len(s)])
            k += len(s)
        self.conf = stream_ref.confirmations(self.plan, p["energy_tol"])

    def confirming(self):
        return [t for t, _ in self.conf]

    def launches(self, ends):
        """Kernel launches of each push (and of the end) by bp_stream_push_host's rule: one scan per push of frames; per
        segment it closes one more scan unless the cut was confirmed on the last frame pushed, and 3 decode launches per
        attempt (a second when the first allowance of min(88 T, 8 T + 64) note slots overflows), the compaction if the
        decode found notes and the note finish if some start in the segment."""
        closed_by, _ = stream_ref.push_schedule(self.plan, self.p["energy_tol"], ends)
        out, prev = [0] * (len(ends) + 1), 0
        for j, e in enumerate(ends):
            out[j] += e > prev
            prev = e
        for k, (a, b, s, e, r) in enumerate(self.plan):
            j = closed_by[k]
            if k < len(self.conf):
                out[j] += self.conf[k][0] != ends[j] - 1
            if e > s and b > a:
                t = e - s
                out[j] += 3 * (2 if self.decoded[k] > min(88 * t, 8 * t + 64) else 1)
                out[j] += (self.decoded[k] > 0) + (self.kept[k] > 0)
        return out


def run(model, out, p, ends, max_seg=0):
    """Pushes ending at the frames `ends`, then the end: (event keys per push and of the end, held frames after each
    push, launches of each)."""
    from basic_pitch_b200.inference import NoteStream

    params = model._params(p["onset_thresh"], p["frame_thresh"], p["min_note_len"], p["energy_tol"], p["infer_onsets"],
                           p["melodia_trick"], p["bends"], p["lo"], p["hi"])  # fmt: skip
    s = NoteStream(model, params, max_seg)
    got, held, nl, t = [], [], [], 0
    for u in ends:
        l0 = model.launch_count
        ev = s.push(out["note"][t:u], out["onset"][t:u], out["contour"][t:u] if p["bends"] else None)
        nl.append(model.launch_count - l0)
        got.append(list(map(ev_key, ev)))
        held.append(s.held_frames)
        STATS["largest_push"] = max(STATS["largest_push"], u - t)
        t = u
    l0 = model.launch_count
    got.append(list(map(ev_key, s.end())))
    nl.append(model.launch_count - l0)
    assert s.held_frames == 0
    STATS["pushes"] += len(ends)
    return got, held, nl


def check(model, out, p, ends, ref: Oracle, label=""):
    """One schedule against the oracle: each push returns exactly the segments it closes, holds exactly the frames the
    open segment needs, and makes the launches the rule gives.  Returns the events of the whole stream."""
    got, held, nl = run(model, out, p, ends, ref.max_seg)
    closed_by, exp_held = stream_ref.push_schedule(ref.plan, p["energy_tol"], ends)
    exp = [[] for _ in range(len(ends) + 1)]
    for k, keys in enumerate(ref.keys):
        exp[closed_by[k]] += keys
    for j in range(len(exp)):
        assert got[j] == exp[j], (label, "push", j, "of", len(ends))
    assert held == exp_held, label
    assert nl == ref.launches(ends), label
    for t, s0 in scan_starts(ref.plan, p["energy_tol"], ends):
        OFFSETS.add(t - s0)
    return [e for g in got for e in g]


def count(ref: Oracle):
    STATS["cases"] += 1
    STATS["cuts"] += len(ref.conf)
    STATS["forced"] += sum(f for _, f in ref.conf)
    for k, (a, b, s, e, r) in enumerate(ref.plan):
        STATS["retried"] += ref.decoded[k] > min(88 * (e - s), 8 * (e - s) + 64) if e > s else 0


def whole_file(model, out, p):
    from basic_pitch_b200.note_creation import note_events_from_arrays

    res = model.decode_arrays([out["note"]], [out["onset"]], [out["contour"]], p["onset_thresh"], p["frame_thresh"],
                              p["min_note_len"], p["energy_tol"], p["infer_onsets"], p["melodia_trick"], True, p["lo"],
                              p["hi"])[0]  # fmt: skip
    return sorted(map(ev_key, note_events_from_arrays(res, out["note"].shape[0])))


def report(what):
    corners = sorted(OFFSETS & {0, 1, 31, 32, 255, 256, 257, 511, 512, 513})
    print(f"\n{what}: so far {STATS['cases']} cases, {STATS['cuts']} cuts ({STATS['forced']} forced), {STATS['pushes']} "
          f"pushes, {STATS['retried']} segments through the slot retry, largest push {STATS['largest_push']} frames; "
          f"confirming frames at {len(OFFSETS)} distinct offsets from the scan start, among them {corners}")


# ------------------------------------------------------------------------------------------------ 1, 2: every set
@pytest.mark.parametrize("name", postsets.NAMES)
def test_every_carved_set_through_the_stream(model, name):
    """Every carved file under every setting of its grid, pushed one frame at a time, 7 / 8 / 9, 255 / 256 / 257 / 31,
    up to each confirming frame, one past it, and all at once; then against the whole-file decode where the stream is
    exact: infer_onsets off, or with the recording's maxima in front (maxima_prefix)."""
    t0 = time.time()
    exact = prefixed = 0
    for label, out, q in streamsets.carved_cases(name):
        p = prm(q)
        ref = Oracle(out, p)
        count(ref)
        conf, n = ref.confirming(), ref.n
        sch = schedules(n, conf)
        for key in ("one", "7-8-9", "255-256-257-31", "to t", "to t + 1", "whole"):
            ev = check(model, out, p, sch[key], ref, f"{label} {key}")
        if not p["infer_onsets"]:
            assert sorted(ev) == whole_file(model, out, p), label
            exact += 1
        elif not (np.isnan(out["note"]).any() or np.isnan(out["onset"]).any()):
            pre = streamsets.maxima_prefix(out, p["lo"], p["hi"])
            mo, mf = stream_ref.whole_maxima(pre, p["lo"], p["hi"])
            assert mf >= stream_ref.whole_maxima(out, p["lo"], p["hi"])[1] and mo >= stream_ref.whole_maxima(out, p["lo"], p["hi"])[0]
            got, _, _ = run(model, pre, p, schedules(pre["note"].shape[0], [])["7-8-9"])
            assert sorted(e for g in got for e in g) == whole_file(model, pre, p), label
            prefixed += 1
    assert exact + prefixed > 0
    report(f"{name} ({exact} exact, {prefixed} with the maxima in front, {time.time() - t0:.1f} s)")


# ------------------------------------------------------------------------------------------------ 3: scan geometry
def test_scan_geometry(model):
    """The placed inputs under every schedule (pushes ending at, one before and two before each confirming frame put
    it at scan offsets 0 and 1); the long stream whole, in pieces of 32 768 and 32 769 frames and up to each confirming
    frame."""
    for label, out, q in streamsets.geometry_cases():
        p = prm(q)
        ref = Oracle(out, p)
        count(ref)
        for key, ends in schedules(ref.n, ref.confirming()).items():
            ev = check(model, out, p, ends, ref, f"{label} {key}")
        assert sorted(ev) == whole_file(model, out, p), label
    assert {0, 1, 255, 256, 257} <= OFFSETS
    out = streamsets.long_stream()
    p = prm(streamsets.LONG_SETTING)
    ref = Oracle(out, p)
    count(ref)
    n = ref.n
    assert n > 2 * streamsets.SCAN_MAX_CTAS * streamsets.SCAN_ROWS_PER_CTA
    for ends in ([n], list(range(32768, n, 32768)) + [n], list(range(32769, n, 32769)) + [n],
                 schedules(n, ref.confirming())["to t"]):
        ev = check(model, out, p, ends, ref, "long stream")
    assert sorted(ev) == whole_file(model, out, p)
    report("scan geometry")


# ------------------------------------------------------------------------------------------------ 4: forced cuts
def test_forced_cuts(model):
    """M = 1, 2, 3, w - 1, w, w + 1 and 64 on carved inputs; quiet cuts confirmed at a + M - 2, a + M - 1 (they win), a + M
    and a + M + 1 (the forced cut comes first)."""
    files = [(postsets.get("long_notes")[0][0], postsets.get("long_notes")[1][0]),
             (postsets.get("pitch_edges")[0][0], postsets.get("pitch_edges")[1][0])]
    for i, (f, q) in enumerate(files):
        f = tuple(a[:900] for a in f)
        out = streamsets.carved(f, q, 7 + i)
        p = prm(q)
        w = q["energy_tol"] + 3
        for m in (1, 2, 3, w - 1, w, w + 1, 64):
            ref = Oracle(out, p, m)
            count(ref)
            assert sum(fc for _, fc in ref.conf) > 0
            sch = schedules(ref.n, ref.confirming())
            for key in ("7-8-9", "to t", "to t + 1", "whole") + (("one",) if m <= 3 or m == 64 else ()):
                check(model, out, p, sch[key], ref, f"file {i} M {m} {key}")
    q = dict(postsets.params(min_note_len=0, infer_onsets=False), energy_tol=11)
    p = prm(q)
    for d in (-2, -1, 0, 1):
        out = streamsets.precedence(40, 11, d)
        ref = Oracle(out, p, 40)
        count(ref)
        forced = [fc for _, fc in ref.conf]
        assert len(forced) >= 4 and all(forced[:4]) == (d >= 0) and any(forced[:4]) == (d >= 0), (d, ref.conf)
        for key, ends in schedules(ref.n, ref.confirming()).items():
            check(model, out, p, ends, ref, f"precedence d {d} {key}")
    report("forced cuts")


# ------------------------------------------------------------------------------------------------ 5: degenerate
def test_degenerate_settings(model):
    base = streamsets.gapped(11, streamsets.gap_lengths(11) * 2)
    for lo, hi in ((0, 0), (50, 20)):  # no column in range: every frame is quiet, one cut at 3
        p = prm(postsets.params(lo_col=lo, hi_col=hi))
        ref = Oracle(base, p)
        assert [b for a, b, s, e, r in ref.plan[:-1]] == [3]
        for key, ends in schedules(ref.n, ref.confirming()).items():
            check(model, base, p, ends, ref, f"range {lo} {hi} {key}")
    for tol in (1, 2, 2**31 - 1):
        out = streamsets.gapped(12, streamsets.gap_lengths(min(tol, 20)) * 2)
        for infer in (False, True):
            p = prm(postsets.params(min_note_len=0, energy_tol=tol, infer_onsets=infer))
            ref = Oracle(out, p)
            count(ref)
            assert (len(ref.conf) == 0) == (tol > 100)
            for key, ends in schedules(ref.n, ref.confirming()).items():
                check(model, out, p, ends, ref, f"tol {tol} {key}")
    # time-constant first segments: max(frame_diff) over them is 0, so their inferred onsets are NaN; later ones are not
    rest = streamsets.gapped(13, streamsets.gap_lengths(11))
    const = {"note": np.concatenate([np.full((40, 88), 0.5, np.float32), np.zeros((20, 88), np.float32), rest["note"]]),
             "onset": np.concatenate([rest["onset"][:60], rest["onset"]]),
             "contour": np.concatenate([rest["contour"][:60], rest["contour"]])}
    for q in (postsets.params(min_note_len=0), postsets.params(melodia_trick=False, min_note_len=0)):
        p = prm(q)
        ref = Oracle(const, p)
        count(ref)
        fd = stream_ref.frame_diff(const["note"], [0])
        seg_ends = [e for a, b, s, e, r in ref.plan]
        assert len(seg_ends) > 3 and fd[: seg_ends[0]].max() == 0 and fd[: seg_ends[1]].max() > 0
        for key, ends in schedules(ref.n, ref.confirming()).items():
            check(model, const, p, ends, ref, f"constant start {key}")
    # 0-frame stream and 0-frame pushes
    p = prm(postsets.params(min_note_len=0))
    empty = {k: v[:0] for k, v in base.items()}
    assert check(model, empty, p, [], Oracle(empty, p)) == []
    assert check(model, empty, p, [0, 0], Oracle(empty, p)) == []
    ref = Oracle(base, p)
    conf = ref.confirming()
    ends = sorted([0, 0, ref.n, ref.n] + [t + 1 for t in conf] * 2 + [t for t in conf])
    check(model, base, p, ends, ref, "0-frame pushes")


# ------------------------------------------------------------------------------------------------ 6: slot retry
def test_slot_allowance_retry(model):
    """A carved crowded file whose segments yield more notes than the first allowance of 8 T + 64 slots: the device
    decodes them again at full capacity and must still equal the oracle."""
    files, grid = postsets.get("crowded")
    retried = 0
    for j, q in enumerate(grid):
        out = streamsets.carved(files[1], q, 40 + j)
        p = prm(q)
        ref = Oracle(out, p)
        count(ref)
        over = [ref.decoded[k] - (8 * (e - s) + 64) for k, (a, b, s, e, r) in enumerate(ref.plan) if e > s]
        retried += sum(x > 0 for x in over)
        for key in ("one", "7-8-9", "to t", "whole"):
            check(model, out, p, schedules(ref.n, ref.confirming())[key], ref, f"crowded {j} {key}")
    assert retried >= 3, retried
    report("slot retry")


# ------------------------------------------------------------------------------------------------ 7: interleaving
def test_two_streams_and_other_entry_points_on_one_model(model):
    """Two streams with different settings pushed alternately on one model, with decode_arrays, decode_grid, evaluate and
    transcribe_arrays called between pushes (they reuse the decode workspaces the streams decode in): each stream must
    give what it gives alone, push by push, with the launches of its own rule."""
    from basic_pitch_b200 import synth
    from basic_pitch_b200.inference import NoteStream

    files, grid = postsets.get("ties")
    a_out = streamsets.carved(tuple(x[:2000] for x in files[0]), grid[1], 3)
    a_p = prm(grid[1])
    b_out = streamsets.gapped(21, streamsets.gap_lengths(4) * 4)
    b_p = prm(postsets.params(onset_thresh=0.3, min_note_len=1, energy_tol=4, lo_col=10, hi_col=80), bends=True)
    refs = [Oracle(a_out, a_p), Oracle(b_out, b_p)]
    ends = [schedules(refs[0].n, refs[0].confirming())["255-256-257-31"], schedules(refs[1].n, refs[1].confirming())["to t"]]
    alone = [run(model, a_out, a_p, ends[0]), run(model, b_out, b_p, ends[1])]
    clip = synth.tones_clip(1.0, seed=4)
    other = streamsets.gapped(22, [30, 5, 40])
    nrefs = [(np.array([[0.1, 0.5]]), np.array([440.0]))]

    def disturb(k):
        g = ([other["note"]], [other["onset"]], [other["contour"]])
        [lambda: model.decode_arrays(*g, 0.3, 0.2, 0, 3),
         lambda: model.decode_grid(*g, [dict(energy_tol=2), dict(min_note_len=0, infer_onsets=False)]),
         lambda: model.evaluate(["notes"], [dict()], grams=g, note_refs=nrefs),
         lambda: model.transcribe_arrays([clip])][k % 4]()

    streams = []
    for out, p in ((a_out, a_p), (b_out, b_p)):
        params = model._params(p["onset_thresh"], p["frame_thresh"], p["min_note_len"], p["energy_tol"],
                               p["infer_onsets"], p["melodia_trick"], p["bends"], p["lo"], p["hi"])  # fmt: skip
        streams.append(NoteStream(model, params))
    got = [([], [], []), ([], [], [])]
    pos, k = [0, 0], 0
    while pos[0] < len(ends[0]) or pos[1] < len(ends[1]):
        for i, (out, p) in enumerate(((a_out, a_p), (b_out, b_p))):
            j = pos[i]
            if j == len(ends[i]):
                continue
            t, u = (ends[i][j - 1] if j else 0), ends[i][j]
            l0 = model.launch_count
            ev = streams[i].push(out["note"][t:u], out["onset"][t:u], out["contour"][t:u])
            got[i][2].append(model.launch_count - l0)
            got[i][0].append(list(map(ev_key, ev)))
            got[i][1].append(streams[i].held_frames)
            pos[i] += 1
            disturb(k)
            k += 1
    for i in range(2):
        l0 = model.launch_count
        got[i][0].append(list(map(ev_key, streams[i].end())))
        got[i][2].append(model.launch_count - l0)
        assert got[i][0] == alone[i][0] and got[i][1] == alone[i][1] and got[i][2] == alone[i][2], i
        assert got[i][2] == refs[i].launches(ends[i]), i
        assert sum(len(g) for g in got[i][0]) > 0
    assert k >= 8


# ------------------------------------------------------------------------------------------------ 8: capacity
def test_take_capacity(model):
    """bp_stream_take with exactly the capacity needed, one note short, one pitch-bend value short: a failed take leaves
    the queue as it was, and later pushes append to it."""
    from basic_pitch_b200 import _lib
    from basic_pitch_b200.inference import Model

    lib = model._lib
    out = streamsets.gapped(31, streamsets.gap_lengths(11) * 2)
    p = prm(postsets.params(min_note_len=0))
    ref = Oracle(out, p)
    s = model.note_stream(0.5, 0.3, 0)
    ptr = lambda a: np.ascontiguousarray(a).ctypes.data  # noqa: E731
    half = ref.confirming()[len(ref.conf) // 2] + 1
    exp = [e for ks in ref.keys for e in ks]

    def push(t, u):
        lib.bp_stream_push_host(s._h, ptr(out["note"][t:u]), ptr(out["onset"][t:u]), ptr(out["contour"][t:u]), u - t)

    def take(n_cap, b_cap):
        notes, arrs = Model._alloc_notes(1, n_cap, b_cap)
        lib.bp_stream_take(s._h, C.byref(notes))
        return arrs

    def need():
        n, b = C.c_int64(0), C.c_int64(0)
        lib.bp_last_required(C.byref(n), C.byref(b))
        return n.value, b.value

    def fails(n_cap, b_cap):
        with pytest.raises(_lib.BpError) as e:
            take(n_cap, b_cap)
        assert e.value.code == _lib.BP_E_CAPACITY
        return need()

    push(0, half)
    first = [ks for ks, j in zip(ref.keys, stream_ref.push_schedule(ref.plan, 11, [half])[0]) if j == 0]
    n_notes, n_bends = sum(map(len, first)), sum(len(k[4]) for ks in first for k in ks)
    assert n_notes > 2 and n_bends > 0
    assert fails(n_notes - 1, n_bends + 100) == (n_notes, 0)
    assert fails(n_notes, n_bends - 1) == (0, n_bends)
    push(half, ref.n)
    lib.bp_stream_end(s._h)
    total_b = sum(len(k[4]) for k in exp)
    assert fails(len(exp), total_b - 1) == (0, total_b)
    arrs = take(len(exp), total_b)  # exactly the need
    from basic_pitch_b200.note_creation import frame_index_to_time

    assert arrs["note_off"][1] == len(exp) and arrs["bend_off"][len(exp)] == total_b
    got = [(float(frame_index_to_time(np.int64(a))), float(frame_index_to_time(np.int64(b))), int(pi),
            int(np.float32(am).view(np.int32)), tuple(int(v) for v in arrs["bends"][arrs["bend_off"][j]:arrs["bend_off"][j + 1]]))
           for j, (a, b, pi, am) in enumerate(zip(arrs["start"], arrs["end"], arrs["pitch"], arrs["amp"]))]  # fmt: skip
    assert got == exp
    assert take(0, 0)["note_off"][1] == 0  # the queue is empty now


# ------------------------------------------------------------------------------------------------ 9: end to end
def test_predict_stream_notes_settings(model):
    """predict_stream_notes with a frequency range, a non-default minimum note length, melodia off and a small
    max_segment_seconds; with one window per step and blocks smaller than a window; a recording shorter than a window;
    no blocks at all.  The events of every step equal the oracle's on the concatenated parts."""
    from basic_pitch_b200 import synth
    from basic_pitch_b200.inference import DEFAULT_MINIMUM_NOTE_LENGTH_MS, predict_stream_notes
    from basic_pitch_b200.note_creation import frequency_to_column_range

    def go(audio, block, wps, **kw):
        blocks = (audio[i : i + block] for i in range(0, len(audio), block))
        steps = list(predict_stream_notes(blocks, model, windows_per_step=wps, **kw))
        assert steps[-1][0]["note"].shape[0] == 0
        out = {k: np.concatenate([part[k] for part, _ in steps]) for k in ("note", "onset", "contour")}
        lo, hi = frequency_to_column_range(kw.get("minimum_frequency"), kw.get("maximum_frequency"))
        mnl = int(np.round(kw.get("minimum_note_length", DEFAULT_MINIMUM_NOTE_LENGTH_MS) / 1000 * (22050 / 256)))
        mss = kw.get("max_segment_seconds")
        p = dict(onset_thresh=kw.get("onset_threshold", 0.5), frame_thresh=kw.get("frame_threshold", 0.3),
                 min_note_len=mnl, energy_tol=11, infer_onsets=True, melodia_trick=kw.get("melodia_trick", True),
                 bends=True, lo=lo, hi=hi)
        ref = Oracle(out, p, 0 if mss is None else max(1, int(np.round(mss * 22050 / 256))))
        ends = list(np.cumsum([part["note"].shape[0] for part, _ in steps[:-1]]))
        closed_by, _ = stream_ref.push_schedule(ref.plan, 11, ends)
        exp = [[] for _ in steps]
        for k, keys in enumerate(ref.keys):
            exp[closed_by[k]] += keys
        assert [list(map(ev_key, ev)) for _, ev in steps] == exp
        return ref, steps

    audio = synth.melody_clip(40.0, seed=5)
    ref, _ = go(audio, 30011, 4, minimum_frequency=150.0, maximum_frequency=900.0, minimum_note_length=60.0,
                melodia_trick=False, max_segment_seconds=0.5)
    assert sum(f for _, f in ref.conf) > 0 and sum(len(k) for k in ref.keys) > 0
    ref, steps = go(audio[: 22050 * 8], 20000, 1)
    assert len(steps) > 4 and sum(len(k) for k in ref.keys) > 0
    ref, steps = go(synth.tones_clip(1.0, seed=2), 5000, 1)  # shorter than one window
    assert ref.n > 0
    steps = list(predict_stream_notes(iter(()), model))
    assert len(steps) == 1 and steps[0][0]["note"].shape[0] == 0 and steps[0][1] == []
