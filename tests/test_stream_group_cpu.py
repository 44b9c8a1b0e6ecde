"""CPU: NumPy models of the stream group's bookkeeping (bp_stream_group_*, csrc/api.cu; DESIGN.md §4.6).

* windowing and commits: which windows each push runs, from which samples of the stream's tail, and how many frames it
  commits, against what run_inference_stream's slicing gives for the same blocks;
* rounds: which segments each decode round takes when one push closes several segments of several streams, against
  oracle/stream_ref.plan and push_schedule."""
import numpy as np
import pytest

from oracle import stream_ref
from tests import streamsets

HOP, WIN, LEAD, PER_WINDOW = 36164, 43844, 3840, 142


def num_frames(n):
    return int(n / HOP * PER_WINDOW) if n > 0 else 0


class GroupAudioModel:
    """One stream of the group: the tail it keeps, the windows it runs and the frames it commits."""

    def __init__(self):
        self.samples, self.win_done, self.tail0, self.n = 0, 0, 0, 0
        self.tail = np.zeros(0, np.float32)

    def windows(self, ending):
        if ending:
            return -(-(self.samples + LEAD) // HOP) if self.samples > 0 else 0
        return (self.samples + LEAD - WIN) // HOP + 1 if self.samples + LEAD >= WIN else 0

    def push(self, block, ending=False):
        """-> (windows run, as arrays of 43 844 samples, frames committed by this call)"""
        self.tail = np.concatenate([self.tail, block])
        self.samples += len(block)
        nw, out = self.windows(ending), []
        for w in range(self.win_done, nw):
            s0 = w * HOP - LEAD
            lo, hi = max(0, -s0), max(max(0, -s0), min(WIN, self.samples - s0))
            win = np.zeros(WIN, np.float32)
            base = s0 - self.tail0  # WinDesc.base relative to the tail
            assert base + lo >= 0 and base + hi <= len(self.tail)
            win[lo:hi] = self.tail[base + lo : base + hi]
            out.append(win)
        self.win_done = max(self.win_done, nw)
        n = num_frames(self.samples) if ending else max(0, (self.win_done - 2) * PER_WINDOW)
        n = max(n, self.n)
        committed, self.n = n - self.n, n
        keep = self.samples if ending else min(self.samples, max(0, self.win_done * HOP - LEAD))
        self.tail, self.tail0 = self.tail[keep - self.tail0 :], keep
        return out, committed


def reference_steps(blocks):
    """run_inference_stream on the blocks with a model that records its windows: per block the windows it ran and the
    frames it yielded, then those of the end."""
    from basic_pitch_b200 import inference as inf

    class Recorder(inf.Model):
        def __init__(self):
            self.wins = []

        def __del__(self):
            pass

        def predict(self, x):
            self.wins += list(np.array(x))
            z = np.zeros((len(x), 172, 88), np.float32)
            return {"note": z, "onset": z, "contour": np.zeros((len(x), 172, 264), np.float32)}

    m, frames, marks = Recorder(), [0], []

    def gen():  # resumed once the stream has yielded every part of the block before
        for b in blocks:
            yield b
            marks.append((len(m.wins), frames[0]))

    for part in inf.run_inference_stream(gen(), m, windows_per_step=5):
        frames[0] += part["note"].shape[0]
    marks.append((len(m.wins), frames[0]))
    steps, w0, f0 = [], 0, 0
    for w, f in marks:
        steps.append((m.wins[w0:w], f - f0))
        w0, f0 = w, f
    return steps


@pytest.mark.parametrize("seed", range(6))
def test_windows_and_commits_follow_run_inference_stream(seed):
    """Random schedules with 0-length blocks, blocks shorter than a hop and blocks of 150 windows."""
    rng = np.random.default_rng(seed)
    n = int(rng.choice([0, 1, 3000, WIN - LEAD - 1, WIN - LEAD, 3 * HOP + 5, 400 * HOP]))
    audio = (np.arange(n) % 1000 + 1).astype(np.float32) * (1 + seed)
    sizes = [0, 1, 100, HOP - 1, HOP, WIN, 150 * HOP] if seed % 2 else [0, 500, 22050]
    blocks, t = [], 0
    while t < n:
        k = int(rng.choice(sizes))
        blocks.append(audio[t : t + k])
        t += k
    steps = reference_steps(blocks)
    g = GroupAudioModel()
    for j, b in enumerate(blocks + [None]):
        wins, c = g.push(np.zeros(0, np.float32), ending=True) if b is None else g.push(b)
        exp_wins, exp_frames = steps[j]
        if b is None and n == 0:  # run_inference_stream also runs the lead-zero window of an empty recording
            exp_wins = []
        assert c == exp_frames, (seed, j)
        assert len(wins) == len(exp_wins) and all(np.array_equal(x, y) for x, y in zip(wins, exp_wins)), (seed, j)
    assert g.n == num_frames(n)


def test_commits_match_the_golden_counts(golden_dir):
    z = np.load(golden_dir / "host_cases.npz")
    for n, nw, nf in zip(z["lens"], z["n_windows"], z["n_frames"]):
        g = GroupAudioModel()
        run = len(g.push(np.ones(int(n), np.float32))[0])
        wins, c = g.push(np.zeros(0, np.float32), ending=True)
        assert run + len(wins) == (int(nw) if n > 0 else 0) and g.n == int(nf), n


def rounds(quiet_of, energy_tol, ends_of, max_seg=0):
    """The group's round loop over streams that push together (ends_of[i]: cumulative frames per push, all of equal
    length; then all end): per push, the list of rounds, each {stream: segment}.  The cut rule is restated from the
    header, frame by frame, as bp_stream's scan finds it."""
    la, w = energy_tol, energy_tol + 3
    after = max(1, energy_tol - 2)
    st = [dict(r=0, a=0, last=-1, scan_from=0, n=0) for _ in quiet_of]

    def begin(s, at):
        return at if at == s["r"] else at - 3

    def first_cut(i):
        s, q, L = st[i], quiet_of[i], st[i]["last"]
        for t in range(s["scan_from"], s["n"]):
            if not q[t]:
                L = t
            elif L is not None and t - L == w:
                return t, L
        return -1, L

    pushes = []
    n_push = len(ends_of[0])
    for j in range(n_push + 1):
        ending = j == n_push
        if not ending:
            for i, s in enumerate(st):
                s["n"] = ends_of[i][j]
        scan, closed, out = list(range(len(st))), set(), []
        while scan:
            batch, again = {}, []
            for i in scan:
                s = st[i]
                t, L = first_cut(i)
                if t >= 0 and (max_seg == 0 or t < s["a"] + max_seg):
                    c = t - la + 1
                    batch[i] = (s["a"], c, begin(s, s["a"]), c + after)
                    s.update(a=c, last=None, scan_from=t + 1)
                    again.append(i)
                elif max_seg > 0 and s["n"] >= s["a"] + max_seg:
                    f = s["a"] + max_seg
                    batch[i] = (s["a"], f, begin(s, s["a"]), f)
                    s.update(r=f, a=f, last=f - 1, scan_from=f)
                    again.append(i)
                else:
                    s.update(last=L, scan_from=s["n"])
                    if ending and i not in closed:
                        closed.add(i)
                        batch[i] = (s["a"], s["n"], begin(s, s["a"]), s["n"])
            if batch:
                out.append(batch)
            scan = again
        pushes.append(out)
    return pushes


@pytest.mark.parametrize("tol,max_seg", [(11, 0), (5, 0), (11, 40), (3, 17)])
def test_rounds_follow_the_plan(tol, max_seg):
    """Streams whose pushes close several segments at once: round k of a push takes the k-th segment each stream closes
    in it, and over the pushes every stream decodes exactly oracle/stream_ref.plan's segments, in order, each in the
    push push_schedule names."""
    cases = []
    for spans, tail in (([30, 40, 25, 60, 35], 40), ([50, 20, 45], 90)):
        n, loud, _, peaks = streamsets.dense_cuts(spans, tol, n_tail=tail)
        cases.append(streamsets.placed(n, loud, peaks))
    cases.append(streamsets.precedence(max(max_seg, 2 * (tol + 3) + 2), tol, 0))
    quiet = [stream_ref.quiet_frames(c["note"], 0.3, 0, 88) for c in cases]
    n_push = 4
    ends = [[int(round(len(q) * (k + 1) / n_push)) for k in range(n_push)] for q in quiet]
    pushes = rounds(quiet, tol, ends, max_seg)
    several = False
    for i, q in enumerate(quiet):
        plan = stream_ref.plan(q, tol, max_seg)
        closed_by, _ = stream_ref.push_schedule(plan, tol, ends[i])
        mine = [(j, seg) for j, rs in enumerate(pushes) for r in rs for sid, seg in r.items() if sid == i]
        exp = [(closed_by[k], (a, b, s, e)) for k, (a, b, s, e, r) in enumerate(plan)]
        assert mine == exp, i
        several |= any(sum(i in r for r in rs) > 1 for rs in pushes)
    assert several
