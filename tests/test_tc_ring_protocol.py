"""CPU: a model of the weight ring of conv_tc_kernel (tc_conv.cu) — one producer, two accumulator slots that skip the
steps they do not use — run on the real MMA programs under random interleavings, with mbarrier parity semantics and
bulk copies that land in any order.  Every full_w wait must see exactly the fill it waits for, every empty_w arrival
must land in the phase of its fill, and nothing may deadlock.  Without the producer's fill counter a slot that skips
more than a ring's worth of steps passes a parity wait on a stale phase; the model must see that too."""
import random

import numpy as np
import pytest

from basic_pitch_b200 import _lib

NOUSE = 0xFFFFFFFF
STAGES = {0: 9, 1: 12, 2: 11}  # tc_smem: contour (fused), onset, note
SHAPES = {0: (8, 8, 3, 39), 1: (32, 8, 5, 5), 2: (32, 1, 7, 7)}


def program(which):
    lib = _lib.load()
    w = np.random.default_rng(0).standard_normal(SHAPES[which]).astype(np.float32)
    sizes = np.zeros(4, np.int32)
    lib.bp_debug_tc_plan(which, w.ctypes.data, sizes.ctypes.data, None, None, None, None, None)
    n_steps, n_groups = int(sizes[1]), int(sizes[3])
    words = np.zeros(2 * n_steps, np.uint32)
    off = np.zeros(n_groups + 1, np.int32)
    lib.bp_debug_tc_plan(which, w.ctypes.data, sizes.ctypes.data, None, None, words.ctypes.data, off.ctypes.data, None)
    return words.reshape(2, n_steps), off, n_groups


class Bar:  # mbarrier: arrival count, completed phases
    def __init__(self, count):
        self.count, self.pending, self.phases = count, count, 0

    def arrive(self, n=1):
        self.pending -= n
        assert self.pending >= 0
        if self.pending == 0:
            self.phases, self.pending = self.phases + 1, self.count

    def passes(self, parity):  # try_wait.parity
        return (self.phases & 1) != parity


def simulate(words, off, items, K, counter, seed):
    rng = random.Random(seed)
    full, empty = [Bar(1) for _ in range(K)], [Bar(8) for _ in range(K)]
    landing, issued = [], [0]

    def producer():
        f = 0
        for g0, g1 in items:
            for s in range(off[g0], off[g1]):
                while not empty[f % K].passes(((f // K) & 1) ^ 1):
                    yield
                assert empty[f % K].phases == f // K and full[f % K].phases == f // K, f
                landing.append(f)
                if words[0][s] == NOUSE or words[1][s] == NOUSE:
                    empty[f % K].arrive(4)  # on behalf of the slot that skips the step
                f += 1
                issued[0] = f
                yield

    def release(f):
        assert empty[f % K].phases == f // K, ("arrival in the wrong phase", f)
        empty[f % K].arrive(4)

    def slot(sl):
        f = 0
        for g0, g1 in items:
            for g in range(g0, g1):
                held = None
                for s in range(off[g], off[g + 1]):
                    if words[sl][s] != NOUSE:
                        if held is not None and f - held >= K:
                            release(held)
                            held = None
                        while counter and issued[0] <= f:
                            yield
                        while not full[f % K].passes((f // K) & 1):
                            yield
                        assert full[f % K].phases == f // K + 1, ("stale phase", sl, f)
                        yield  # the MMAs of fill f are issued; those of the held fill complete
                        if held is not None:
                            release(held)
                        held = f
                    f += 1
                    if rng.random() < 0.3:
                        yield
                if held is not None:
                    release(held)
                for _ in range(rng.randrange(60)):  # epilogue
                    yield

    actors = [producer(), slot(0), slot(1)]
    alive = [True, True, True]
    for _ in range(2_000_000):
        if not any(alive):
            return "ok"
        if landing and rng.random() < 0.4:  # a bulk copy completes, in any order
            f = landing.pop(rng.randrange(len(landing)))
            full[f % K].arrive()
        i = rng.randrange(3)
        if alive[i]:
            try:
                next(actors[i])
            except StopIteration:
                alive[i] = False
            except AssertionError as e:
                return f"fail {e}"
    return "deadlock"


def work(n_groups, rng):  # four items of one CTA under a random work split
    n_split = rng.choice([1, 2, 3, n_groups])
    return [(q * n_groups // n_split, (q + 1) * n_groups // n_split) for q in rng.choices(range(n_split), k=4)]


@pytest.mark.parametrize("which", [0, 1, 2])
def test_ring_protocol_holds(which):
    words, off, n_groups = program(which)
    for seed in range(6):
        res = simulate(words, off, work(n_groups, random.Random(seed)), STAGES[which], True, seed)
        assert res == "ok", (seed, res)


def test_ring_model_sees_the_stale_phase_without_the_fill_counter():
    words, off, n_groups = program(0)
    res = [simulate(words, off, work(n_groups, random.Random(s)), STAGES[0], False, s) for s in range(4)]
    assert any(r.startswith("fail") or r == "deadlock" for r in res), res
