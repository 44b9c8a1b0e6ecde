"""GPU: the front end stage by stage (bp_debug_frontend), under the four weight sets, on path 0 (decimate_kernel /
decimate_tail_kernel, cqt_kernel, lognorm_kernel) and path 1 (the same chain, cqt_tc_kernel, lognorm_split_kernel):

  * every decimation stage x_{s+1} against float64 from the kernel's own x_s, every octave's log-magnitudes against
    float64 from the kernel's own x_o, with the per-stage bounds of tests/error_bounds.py (the largest err/bound per
    stage, octave, path and set is printed; <= 1 passes);
  * the chain bit-identical on every path, path 2's front-end buffers path 1's bits;
  * the per-window min / max exactly the min / max of the raw log-magnitudes, and the normalised y and both planes of
    the split operand bit-exact to a float32 restatement, including every padding row and bin;
  * window boundaries at every position of the CQT's 128-frame M-tiles, batches of 1, a ragged last M-tile and a full
    chunk; the on-device window views (WinDesc zero fill) of run_inference_arrays;
  * a negative control: the same check scores the GPU's output against a faulted reference and must fail."""
import gc

import numpy as np
import pytest

from tests import error_bounds as eb
from tests import weightsets
from tests.test_frontend_bounds import octave_with_fault
from tests.test_gpu_parity import _edge_windows
from tests.test_gpu_weightsets import _extra_windows, blob_paths, models  # noqa: F401  (module fixtures)

pytestmark = pytest.mark.gpu

N = 43844
HOP = 36164
f32 = np.float32


def _contrast_windows():
    """loudness contrast inside one batch: full-scale noise, 1e-4 noise, silence, and one window loud in its first half
    and 1e-5 in its second"""
    rng = np.random.default_rng(23)
    out = np.zeros((4, N), f32)
    out[0] = rng.uniform(-1, 1, N)
    out[1] = 1e-4 * rng.uniform(-1, 1, N)
    out[3] = rng.uniform(-1, 1, N) * np.where(np.arange(N) < N // 2, 1.0, 1e-5)
    return out


@pytest.fixture(scope="module")
def windows():
    return np.concatenate([_edge_windows(), _extra_windows(), _contrast_windows()]).astype(f32)


def read_frontend(model, n, path):
    """chain, raw log-magnitudes, min / max, (split operand and its layout on paths 1 / 2), normalised y of the last
    forward call"""
    lib, h = model._lib, model.handle
    _, _, stride = eb.chain_layout()
    fe = {"chain": np.empty((n, stride), f32), "log": np.empty((n, 172, 309), f32), "minmax": np.empty((n, 2), f32)}
    for which, key in enumerate(("chain", "log", "minmax")):
        lib.bp_debug_frontend(h, which, fe[key].ctypes.data, n)
    if path >= 1:
        lay = np.zeros(5, np.int32)
        lib.bp_debug_split_layout(h, lay.ctypes.data)
        fe["layout"] = lay
        fe["yhl"] = np.empty((2, lay[4], lay[0], 8), np.uint16)
        lib.bp_debug_frontend(h, 3, fe["yhl"].ctypes.data, n)
    fe["y"] = np.empty((n, 172, 309), f32)  # after the raw read: on paths 1 / 2 this normalises `y` in place
    lib.bp_debug_activation(h, 0, fe["y"].ctypes.data, n)
    return fe


def run(model, x, path):
    model.set_path(path)
    model._lib.bp_model_set_debug_frontend(model.handle, 1)
    try:
        model.predict(x)
        return read_frontend(model, len(x), path)
    finally:
        model._lib.bp_model_set_debug_frontend(model.handle, 0)
        model.set_path(1)


def signals(fe, x):
    """x_0 (the windows) .. x_8 as the kernels read them"""
    off, ln, _ = eb.chain_layout()
    return [np.asarray(x, f32)] + [fe["chain"][:, off[o] : off[o] + ln[o]] for o in range(1, 9)]


def check_exact(fe, w, label):
    """min / max, normalised y and the split operand: exact"""
    log = fe["log"]
    mm = np.stack([log.min(axis=(1, 2)), log.max(axis=(1, 2))], 1)
    bad = np.nonzero((fe["minmax"] != mm).any(axis=1))[0]
    assert not len(bad), f"{label}: min / max of windows {bad.tolist()}: {fe['minmax'][bad]} != {mm[bad]}"
    y = eb.lognorm_f32(log, fe["minmax"], w)
    np.testing.assert_array_equal(fe["y"].view(np.uint32), y.view(np.uint32), err_msg=f"{label}: normalised y")
    if "yhl" in fe:
        rows_stride, rows_used, lead, rpw, chunks8 = (int(v) for v in fe["layout"])
        assert rows_used <= rows_stride and fe["yhl"].shape[1] == chunks8
        exp = eb.split_operand(y, rows_used, lead, rpw, chunks8)
        got = fe["yhl"][:, :, :rows_used]
        if not np.array_equal(got, exp):
            pl, c8, row, j = np.argwhere(got != exp)[0]
            pytest.fail(f"{label}: split operand differs first at plane {pl}, chunk {c8}, row {row}, bin {8 * c8 + j} "
                        f"({np.count_nonzero(got != exp)} elements)")


def stage_ratios(fe, x, w, path):
    """largest err/bound of every decimation stage and every octave, from the kernel's own inputs"""
    xs = signals(fe, x)
    r = {f"dec{s}": eb.ratio(xs[s + 1], *eb.decimate_stage(xs[s], w["lowpass"])) for s in range(8)}
    for o in range(9):
        ref, bound, g = eb.cqt_octave(xs[o], w, o, path)
        r[f"oct{o}"] = eb.ratio(fe["log"][..., g], ref, bound)
    return r


def check_bounds(fe, x, w, path, label):
    r = stage_ratios(fe, x, w, path)
    print(f"{label}: max err/bound " + " ".join(f"{k}={v:.2e}" for k, v in r.items()))
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, (label, bad)


def split_distances(fe, x, w):
    """per octave, how much closer the tensor-core path's log-magnitudes lie to the three-way split than to a two-way
    split, summed over the octave (error_bounds.split_distance): both producer paths of cqt_tc_kernel (octaves 0..2
    split per row, octaves >= 3 split a staged segment) must keep all three planes of A"""
    xs = signals(fe, x)
    d = {}
    for o in range(9):
        ref3, _, g = eb.cqt_octave(xs[o], w, o, 1)
        ref2, _, _ = eb.cqt_octave(xs[o], w, o, 1, proj=octave_with_fault(xs[o], w, o, ("split2", o, None)))
        d[o] = eb.split_distance(fe["log"][..., g], ref3, ref2)
    return d


def assert_same_bits(a, b, keys, label):
    for k in keys:
        np.testing.assert_array_equal(a[k].view(np.uint8), b[k].view(np.uint8), err_msg=f"{label}: {k}")


@pytest.mark.parametrize("wset", weightsets.NAMES)
def test_frontend_stage_by_stage(models, windows, wset):
    model, w = models[wset], weightsets.get(wset)
    fe = {}
    for path in (0, 1, 2):
        fe[path] = run(model, windows, path)
        check_exact(fe[path], w, f"{wset} path {path}")
    for path in (0, 1):
        check_bounds(fe[path], windows, w, path, f"{wset} path {path}")
    d = split_distances(fe[1], windows, w)
    print(f"{wset} path 1: sum |err| two-way / three-way split " + " ".join(f"oct{o}={v:.3g}" for o, v in d.items()))
    assert min(d.values()) > 1.5, (wset, d)
    assert_same_bits(fe[0], fe[1], ("chain",), f"{wset}: path 0 vs path 1")
    assert_same_bits(fe[2], fe[1], ("chain", "log", "minmax", "yhl", "y"), f"{wset}: path 2 vs path 1")


def _boundary_batch(n):
    """windows alternating silence, 1e-4-amplitude noise and full-scale noise"""
    rng = np.random.default_rng(7)
    x = np.zeros((n, N), f32)
    for b in range(n):
        if b % 3 == 1:
            x[b] = 1e-4 * rng.uniform(-1, 1, N)
        elif b % 3 == 2:
            x[b] = rng.uniform(-1, 1, N)
    return x


def test_window_boundaries_inside_the_cqt_mtiles(models):
    """Window b starts at frame 172 b, and 172 b mod 128 takes 32 values: 33 windows put a window boundary at every
    position a warp of cqt_tc_kernel's epilogue can straddle (uniform and split branch of the min / max atomics).  Also
    n = 1, a ragged last M-tile (n = 3) and a full chunk, whose windows must carry the bits of the checked 33-window
    batch (batch-size independence)."""
    model, w = models["dense"], weightsets.get("dense")
    assert sorted({172 * b % 128 for b in range(33)}) == list(range(0, 128, 4))
    x = _boundary_batch(33)
    for path in (0, 1):
        ref = run(model, x, path)
        check_exact(ref, w, f"33 windows, path {path}")
        check_bounds(ref, x, w, path, f"dense path {path} (33 windows)")
    chunk = int(model._lib.bp_model_chunk_windows(model.handle))
    for n in (1, 3, chunk):
        xn = np.ascontiguousarray(np.tile(x[:3], (-(-n // 3), 1))[:n])
        fe = run(model, xn, 1)
        check_exact(fe, w, f"{n} windows, path 1")
        for b in range(n):
            for k in ("log", "minmax"):
                np.testing.assert_array_equal(fe[k][b], ref[k][b % 3], err_msg=f"batch of {n}, window {b}: {k}")
            np.testing.assert_array_equal(fe["chain"][b], ref["chain"][b % 3], err_msg=f"batch of {n}, window {b}")
    if chunk == 184:  # H100 SXM
        print("full chunk of 184 windows checked")


def test_window_views_of_run_inference(models):
    """On-device windowing (WinDesc lo / hi zero fill in decimation stage 0 and in the reflect-padded octave-0 gather of
    both CQT kernels): the chain and the raw log-magnitudes of run_inference_arrays on one clip equal those of predict()
    on the host's windows of that clip, bit for bit."""
    from basic_pitch_b200 import synth
    from oracle import host_ref

    model = models["dense"]
    long = synth.random_notes_clip(N / 22050.0 + 0.1, seed=57)[:N]
    lib, h = model._lib, model.handle
    for path in (1, 0):
        model.set_path(path)
        lib.bp_model_set_debug_frontend(h, 1)
        try:
            for n in (1, HOP - 1, HOP + 1, N):
                clip = long[:n]
                win = host_ref.window_audio(clip)
                if win.ndim == 3:
                    win = win[..., 0]
                nw = len(win)
                model.run_inference_arrays([clip])
                _, _, stride = eb.chain_layout()
                got = {"chain": np.empty((nw, stride), f32), "log": np.empty((nw, 172, 309), f32)}
                lib.bp_debug_frontend(h, 0, got["chain"].ctypes.data, nw)
                lib.bp_debug_frontend(h, 1, got["log"].ctypes.data, nw)
                model.predict(np.ascontiguousarray(win, f32))
                exp = {"chain": np.empty_like(got["chain"]), "log": np.empty_like(got["log"])}
                lib.bp_debug_frontend(h, 0, exp["chain"].ctypes.data, nw)
                lib.bp_debug_frontend(h, 1, exp["log"].ctypes.data, nw)
                assert_same_bits(got, exp, ("chain", "log"), f"path {path}, clip of {n} samples ({nw} windows)")
        finally:
            lib.bp_model_set_debug_frontend(h, 0)
            model.set_path(1)


def test_negative_control_on_gpu_data(models, windows):
    """The per-stage check has teeth on real GPU data: scored against a reference whose stage 7 drops low-pass tap 255,
    the GPU's own x_8 fails it.  A two-way instead of the three-way split of octave 8 stays inside the worst-case bound
    (the 2 K u accumulation term of the truncating MMA is as large as the two-way split's error), so there the GPU's
    log-magnitudes must instead lie closer, summed over the octave, to the three-way reference than to the two-way
    one by at least half again (a kernel that lost a plane lies closer to the two-way one: ratio < 1) (error_bounds.split_distance)."""
    model, w = models["dense"], weightsets.get("dense")
    fe = run(model, windows, 1)
    xs = signals(fe, windows)
    h = np.asarray(w["lowpass"], np.float64).copy()
    h[255] = 0.0
    ref, _ = eb.decimate_stage(xs[7], h)
    _, bound = eb.decimate_stage(xs[7], w["lowpass"])
    r_dec = eb.ratio(xs[8], ref, bound)
    ref3, bound, g = eb.cqt_octave(xs[8], w, 8, 1)
    ref2, _, _ = eb.cqt_octave(xs[8], w, 8, 1, proj=octave_with_fault(xs[8], w, 8, ("split2", 8, None)))
    got = fe["log"][..., g]
    r2, r3 = eb.ratio(got, ref2, bound), eb.ratio(got, ref3, bound)
    d = eb.split_distance(got, ref3, ref2)
    print(f"GPU output against faulted references: stage 7 without tap 255 {r_dec:.3g}; octave 8 err/bound three-way "
          f"{r3:.3g}, two-way {r2:.3g}; sum |err| two-way / three-way {d:.3g}")
    assert r_dec > 1.0 and r3 <= 1.0 and d > 1.5, (r_dec, r3, d)


def test_frontend_debug_switch_off_keeps_the_launch_sequence(blob_paths, windows):
    """bp_model_set_debug_frontend off: the forward launches exactly what it launched before the switch existed; on: the
    same launches (a device copy only).  The raw log-magnitudes of path 0 are only available with the switch on."""
    from basic_pitch_b200 import _lib
    from basic_pitch_b200.inference import Model

    model = Model(blob_paths["trained"])
    try:
        x = windows[:4]
        counts = {}
        for path in (0, 1):
            model.set_path(path)
            for on in (0, 1):
                model._lib.bp_model_set_debug_frontend(model.handle, on)
                c0 = model.launch_count
                model.predict(x)
                counts[(path, on)] = model.launch_count - c0
            model._lib.bp_model_set_debug_frontend(model.handle, 0)
        assert counts[(0, 0)] == counts[(0, 1)] and counts[(1, 0)] == counts[(1, 1)], counts
        model.set_path(0)
        model.predict(x)
        buf = np.empty((4, 172, 309), f32)
        with pytest.raises(_lib.BpError):
            model._lib.bp_debug_frontend(model.handle, 1, buf.ctypes.data, 4)
        with pytest.raises(_lib.BpError):  # no split operand on path 0
            model._lib.bp_debug_frontend(model.handle, 3, buf.ctypes.data, 4)
    finally:
        del model
        gc.collect()
