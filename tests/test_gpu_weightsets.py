"""GPU: the forward kernels (decimation chain, CQT projection, the three fused tensor-core convolutions, edge_fix_kernel)
under the synthetic parameter sets of tests/weightsets.py, against the float64 oracle with the per-element bounds of
tests/error_bounds.py, on every forward path and every work split of the convolutions; and several models with
different weights in one process.

Each comparison prints its largest err/bound ratio (<= 1 passes)."""
import gc

import numpy as np
import pytest

from tests import error_bounds as eb
from tests import weightsets
from tests.test_gpu_parity import _edge_windows

pytestmark = pytest.mark.gpu

N = 43844
HOP = 36164
POSTS = ("note", "onset", "contour")


def _extra_windows():
    """clicks at the first, a mid-frame and the last sample; a +-1 square wave at the Nyquist rate (the stop band of
    every decimation stage); a DC offset; a chirp over the full band"""
    out = np.zeros((6, N), np.float32)
    for i, s in enumerate((0, 127, N - 1)):
        out[i, s] = 1.0
    out[3] = np.where(np.arange(N) % 2 == 0, 1.0, -1.0)
    out[4] = 0.5
    t = np.arange(N) / 22050.0
    f0, f1, dur = 20.0, 11000.0, N / 22050.0
    out[5] = 0.8 * np.sin(2 * np.pi * (f0 * t + (f1 - f0) * t * t / (2 * dur)))
    return out


@pytest.fixture(scope="module")
def windows():
    return np.concatenate([_edge_windows(), _extra_windows()])


@pytest.fixture(scope="module")
def blob_paths(tmp_path_factory):
    d = tmp_path_factory.mktemp("weightsets")
    paths = {}
    for name in weightsets.NAMES:
        paths[name] = d / f"{name}.bpw"
        paths[name].write_bytes(weightsets.blob(name))
    return paths


@pytest.fixture(scope="module")
def models(blob_paths):
    from basic_pitch_b200.inference import Model

    ms = {name: Model(p) for name, p in blob_paths.items()}
    yield ms
    ms.clear()
    gc.collect()


_E2E = {}


def _e2e(x_key, x, wset, eps):
    """end-to-end bounds (from the audio) are the same for every model of a set: computed once"""
    k = (x_key, wset, eps)
    if k not in _E2E:
        _E2E[k] = eb.forward_bounds(x, weightsets.get(wset), eps, eps)
    return _E2E[k]


def _activation(model, which, shape):
    buf = np.empty(shape, np.float32)
    model._lib.bp_debug_activation(model.handle, which, buf.ctypes.data, shape[0])
    return buf


def _check_forward(model, wset, x, path, x_key, label=""):
    """predict() on `path`, every activation the path exposes and the three posteriorgrams against the oracle"""
    n = x.shape[0]
    eps = 0.0 if path == 0 else eb.EPS_SPLIT
    model.set_path(path)
    try:
        out = model.predict(x)
        y = _activation(model, 0, (n, 172, 309))
        acts = {"_y": y}
        if path in (0, 2):
            acts["_c1"] = _activation(model, 1, (n, 8, 172, 264))
        if path == 0:
            acts["_n1"] = _activation(model, 2, (n, 32, 172, 88))
            acts["_o1"] = _activation(model, 3, (n, 32, 172, 88))
    finally:
        model.set_path(1)
    w = weightsets.get(wset)
    e2e = _e2e(x_key, x, wset, eps)
    local = eb.forward_bounds(x, w, eps, eps, y_in=y, contour_in=out["contour"], note_in=out["note"])
    r = {"_y": eb.ratio(y, e2e["_y"], e2e["b_y"])}
    for k, v in acts.items():
        if k != "_y":
            r[k] = eb.ratio(v, local[k], local["b" + k])
    for k in POSTS:
        r[k] = eb.logit_check(out[k], local["l_" + k], local["b_" + k])
        r[k + "(e2e)"] = eb.logit_check(out[k], e2e["l_" + k], e2e["b_" + k])
    print(f"{wset} path {path}{label}: max err/bound " + " ".join(f"{k}={v:.2e}" for k, v in r.items()))
    bad = {k: v for k, v in r.items() if not v <= 1.0}
    assert not bad, (wset, path, bad)
    return out


@pytest.mark.parametrize("path", [1, 2, 0])
@pytest.mark.parametrize("wset", weightsets.NAMES)
def test_forward_paths_vs_float64_oracle(models, windows, wset, path):
    _check_forward(models[wset], wset, windows, path, "windows")


# ---------------------------------------------------------------------------------------------------------------------
# work splits of the tensor-core convolutions
# ---------------------------------------------------------------------------------------------------------------------
# (rows per window, M-tile rows that finish frames, frequency groups) of each launch_conv_tc call: 64-row M-tiles
# overlap by KH2 - 1 rows when the next conv is fused (tc_contour_spec / tc_onset_spec / tc_note_spec, tc_conv.cu)
LAYERS = {
    "contour (fused, path 1)": (174, 64 - 4, 9),
    "contour (path 2)": (174, 64, 9),
    "onset": (174, 64 - 2, 12),
    "note": (175, 64 - 6, 12),
}


def n_split(n_windows, rows_per_window, ms, n_groups, n_sms):
    """launch_conv_tc's choice of the number of frequency-group runs per M-tile (tc_conv.cu:1052-1062)"""
    n_mtiles = -(-n_windows * rows_per_window // ms)
    best, split = 1e30, 1
    for s in range(1, n_groups + 1):
        waves = -(-n_mtiles * s // n_sms)
        cost = waves * (-(-n_groups // s) + 0.5)
        if cost < best - 1e-9:
            best, split = cost, s
    return split


def _sweep_sizes(chunk, n_sms):
    """batch sizes (<= one chunk) that reach every split class of every layer, greedy; and the classes per layer"""
    classes = {k: {} for k in LAYERS}
    for n in range(1, chunk + 1):
        for k, (rpw, ms, ng) in LAYERS.items():
            classes[k].setdefault(n_split(n, rpw, ms, ng, n_sms), []).append(n)
    need = {(k, c) for k in LAYERS for c in classes[k]}
    sizes = []
    while need:
        best = max(range(1, chunk + 1), key=lambda n: (sum((k, c) in need for k in LAYERS for c in classes[k] if n in classes[k][c]), -n))
        sizes.append(best)
        need -= {(k, c) for k in LAYERS for c in classes[k] if best in classes[k][c]}
    return sorted(sizes), {k: sorted(v) for k, v in classes.items()}


@pytest.mark.parametrize("wset", ["trained", "dense"])
def test_every_work_split_gives_bit_identical_windows(models, windows, wset):
    """The kernels document that a frame's value does not depend on the batch around it.  Batch sizes are chosen so
    that every split class of every layer (the tile-range boundaries edge_fix_kernel finishes move with it) is reached
    on this device; three distinct windows tiled to each size must give bit-identical posteriorgrams at every size and
    position, and match the oracle once."""
    import torch

    model = models[wset]
    n_sms = torch.cuda.get_device_properties(model.device).multi_processor_count
    chunk = int(model._lib.bp_model_chunk_windows(model.handle))
    sizes, classes = _sweep_sizes(chunk, n_sms)
    reached = {k: sorted({n_split(n, *LAYERS[k], n_sms) for n in sizes}) for k in LAYERS}
    print(f"{n_sms} SMs, chunk {chunk}: batch sizes {sizes}; split classes {reached}")
    assert reached == classes
    if n_sms == 132 and chunk == 184:  # H100 SXM
        assert classes["contour (fused, path 1)"] == classes["contour (path 2)"] == [1, 2, 3, 5, 9]
        assert classes["onset"] == classes["note"] == [1, 2, 3, 4, 6, 12]
    base = windows[[0, 1, 8]]  # two music windows and the click at sample 20 000
    for path in (1, 2):
        ref = _check_forward(model, wset, base, path, "sweep", label=" (3 distinct windows)")
        model.set_path(path)
        try:
            for n in sizes:
                x = np.ascontiguousarray(np.tile(np.roll(base, n % 3, axis=0), (-(-n // 3), 1))[:n])
                got = model.predict(x)
                for i in range(n):
                    j = (i - n % 3) % 3
                    for k in POSTS:
                        if not np.array_equal(got[k][i], ref[k][j]):
                            d = float(np.abs(got[k][i] - ref[k][j]).max())
                            pytest.fail(f"{wset} path {path}: batch of {n}, window {i} (= distinct window {j}): {k} differs by {d:.3e}")
        finally:
            model.set_path(1)


def test_run_inference_arrays_under_dense_weights(models):
    """On-device windowing (WinDesc zero fill) and unwrap at the window-boundary clip lengths, under weights whose every
    tap counts: bit-identical to host windowing + predict() + unwrap, and predict() within the bounds of the oracle."""
    from basic_pitch_b200 import synth
    from oracle import host_ref

    model = models["dense"]
    long = synth.random_notes_clip((3 * HOP + 1) / 22050.0 + 0.1, seed=57)[: 3 * HOP + 1]
    clips = [long[:n] for n in (1, HOP - 1, HOP, HOP + 1, N, 3 * HOP + 1)]
    wins = [host_ref.window_audio(c) for c in clips]
    x = np.concatenate(wins)
    raw = _check_forward(model, "dense", x, 1, "clips", label=" (windows of the clips)")
    outs = model.run_inference_arrays(clips)
    i0 = 0
    for clip, win, out in zip(clips, wins, outs):
        for k in POSTS:
            exp = host_ref.unwrap(raw[k][i0 : i0 + len(win)], len(clip))
            assert out[k].shape == exp.shape, (len(clip), k)
            np.testing.assert_array_equal(out[k], exp, err_msg=f"{k}, clip of {len(clip)} samples")
        i0 += len(win)


# ---------------------------------------------------------------------------------------------------------------------
# several models in one process
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [("sparse", "trained", "dense"), ("dense", "trained", "sparse")])
def test_models_with_different_weights_in_one_process(blob_paths, windows, order):
    """The MMA programs live in __constant__ memory shared by every model of the process; the weight-dependent values
    are kernel parameters of each model's launches.  Models created in either order, called interleaved, must each
    compute the oracle under their OWN weights, and give the same bits on every call."""
    from basic_pitch_b200.inference import Model

    x = windows[[0, 1, 6, 8, 12]]
    ms = {name: Model(blob_paths[name]) for name in order}
    try:
        first = {name: _check_forward(ms[name], name, x, 1, "multi", label=f" ({'/'.join(order)})") for name in order}
        for name in reversed(order):
            again = ms[name].predict(x)
            for k in POSTS:
                np.testing.assert_array_equal(again[k], first[name][k], err_msg=f"{name} {k}, second call")
    finally:
        ms.clear()
        gc.collect()


def test_models_with_different_weights_run_concurrently(models, windows):
    """bp_forward_device only enqueues on the caller's stream (bp_b200.h).  Model A's call is queued on stream S1 behind
    a ~0.5 s sleep; model B, with other weights, is then called on stream S2 and must return while A's work is still
    pending: no call drains the device for another model.  Both results must be the bits of each model's own serial
    call, which matches the oracle under that model's weights."""
    import torch

    x = windows[[0, 1, 6, 8, 12]]
    n = len(x)
    pair = {"trained": models["trained"], "dense": models["dense"]}
    ref = {name: _check_forward(m, name, x, 1, "concurrent", label=" (serial)") for name, m in pair.items()}
    dev = torch.device("cuda", pair["trained"].device)
    d_x = torch.from_numpy(x).to(dev)
    outs = {name: [torch.empty((n, 172, w), dtype=torch.float32, device=dev) for w in (88, 88, 264)] for name in pair}
    streams = {"trained": torch.cuda.Stream(dev), "dense": torch.cuda.Stream(dev)}

    def forward(name):
        m, o = pair[name], outs[name]
        m._lib.bp_forward_device(m.handle, d_x.data_ptr(), n, o[0].data_ptr(), o[1].data_ptr(), o[2].data_ptr(),
                                 streams[name].cuda_stream)

    for name in pair:  # both workspaces at this batch size: no allocation below
        forward(name)
    torch.cuda.synchronize(dev)
    a_done = torch.cuda.Event()
    with torch.cuda.stream(streams["trained"]):
        torch.cuda._sleep(1_000_000_000)  # SM clock cycles: about 0.5 s
    forward("trained")
    a_done.record(streams["trained"])
    forward("dense")
    a_pending = not a_done.query()
    torch.cuda.synchronize(dev)
    assert a_pending, "model B's bp_forward_device waited for model A's work on another stream"
    for name in pair:
        for k, t in zip(POSTS, outs[name]):
            np.testing.assert_array_equal(t.cpu().numpy(), ref[name][k], err_msg=f"{name} {k}, concurrent call")


def test_refresh_with_other_weights_and_restore(blob_paths, windows):
    """bp_model_refresh re-derives everything from the parameter block: write `sparse` into a trained model's block,
    refresh, compare with the oracle under `sparse`, restore, and get the original bits back."""
    import torch

    from basic_pitch_b200 import engine
    from basic_pitch_b200.inference import Model

    x = windows[[0, 1, 8]]
    model, donor = Model(blob_paths["trained"]), Model(blob_paths["sparse"])
    try:
        before = model.predict(x)
        block = engine.param_block_tensor(model)
        saved = block.clone()
        block.copy_(engine.param_block_tensor(donor))
        torch.cuda.synchronize(model.device)
        del donor
        gc.collect()
        model._lib.bp_model_refresh(model.handle)
        _check_forward(model, "sparse", x, 1, "refresh", label=" (trained model refreshed to sparse)")
        block.copy_(saved)
        torch.cuda.synchronize(model.device)
        model._lib.bp_model_refresh(model.handle)
        after = model.predict(x)
        for k in POSTS:
            np.testing.assert_array_equal(after[k], before[k], err_msg=f"{k} after restoring the trained block")
    finally:
        del model
        gc.collect()
