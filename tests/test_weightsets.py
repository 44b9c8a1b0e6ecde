"""CPU: the synthetic parameter sets (tests/weightsets.py) have teeth, and the error bounds (tests/error_bounds.py) are
both valid and tight enough to matter."""
import numpy as np
import pytest

from oracle import model_ref
from tests import error_bounds as eb
from tests import weightsets

STAGES = ("_y", "_c1", "_n1", "_o1")
POSTS = ("note", "onset", "contour")


def _windows():
    from basic_pitch_b200 import synth

    rng = np.random.default_rng(3)
    noise = rng.uniform(-1, 1, (1, 43844)).astype(np.float32)
    return np.concatenate([synth.window_batch(3, seed=2), noise])


@pytest.mark.parametrize("wset", weightsets.NAMES)
def test_weight_set_is_live(wset):
    """A comparison under a set whose posteriorgrams saturate, or whose log-spectrum sits on the 1e-10 power floor,
    proves nothing: at least half of each posteriorgram lies in [0.02, 0.98], and most CQT bins are above the floor."""
    import torch

    o = model_ref.forward(_windows(), weightsets.get(wset), dtype=torch.float64, return_intermediates=True)
    for k in POSTS:
        live = float(((o[k] >= 0.02) & (o[k] <= 0.98)).mean())
        print(f"{wset} {k}: {live:.3f} of the cells in [0.02, 0.98]")
        assert live >= 0.5, (wset, k, live)
    floor = float((o["_mag"] ** 2 < 1e-9).mean())
    assert floor < 0.25, (wset, floor)
    for k in ("_c1", "_n1", "_o1"):  # ReLU layers neither dead nor linear
        active = float((o[k] > 0).mean())
        assert 0.2 < active < 0.9, (wset, k, active)


def test_weight_sets_cover_what_the_trained_weights_leave_out():
    tr, dense, edge, sparse = (weightsets.get(n) for n in ("trained", "dense", "edge_taps", "sparse"))
    k_tr = np.abs(tr["cqt_real"]) + np.abs(tr["cqt_imag"])
    assert not k_tr[:, :21].any() and not k_tr[:, 236:].any()  # the gap these sets close
    for w in (dense, edge, sparse):
        k = np.abs(w["cqt_real"] + 1j * w["cqt_imag"].astype(np.complex64))
        np.testing.assert_allclose(k.sum(axis=1), 1.0, rtol=1e-5)  # unit L1 norm per bin, like the trained kernels
        assert 0.8 < np.linalg.norm(w["lowpass"]) < 1.2 and (w["cqt_scale"] > 0).all()
    k_d = np.abs(dense["cqt_real"]) + np.abs(dense["cqt_imag"])
    assert (k_d > 0).all()
    k_e = np.abs(edge["cqt_real"]) + np.abs(edge["cqt_imag"])
    assert (k_e[:, :32] > 0).all() and (k_e[:, 224:] > 0).all() and not k_e[:, 32:224].any()
    for layer in ("contour1", "contour2", "note1", "note2", "onset1", "onset2"):
        we, ws = edge[layer + "_w"], sparse[layer + "_w"]
        kh, kw = we.shape[2:]
        inner = we[:, :, 1 : kh - 1, 1 : kw - 1]
        assert not inner.any() and (we[:, :, [0, -1], :] != 0).all() and (we[:, :, :, [0, -1]] != 0).all(), layer
        assert np.count_nonzero(ws) == ws.shape[0] * ws.shape[1] and (ws[:, :, kh // 2, kw // 2] != 0).all(), layer
        b = dense[layer + "_b"]
        if b.size > 1:
            assert (b > 0).any() and (b < 0).any(), layer


def _ratios(o, b):
    r = {k: eb.ratio(o[k], b[k], b["b" + k]) for k in STAGES}
    r.update({k: eb.logit_check(o[k], b["l_" + k], b["b_" + k]) for k in POSTS})
    return r


@pytest.mark.parametrize("wset", weightsets.NAMES)
def test_error_bounds_hold_for_the_float32_oracle(wset):
    """The float32 oracle is a float32 implementation of the same graph: with eps = 0 it must lie within the bounds,
    end to end from the audio and stage by stage from its own intermediate inputs."""
    x = _windows()
    w = weightsets.get(wset)
    o = model_ref.forward(x, w, return_intermediates=True)
    for mode, kw in (("end-to-end", {}), ("per-stage", dict(y_in=o["_y"], contour_in=o["contour"], note_in=o["note"]))):
        r = _ratios(o, eb.forward_bounds(x, w, **kw))
        print(f"{wset} {mode}: max err/bound " + " ".join(f"{k}={v:.2e}" for k, v in r.items()))
        for k, v in r.items():
            assert v <= 1.0, (wset, mode, k, v)


def _drop(w, key, idx):
    d = {k: v.copy() for k, v in w.items()}
    d[key][idx] = 0.0
    return d


def test_error_bounds_catch_a_dropped_tap():
    """One tap dropped from one layer (what a kernel that misses an edge of its contraction computes) leaves the bound
    of the tensor-core paths (eps = EPS_SPLIT) of that stage — checked under `dense`, where every tap is non-zero."""
    x = _windows()
    w = weightsets.get("dense")
    ref = eb.forward_bounds(x, w, eb.EPS_SPLIT, eb.EPS_SPLIT)
    # (the end-to-end bound of the low-pass taps is weakest at its small edge taps: tap 255 is checked here)
    for keys, idx in ((("cqt_real", "cqt_imag"), (slice(None), 0)), (("cqt_real", "cqt_imag"), (slice(None), 255)),
                      (("lowpass",), 255)):
        d = w
        for key in keys:
            d = _drop(d, key, idx)
        r = eb.ratio(eb.forward_bounds(x, d)["_y"], ref["_y"], ref["b_y"])
        print(f"{keys} tap {idx} dropped: _y err/bound {r:.1f}")
        assert r > 1.0, (keys, idx, r)
    o = model_ref.forward(x, w, return_intermediates=True)
    given = dict(y_in=o["_y"], contour_in=o["contour"], note_in=o["note"])
    ref = eb.forward_bounds(x, w, eb.EPS_SPLIT, eb.EPS_SPLIT, **given)
    cases = (
        ("contour1_w", (7, 7, 2, 38), "_c1"), ("contour1_w", (0, 0, 0, 0), "_c1"), ("contour2_w", (0, 7, 4, 4), "l_contour"),
        ("note1_w", (3, 0, 6, 6), "_n1"), ("note2_w", (0, 5, 0, 2), "l_note"),
        ("onset1_w", (3, 7, 4, 4), "_o1"), ("onset2_w", (0, 0, 2, 2), "l_onset"), ("onset2_w", (0, 5, 0, 2), "l_onset"),
    )  # fmt: skip
    for key, idx, stage in cases:
        got = eb.forward_bounds(x, _drop(w, key, idx), **given)
        bkey = "b" + stage if stage.startswith("_") else "b_" + stage[2:]
        r = eb.ratio(got[stage], ref[stage], ref[bkey])
        print(f"{key}{list(idx)} dropped: {stage} err/bound {r:.1f}")
        assert r > 1.0, (key, idx, stage, r)
