"""Synthetic parameter sets for the forward kernels (CPU only: plain NumPy, deterministic).

The shipped weights leave parts of the kernels unobserved: the CQT kernels are zero on taps 0-20 and 236-255 of every
bin, the low-pass edge taps are 1e-4 of its peak, and the conv weight tiles happen to be pairwise distinct.  These sets
make every tap count:

  dense      every tensor random: complex CQT kernels on all 256 taps (unit L1 norm per bin, like the trained ones), a
             randomly perturbed low-pass of L2 norm 1 (eight decimation stages neither vanish nor explode), positive random
             cqt_scale, conv weights N(0, gain^2 / fan_in), mixed-sign biases (ReLU clips a sizeable fraction)
  edge_taps  the CQT kernels live only on taps 0-31 and 224-255 (reflect padding of the first and last frame), conv1 and
             conv2 weights only on the outermost time and frequency taps (zero rows between windows, frequency halo,
             harmonic-stack edge gating)
  sparse     one centre tap per (co, ci) in every conv: the weight tiles of the tensor-core programs collapse to a few
             distinct contents, which used to change the programs themselves
  trained    the shipped weights

Every set is checked for liveness (tests/test_weightsets.py): a comparison under a set whose posteriorgrams saturate
or whose log-spectrum sits on the power floor would prove nothing.
"""
from __future__ import annotations

import functools
from typing import Dict

import numpy as np

NAMES = ("trained", "dense", "edge_taps", "sparse")

# conv1 / conv2 layers: name -> weight shape (co, ci, kh, kw)
_CONVS = {
    "contour1": (8, 8, 3, 39),
    "contour2": (1, 8, 5, 5),
    "note1": (32, 1, 7, 7),
    "note2": (1, 32, 7, 3),
    "onset1": (32, 8, 5, 5),
    "onset2": (1, 33, 3, 3),
}
# weight gain per layer: He-like for the ReLU layers; the last convs are scaled so that the logits of the
# posteriorgrams mostly stay within a few units of zero
_GAIN = {"contour1": 1.5, "contour2": 1.2, "note1": 1.5, "note2": 1.2, "onset1": 1.5, "onset2": 1.2}
_BIAS = {"contour1": 0.3, "contour2": 0.0, "note1": 0.3, "note2": 0.0, "onset1": 0.3, "onset2": 0.0}


def _trained() -> Dict[str, np.ndarray]:
    from basic_pitch_b200 import ICASSP_2022_MODEL_PATH, weights

    return weights.load(ICASSP_2022_MODEL_PATH)


def _cqt_kernels(rng, taps: np.ndarray):
    k = np.zeros((36, 256), np.complex128)
    k[:, taps] = rng.standard_normal((36, len(taps))) + 1j * rng.standard_normal((36, len(taps)))
    k /= np.abs(k).sum(axis=1, keepdims=True)
    return k.real.astype(np.float32), k.imag.astype(np.float32)


def _conv(rng, name: str, mask=None):
    co, ci, kh, kw = _CONVS[name]
    w = rng.standard_normal((co, ci, kh, kw))
    if mask is not None:
        w = w * mask
    fan_in = ci * kh * kw if mask is None else max(1, int(mask.sum()))
    w *= _GAIN[name] / np.sqrt(fan_in)
    b = _BIAS[name] * rng.standard_normal(co) - (0.1 if co > 1 else 0.0)
    return w.astype(np.float32), b.astype(np.float32)


def _dsp(rng, taps: np.ndarray) -> Dict[str, np.ndarray]:
    re, im = _cqt_kernels(rng, taps)
    # the shipped half-band low-pass with every tap perturbed (1 % of its peak), scaled to L2 norm 1: all 256 taps
    # count, and its L1 norm (4.4; a white random FIR has ~13) keeps the worst-case error bound of the eight-stage
    # chain, which grows like ||lowpass||_1^8, usable
    lp = _trained()["lowpass"].astype(np.float64)
    lp = lp + 0.01 * np.abs(lp).max() * rng.standard_normal(256)
    lp /= np.linalg.norm(lp)
    return {
        "cqt_real": re,
        "cqt_imag": im,
        "lowpass": lp.astype(np.float32),
        "cqt_scale": rng.uniform(10.0, 200.0, 309).astype(np.float32),
        "bn_scale": np.array([2.5], np.float32),
        "bn_bias": np.array([-0.9], np.float32),
    }


def _edge_mask(shape):
    m = np.zeros(shape)
    m[:, :, [0, -1], :] = 1.0
    m[:, :, :, [0, -1]] = 1.0
    return m


def _centre_mask(shape):
    m = np.zeros(shape)
    m[:, :, shape[2] // 2, shape[3] // 2] = 1.0
    return m


def _synthetic(name: str) -> Dict[str, np.ndarray]:
    rng = np.random.default_rng({"dense": 101, "edge_taps": 202, "sparse": 303}[name])
    taps = np.r_[0:32, 224:256] if name == "edge_taps" else np.arange(256)
    w = _dsp(rng, taps)
    for layer, shape in _CONVS.items():
        mask = _edge_mask(shape) if name == "edge_taps" else _centre_mask(shape) if name == "sparse" else None
        w[layer + "_w"], w[layer + "_b"] = _conv(rng, layer, mask)
    return w


@functools.lru_cache(maxsize=None)
def _get(name: str) -> Dict[str, np.ndarray]:
    from basic_pitch_b200 import weights

    if name not in NAMES:
        raise KeyError(name)
    w = _trained() if name == "trained" else _synthetic(name)
    weights.validate(w, source=name)
    for v in w.values():
        v.setflags(write=False)
    return w


def get(name: str) -> Dict[str, np.ndarray]:
    """The parameter set `name` (read-only arrays; copy before changing)."""
    return _get(name)


def blob(name: str) -> bytes:
    """`name` packed as a BPW1 weight blob (what bp_model_create reads)."""
    from basic_pitch_b200 import weights

    return weights.pack(get(name))
