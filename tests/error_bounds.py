"""Per-element error bounds for the forward pass (CPU only: float64 torch / NumPy).

`forward_bounds` recomputes the oracle (oracle/model_ref.py) in float64 and carries, next to every value, a rigorous
first-order bound on how far a float32 implementation of the same graph may be from it.  The GPU tests compare each
activation the library exposes, and the three posteriorgrams in logit space, against these bounds instead of fixed
tolerances; a kernel that drops or misplaces one tap leaves them by orders of magnitude (tests/test_weightsets.py
checks both directions on the CPU).

Model of the arithmetic (u = 2^-24, the float32 unit roundoff):
  * a dot product of K terms accumulated in float32 errs by at most K u sum|terms|; the tensor cores do not round
    to nearest inside an MMA, so 2 K u is used
  * operands split into bf16 hi + lo (both sides, three products) lose eps = 3 * 2^-16 < 2^-14 of sum|terms|
  * decimation (scalar FMAs, round to nearest): E_{s+1} = |lowpass| * E_s + 256 u (|lowpass| * (|x_s| + E_s))
  * CQT:  e = |kernel| * E_o + (eps_cqt + 2 * 256 u) (|kernel| * (|x_o| + E_o)), times cqt_scale; the magnitude, the
    power, 10 log10(P + 1e-10) (evaluated on the interval of P, plus the error of a fast hardware log2: 2^-21 absolute
    + 2 ulp of |log2|), the per-window min / max normalisation (evaluated on the interval ends of the min, the max and
    the cell) and the folded BatchNorm follow with their own rounding
  * a convolution: B_out = conv(B_in, |w|) + (eps + 2 K u) conv(|x| + B_in, |w|) + u (|out| + |bias|), K = fan-in;
    ReLU is 1-Lipschitz
  * a sigmoid: the bound of its logit times the largest slope on [l - B, l + B], plus the error of a fast exp
    ((2 + 1.16 |l|) ulp relative, which moves the logit by the same amount) and the final rounding
Posteriorgrams are compared in logit space (`logit_check`): a sigmoid output hides logit errors by p (1 - p).
"""
from __future__ import annotations

from typing import Dict

import numpy as np
import torch
import torch.nn.functional as F

from oracle import model_ref

U = 2.0 ** -24
EPS_SPLIT = 2.0 ** -14  # bf16 hi/lo split of both operands, hi*hi + hi*lo + lo*hi: 3 * 2^-16 of sum|terms|
DB = 10.0 / np.log(10.0)


def _t(a) -> torch.Tensor:
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64))


def _exp_err(l):
    """relative error of a fast float32 exp(-l) (ex2.approx based: 2 + 1.16 |l| ulp), as a logit error"""
    return (2.0 + 1.16 * np.abs(l)) * 2.0 ** -23


def _sig(l):
    return 1.0 / (1.0 + np.exp(-l))


def _sigmoid_bound(l, bl):
    """|sigmoid(l') - sigmoid(l)| for |l' - l| <= bl, plus the float32 evaluation of sigmoid(l')"""
    far = np.maximum(np.abs(l) - bl, 0.0)
    slope = _sig(far) * (1.0 - _sig(far))
    p = _sig(l)
    return slope * bl + _exp_err(l) * p * (1.0 - p) + 2 * U


def _conv(x, b_x, w, bias, eps, stride=(1, 1), pad=(0, 0, 0, 0)):
    """value, bound of conv2d(pad(x), w) + bias (pad = (left_f, right_f, top_t, bottom_t), zero filled)"""
    wt, aw = _t(w), _t(np.abs(w))
    k = w.shape[1] * w.shape[2] * w.shape[3] + 1
    z = F.conv2d(F.pad(x, pad), wt, _t(bias), stride=stride)
    prop = F.conv2d(F.pad(b_x, pad), aw, stride=stride)
    mag = F.conv2d(F.pad(x.abs() + b_x, pad), aw, stride=stride)
    bz = prop + (eps + 2 * k * U) * mag + U * (z.abs() + _t(np.abs(bias))[None, :, None, None])
    return z, bz


def _cqt_bounds(audio: np.ndarray, w: Dict[str, np.ndarray], eps_cqt: float):
    """(B, 43844) -> y after BatchNorm (B, 172, 309) and its bound, plus per-stage diagnostics"""
    x = _t(audio)[:, None, :]
    e = torch.zeros_like(x)
    k_re, k_im = _t(w["cqt_real"])[:, None, :], _t(w["cqt_imag"])[:, None, :]
    ak_re, ak_im = k_re.abs(), k_im.abs()
    lp = _t(w["lowpass"])[None, None, :]
    alp = lp.abs()
    re_l, im_l, ere_l, eim_l = [], [], [], []
    hop = 256
    for o in range(model_ref.N_OCTAVES):
        p = F.pad(x, (128, 128), mode="reflect")
        pe = F.pad(e, (128, 128), mode="reflect")
        pa = p.abs() + pe
        re_l.insert(0, F.conv1d(p, k_re, stride=hop))
        im_l.insert(0, -F.conv1d(p, k_im, stride=hop))
        ere_l.insert(0, F.conv1d(pe, ak_re, stride=hop) + (eps_cqt + 2 * 256 * U) * F.conv1d(pa, ak_re, stride=hop))
        eim_l.insert(0, F.conv1d(pe, ak_im, stride=hop) + (eps_cqt + 2 * 256 * U) * F.conv1d(pa, ak_im, stride=hop))
        if o < model_ref.N_OCTAVES - 1:
            xa = F.pad(x.abs() + e, (127, 127))
            e = F.conv1d(F.pad(e, (127, 127)), alp, stride=2) + 256 * U * F.conv1d(xa, alp, stride=2)
            x = F.conv1d(F.pad(x, (127, 127)), lp, stride=2)
            hop //= 2
    sc = _t(w["cqt_scale"])[None, :, None]
    re = torch.cat(re_l, 1)[:, -model_ref.N_BINS :] * sc
    im = torch.cat(im_l, 1)[:, -model_ref.N_BINS :] * sc
    ere = torch.cat(ere_l, 1)[:, -model_ref.N_BINS :] * sc
    eim = torch.cat(eim_l, 1)[:, -model_ref.N_BINS :] * sc
    mag = torch.sqrt(re * re + im * im)
    bmag = torch.sqrt(ere * ere + eim * eim) + 4 * U * mag
    mag, bmag = mag.transpose(1, 2).numpy(), bmag.transpose(1, 2).numpy()  # (B, 172, 309)
    # 10 log10(P + 1e-10) over the interval of the power, so bins whose power is lost in the error of the projection
    # are bounded by the floor instead of by a first-order term; then the hardware log and the rounding
    power = mag * mag
    bp = 2 * mag * bmag + bmag * bmag + 2 * U * (power + 1e-10)
    lpw = DB * np.log(power + 1e-10)
    l_err = DB * np.log(2.0) * (2.0 ** -21 + 2.0 ** -22 * np.abs(np.log2(power + 1e-10))) + 3 * U * np.abs(lpw)
    l_lo = DB * np.log(np.maximum(power - bp, 0.0) + 1e-10) - l_err
    l_hi = DB * np.log(power + bp + 1e-10) + l_err
    bl = np.maximum(lpw - l_lo, l_hi - lpw)
    # normalisation y = (L - min L) / max(L - min L) per window, evaluated on the interval ends: the min and the max
    # of the window move with the error of the cells that hold them, the numerator with the cell's own
    ax = (1, 2)
    mn = lpw.min(axis=ax, keepdims=True)
    off = lpw - mn
    mx = off.max(axis=ax, keepdims=True)
    mn_lo, mn_hi = l_lo.min(axis=ax, keepdims=True), l_hi.min(axis=ax, keepdims=True)
    mx_lo = np.maximum(l_lo.max(axis=ax, keepdims=True) - mn_hi, 0.0)
    mx_hi = l_hi.max(axis=ax, keepdims=True) - mn_lo
    num_lo, num_hi = np.maximum(l_lo - mn_hi, 0.0), l_hi - mn_lo
    with np.errstate(divide="ignore", invalid="ignore"):
        y = np.where(mx == 0, 0.0, off / mx)
        y_lo = num_lo / mx_hi
        y_hi = np.where(mx_lo > 0, num_hi / mx_lo, 1.0)
        by = np.where(mx_lo > 0, np.maximum(y - y_lo, y_hi - y) * (1 + 4 * U) + 4 * U * y, 1.0)
    by = np.minimum(by, 1.0)  # both sides lie in [0, 1]
    bs, bb = float(w["bn_scale"][0]), float(w["bn_bias"][0])
    yb = y * bs + bb
    byb = abs(bs) * by + 2 * U * (np.abs(y * bs) + abs(bb))
    return yb, byb, dict(mag=mag, b_mag=bmag, log=lpw, b_log=bl)


def forward_bounds(audio: np.ndarray, w: Dict[str, np.ndarray], eps_cqt: float = 0.0, eps_conv: float = 0.0,
                   y_in=None, contour_in=None, note_in=None):
    """float64 oracle + per-element bounds.  eps_cqt / eps_conv: split-operand error of the CQT projection / the convs
    (EPS_SPLIT on the tensor-core paths, 0 for plain float32).
    Returns values `_y`, `_c1`, `_n1`, `_o1`, `l_contour`, `l_note`, `l_onset` (logits) and `b<key>` bounds.

    End to end, the worst-case bound of the eight-stage decimation chain grows like ||lowpass||_1^8 and swamps the
    convolutions behind it.  So each stage can also be checked on the input the implementation actually fed it:
    y_in (B, 172, 309) replaces the log-spectrum in front of the contour / onset convs, contour_in (B, 172, 264) the
    contour posteriorgram in front of the note conv, note_in (B, 172, 88) the note posteriorgram in front of the onset
    conv2; each is taken as exact up to one float32 rounding.  `_y` and its bound always come from the audio."""
    a = np.ascontiguousarray(audio, np.float32).astype(np.float64)
    if a.ndim == 3:
        a = a[..., 0]

    def given(v, ch_axis=True):
        v = _t(v)
        v = v[:, None] if ch_axis else v
        return v, 2 * U * v.abs()

    with torch.no_grad():
        yb, byb, diag = _cqt_bounds(a, w, eps_cqt)
        y, by = given(y_in, False) if y_in is not None else (_t(yb), _t(byb))
        h, bh = model_ref.harmonic_stack(y), model_ref.harmonic_stack(by)
        z, bz = _conv(h, bh, w["contour1_w"], w["contour1_b"], eps_conv, pad=(19, 19, 1, 1))
        c1 = torch.relu(z)
        lc, blc = _conv(c1, bz, w["contour2_w"], w["contour2_b"], eps_conv, pad=(2, 2, 2, 2))
        if contour_in is not None:
            pc, bpc = given(contour_in)
        else:
            pc, bpc = torch.sigmoid(lc), _t(_sigmoid_bound(lc.numpy(), blc.numpy()))
        z, bz_n = _conv(pc, bpc, w["note1_w"], w["note1_b"], eps_conv, stride=(1, 3), pad=(2, 2, 3, 3))
        n1 = torch.relu(z)
        ln, bln = _conv(n1, bz_n, w["note2_w"], w["note2_b"], eps_conv, pad=(1, 1, 3, 3))
        if note_in is not None:
            pn, bpn = given(note_in)
        else:
            pn, bpn = torch.sigmoid(ln), _t(_sigmoid_bound(ln.numpy(), bln.numpy()))
        z, bz_o = _conv(h, bh, w["onset1_w"], w["onset1_b"], eps_conv, stride=(1, 3), pad=(1, 1, 2, 2))
        o1 = torch.relu(z)
        lo, blo = _conv(torch.cat((pn, o1), 1), torch.cat((bpn, bz_o), 1), w["onset2_w"], w["onset2_b"], eps_conv,
                        pad=(1, 1, 1, 1))
    out = {
        "_y": yb, "b_y": byb,
        "_c1": c1.numpy(), "b_c1": bz.numpy(),
        "_n1": n1.numpy(), "b_n1": bz_n.numpy(),
        "_o1": o1.numpy(), "b_o1": bz_o.numpy(),
        "l_contour": lc[:, 0].numpy(), "b_contour": blc[:, 0].numpy(),
        "l_note": ln[:, 0].numpy(), "b_note": bln[:, 0].numpy(),
        "l_onset": lo[:, 0].numpy(), "b_onset": blo[:, 0].numpy(),
    }  # fmt: skip
    out.update({"_" + k: v for k, v in diag.items()})
    return out


def ratio(got: np.ndarray, ref: np.ndarray, bound: np.ndarray) -> float:
    """max |got - ref| / bound over all elements (<= 1: within the bound)"""
    got = np.asarray(got, np.float64)
    assert got.shape == ref.shape == bound.shape, (got.shape, ref.shape, bound.shape)
    return float((np.abs(got - ref) / bound).max())


def logit_check(p_got: np.ndarray, l_ref: np.ndarray, b_ref: np.ndarray) -> float:
    """A float32 posteriorgram against the float64 logit and its bound, in logit space: max err / bound.
    The bound grows by what a float32 p can resolve (rounding of p, 4 u / (1 - p), and of the fast exp); cells where p
    rounded to exactly 0 or 1 have no finite logit and only have to agree on the side."""
    p = np.asarray(p_got, np.float64)
    assert p.shape == l_ref.shape == b_ref.shape, (p.shape, l_ref.shape)
    sat1, sat0 = p >= 1.0, p <= 0.0
    assert not (sat1 & (l_ref + b_ref < 15.0)).any(), "posteriorgram 1.0 where the logit is well below saturation"
    assert not (sat0 & (l_ref - b_ref > -80.0)).any(), "posteriorgram 0.0 where the logit is well above underflow"
    ok = ~(sat0 | sat1)
    pc = np.clip(p, 2.0 ** -149, 1.0 - 2.0 ** -24)
    l_got = np.log(pc) - np.log1p(-pc)
    bound = b_ref + _exp_err(l_ref) + 4 * U * (1.0 + 1.0 / (1.0 - pc)) + 4 * U
    r = np.where(ok, np.abs(l_got - l_ref) / bound, 0.0)
    return float(r.max())
