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

End to end, the front end's bound of `_y` is loose (median 0.67 where y spans 2.5 under the trained weights), so the
front end is also checked stage by stage, each stage from the float32 input the kernel actually read, taken as exact
(tests/test_frontend_bounds.py on the CPU, tests/test_gpu_frontend.py on the kernels' own buffers):
  * decimation stage s: x_{s+1}[n] = sum_k h[k] x_s[2n + k - 127], zero-padded; bound gamma_256 sum |h||x_s|
    (`decimate_stage`)
  * octave o of the constant-Q projection from x_o (octave 0: the window with its zero fill): reflect padding of 128,
    hop 256 >> o, the octave's bins (g = (8 - o) 36 + bin - 15 >= 0), magnitude * cqt_scale, 10 log10(P + 1e-10) on
    the interval of P (`cqt_octave`).  Path 0 (FMAs): gamma_256 sum |k||x_o|.  Paths 1 / 2: (EPS_CQT3 + 2 K u (1 + 2^-5))
    sum |k||x_o|, EPS_CQT3 = 4.02 u the three-way split's dropped terms (derived next to the constant)
  * min / max: exact; normalisation and its bf16 hi / lo split: bit-exact float32 restatements (`lognorm_f32`,
    `split_operand`)
The 2 K u accumulation term of the tensor-core projection is as large as the whole error of a two-way split on real
signals, so the per-element bound cannot tell a two-way from the three-way split; `split_distance` can.
"""
from __future__ import annotations

import functools
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


def _log_power(re, im, ere, eim):
    """re, im (scaled by cqt_scale) with bounds ere, eim -> magnitude and its bound, 10 log10(P + 1e-10) and the ends of
    its interval.  The log is evaluated on the interval of the power, so bins whose power is lost in the error of the
    projection are bounded by the floor instead of by a first-order term; then the hardware log and the rounding."""
    mag = np.sqrt(re * re + im * im)
    bmag = np.sqrt(ere * ere + eim * eim) + 4 * U * mag
    power = mag * mag
    bp = 2 * mag * bmag + bmag * bmag + 2 * U * (power + 1e-10)
    lpw = DB * np.log(power + 1e-10)
    l_err = DB * np.log(2.0) * (2.0 ** -21 + 2.0 ** -22 * np.abs(np.log2(power + 1e-10))) + 3 * U * np.abs(lpw)
    l_lo = DB * np.log(np.maximum(power - bp, 0.0) + 1e-10) - l_err
    l_hi = DB * np.log(power + bp + 1e-10) + l_err
    return mag, bmag, lpw, l_lo, l_hi


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
    t = lambda v: v.transpose(1, 2).numpy()  # noqa: E731  (B, 172, 309)
    mag, bmag, lpw, l_lo, l_hi = _log_power(t(re), t(im), t(ere), t(eim))
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
    """max |got - ref| / bound over all elements (<= 1: within the bound; an exact element whose bound is 0, e.g. a
    decimation stage over silence, counts 0; a NaN anywhere makes the result NaN, which fails `<= 1`)"""
    got = np.asarray(got, np.float64)
    assert got.shape == ref.shape == bound.shape, (got.shape, ref.shape, bound.shape)
    err = np.abs(got - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.where((err == 0) & (bound == 0), 0.0, err / bound).max())


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


# ---------------------------------------------------------------------------------------------------------------------
# Front end stage by stage: each stage from the float32 input the implementation actually read, taken as exact
# ---------------------------------------------------------------------------------------------------------------------
# Three-way bf16 split of both operands of the tensor-core CQT (cqt_tc.cu): x = hi + mid + lo + r with hi = rn(x),
# mid = rn(x - hi), lo = rn(x - hi - mid), rn to bf16 (8-bit significand, unit roundoff 2^-8; both differences are exact
# in float32).  |x - hi| <= 2^-8 |x|, |mid| <= (1 + 2^-8) 2^-8 |x|, |x - hi - mid| <= 2^-16 |x|,
# |lo| <= (1 + 2^-8) 2^-16 |x|, |r| <= 2^-24 |x|.  Of the sixteen products of a * w the kernel keeps hi*hi, hi*mid,
# mid*hi, hi*lo, lo*hi, mid*mid (each exact in float32); what it drops is
#   r_a w + (a - r_a) r_w                 <= (2 + 2^-24) 2^-24 |a||w|
#   mid*lo + lo*mid                       <= 2 (1 + 2^-8)^2 2^-24 |a||w|
#   lo*lo                                 <= (1 + 2^-8)^2 2^-32 |a||w|
# in all < 4.02 * 2^-24 |a||w|.
# Accumulation: the six kept products of all 256 taps sum in magnitude to T <= (1 + 2^-7)^2 (1 + 2^-7 + 3 * 2^-16)
# sum |a||w| < (1 + 2^-5) sum |a||w|.  They reach one accumulator through 96 wgmma updates (4 K-chunks x 4 k-steps x 6
# products), update i adding 16 exact products P_i to the accumulator d_{i-1}.  One update is modelled as erring by at
# most c 2u (|d_{i-1}| + sum |P_i|): the truncation of its result to float32 (< 2u relative) plus the truncating
# alignment of its 17 addends to the largest exponent, c <= 1 + 17 * 2^-g with g guard bits.  To first order the
# errors add up to c 2u sum_i (|d_{i-1}| + sum |P_i|) <= c 2u (95 T + T) = c 2u 96 T, since every partial sum |d| <= T.
# The 2 K u T with K = 256 used here therefore covers c <= 256 / 96 = 2.67, i.e. g >= 4 guard bits in the alignment
# (1 + 17/16 = 2.06).  The alignment width is not documented; it is the one assumption about the hardware in this bound,
# and the GPU test holds cqt_tc_kernel's output to it (largest err/bound 0.38 on an H100 SXM).
EPS_CQT3 = 4.02 * U
ACC_TC = 2 * 256 * U * (1 + 2.0 ** -5)  # truncating MMA accumulation of the 6 * 256 products, per sum |a||w|
ACC_FMA = 256 * U / (1 - 256 * U)  # gamma_256: 256 FMAs, round to nearest, any order


@functools.lru_cache(maxsize=None)
def chain_layout():
    """(offsets, lengths, stride) of the decimation chain buffer, from the library (bp_debug_chain_layout):
    x_o (o >= 1) of window b is chain[b, offsets[o] : offsets[o] + lengths[o]]; lengths[0] is the window."""
    import ctypes

    from basic_pitch_b200 import _lib

    off, ln, st = np.zeros(9, np.int32), np.zeros(9, np.int32), ctypes.c_int32()
    _lib.load().bp_debug_chain_layout(off.ctypes.data, ln.ctypes.data, ctypes.byref(st))
    return tuple(int(v) for v in off), tuple(int(v) for v in ln), int(st.value)


def decimate_stage(x: np.ndarray, h: np.ndarray):
    """x_{s+1}[n] = sum_k h[k] x_s[2n + k - 127], zero-padded, for a (B, len_s) input taken as exact -> value (float64)
    and bound gamma_256 sum_k |h[k]| |x_s[2n + k - 127]|"""
    xt = _t(x)[:, None]
    lp = _t(h)[None, None]
    n_out = (x.shape[1] - 2) // 2 + 1
    v = F.conv1d(F.pad(xt, (127, 127)), lp, stride=2)[:, 0, :n_out]
    m = F.conv1d(F.pad(xt.abs(), (127, 127)), lp.abs(), stride=2)[:, 0, :n_out]
    return v.numpy(), ACC_FMA * m.numpy()


def reflect_index(length: int, shift_lo: int = 0, shift_hi: int = 0) -> np.ndarray:
    """signal index of padded position p - 128 (p < length + 256) under reflect padding of 128; shift_lo / shift_hi move
    the reflection at either end (0 = torch / the kernels)"""
    i = np.arange(-128, length + 128)
    i = np.where(i < 0, -i - shift_lo, i)
    return np.where(i >= length, 2 * (length - 1) - i + shift_hi, i)


def octave_frames(x: np.ndarray, o: int, index=None) -> np.ndarray:
    """(B, len_o) -> the (B, 172, 256) operand of octave o: frame t reads the reflect-padded signal at t * hop + k"""
    hop = 256 >> o
    idx = reflect_index(x.shape[1]) if index is None else index
    pos = np.arange(model_ref.N_FRAMES)[:, None] * hop + np.arange(256)[None, :]
    return np.asarray(x, np.float64)[:, idx[pos]]


def octave_bins(o: int):
    """(first kernel bin, first global bin) of octave o: global bin g = (8 - o) * 36 + bin - 15 for g >= 0"""
    g0 = (8 - o) * 36 - 15
    return max(0, -g0), max(0, g0)


def cqt_kernel_matrix(w) -> np.ndarray:
    """(256, 72) float64: columns interleave the real and imaginary kernels of the 36 bins (the sign of the imaginary
    part does not reach the magnitude)"""
    k = np.empty((256, 72))
    k[:, 0::2] = np.asarray(w["cqt_real"], np.float64).T
    k[:, 1::2] = np.asarray(w["cqt_imag"], np.float64).T
    return k


def cqt_octave(x: np.ndarray, w: Dict[str, np.ndarray], o: int, path: int, proj=None):
    """Log-magnitudes of octave o from the (B, len_o) float32 signal x_o the kernel read (octave 0: the window with its
    zero fill), taken as exact: (value, bound), each (B, 172, bins of the octave), and the octave's global bins.
    path 0: 256 FMAs per column (cqt_kernel); paths 1, 2: the three-way split and the truncating MMA (cqt_tc_kernel).
    `proj` (B, 172, 72) replaces the float64 projection as the value (a fault or an emulation to score)."""
    a = octave_frames(x, o)
    k = cqt_kernel_matrix(w)
    c = a @ k if proj is None else np.asarray(proj, np.float64)
    mabs = np.abs(a) @ np.abs(k)
    e = (ACC_FMA if path == 0 else EPS_CQT3 + ACC_TC) * mabs
    b0, g0 = octave_bins(o)
    s = np.asarray(w["cqt_scale"], np.float64)[g0 : g0 + 36 - b0]
    re, im, ere, eim = c[..., 0::2][..., b0:], c[..., 1::2][..., b0:], e[..., 0::2][..., b0:], e[..., 1::2][..., b0:]
    _, _, lpw, l_lo, l_hi = _log_power(re * s, im * s, ere * s, eim * s)
    return lpw, np.maximum(lpw - l_lo, l_hi - lpw), np.arange(g0, g0 + 36 - b0)


def bf16_rn(v: np.ndarray) -> np.ndarray:
    """float32 -> bf16 bits (uint16), round to nearest even (__float2bfloat16_rn for finite values)"""
    u = np.ascontiguousarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def bf16_value(h: np.ndarray) -> np.ndarray:
    return (h.astype(np.uint32) << 16).view(np.float32)


def split3(v: np.ndarray):
    """the three bf16 planes of cqt_tc.cu as float32 values: hi, mid, lo"""
    v = np.asarray(v, np.float32)
    hi = bf16_value(bf16_rn(v))
    r1 = v - hi
    mid = bf16_value(bf16_rn(r1))
    return hi, mid, bf16_value(bf16_rn(r1 - mid))


def lognorm_f32(log: np.ndarray, minmax: np.ndarray, w: Dict[str, np.ndarray]) -> np.ndarray:
    """lognorm_kernel / lognorm_split_kernel in float32, operation by operation: (L - mn) / (mx - mn) * bn_scale +
    bn_bias per window, 0 * bn_scale + bn_bias when mx == mn.  log (B, 172, 309), minmax (B, 2) -> exact bits"""
    f = np.float32
    log = np.asarray(log, f)
    mn = np.asarray(minmax[:, 0], f)[:, None, None]
    mx = (np.asarray(minmax[:, 1], f)[:, None, None] - mn).astype(f)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = np.where(mx == 0, f(0), ((log - mn).astype(f) / mx).astype(f)).astype(f)
    return ((q * f(w["bn_scale"][0])).astype(f) + f(w["bn_bias"][0])).astype(f)


def split_operand(y: np.ndarray, rows_total: int, lead: int, rows_per_window: int, chunks8: int) -> np.ndarray:
    """lognorm_split_kernel's output for normalised windows y (B, 172, 309): bf16 bits [2][chunks8][rows_total][8],
    hi = rn(v), lo = rn(v - hi); row lead + b * rows_per_window + t holds frame t of window b, everything else is 0"""
    n = y.shape[0]
    v = np.zeros((rows_total, chunks8 * 8), np.float32)
    rows = lead + np.arange(n)[:, None] * rows_per_window + np.arange(model_ref.N_FRAMES)[None, :]
    v[rows.reshape(-1), : y.shape[2]] = y.reshape(-1, y.shape[2])
    hi = bf16_rn(v)
    lo = bf16_rn(v - bf16_value(hi))
    out = np.stack([hi, lo]).reshape(2, rows_total, chunks8, 8)
    return np.ascontiguousarray(out.transpose(0, 2, 1, 3))


def split_distance(got: np.ndarray, ref3: np.ndarray, ref2: np.ndarray) -> float:
    """sum |got - ref2| / sum |got - ref3| over an octave's log-magnitudes: how much closer `got` lies to the three-way
    split (ref3, float64) than to a two-way split (ref2).  The worst-case bound cannot tell the two apart (EPS_CQT3)."""
    g = np.asarray(got, np.float64)
    return float(np.abs(g - ref2).sum() / max(np.abs(g - ref3).sum(), 1e-300))
