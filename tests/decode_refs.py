"""References for the text-generation kernels, in the style of ``kernel_refs``: the counter-based Philox generator the sampler and dropout
draw from, the law of top-p (nucleus) sampling in float64, and a float64 reference with its error bound for the decode GEMV
(``gemv_skinny`` / ``gemv_fused``).  Nothing here needs CUDA.

Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC 2011) as ``Philox`` in csrc/pfx_common.cuh uses it: the
key is the 64-bit seed (low word first), the counter words 0 and 1 are the 64-bit counter (low word first) and words 2 and 3 are the fixed
0x243F6A88, 0x85A308D3.  ``uniform`` is word 0 shifted right by 8 and scaled by 2^-24, a float32 in [0, 1).

Top-p law: draw the threshold u = uniform * top_p (one float32 product, as the kernel forms it), sort the row by descending probability
with ties in ascending index order, and return the first token whose cumulative mass reaches u.  If rounding leaves u above the whole
row's mass, the last token of positive probability in that order is returned.

GEMV bound: every bound is absolute (``dict(scale=E, approx=1.0)``, the form ``swiglu_refs`` uses), so the elementwise test reads
|got - ref| <= 4 (u (|ref| + tiny) + E), with E the error the kernel may make before its final rounding to the output dtype (module
docstring of ``gemv_ref``).
"""
from __future__ import annotations

import math

import numpy as np
import torch

import kernel_refs as R
import swiglu_refs as S

__all__ = ["philox4x32", "philox", "uniform", "keep8", "topp_threshold", "sorted_mass", "topp_expected", "gemv_ref"]

_M0, _M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint32(0x9E3779B9), np.uint32(0xBB67AE85)
_C2, _C3 = 0x243F6A88, 0x85A308D3
_LO = np.uint64(0xFFFFFFFF)


def philox4x32(ctr, key, rounds=10):
    """Philox4x32 of four-word counters ``ctr`` [..., 4] and two-word keys ``key`` [..., 2] (uint32, broadcast) -> uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint32)
    key = np.asarray(key, dtype=np.uint32)
    shape = np.broadcast_shapes(ctr.shape[:-1], key.shape[:-1])
    c = [np.broadcast_to(ctr[..., i], shape).astype(np.uint32) for i in range(4)]
    k0, k1 = (np.broadcast_to(key[..., i], shape).astype(np.uint32) for i in range(2))
    with np.errstate(over="ignore"):                               # uint32 key bumps wrap by design
        for _ in range(rounds):
            c, k0, k1 = _round(c, k0, k1)
    return np.stack(c, -1)


def _round(c, k0, k1):
    """One Philox round on the counter words c and the key (k0, k1) -> (c, k0 + W0, k1 + W1)."""
    p0 = _M0 * c[0].astype(np.uint64)
    p1 = _M1 * c[2].astype(np.uint64)
    hi0, lo0 = (p0 >> np.uint64(32)).astype(np.uint32), (p0 & _LO).astype(np.uint32)
    hi1, lo1 = (p1 >> np.uint64(32)).astype(np.uint32), (p1 & _LO).astype(np.uint32)
    return [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0], k0 + _W0, k1 + _W1


def _words(v):
    v = np.asarray(v, dtype=np.uint64)
    return (v & _LO).astype(np.uint32), (v >> np.uint64(32)).astype(np.uint32)


def philox(seed, counter):
    """``Philox::gen(seed, counter)``: uint32 [..., 4] for uint64 counters (array or scalar)."""
    s0, s1 = _words(seed)
    c0, c1 = _words(counter)
    ctr = np.stack([c0, c1, np.full_like(c0, _C2), np.full_like(c0, _C3)], -1)
    return philox4x32(ctr, np.stack([s0, s1], -1))


def uniform(seed, counter):
    """``Philox::uniform(seed, counter)``: float32 in [0, 1), exactly as the kernels compute it."""
    x = philox(seed, counter)[..., 0]
    return (x >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)


def keep8(seed, offset, n_vec, thresh16):
    """``Philox::keep8`` for vectors 0 .. n_vec - 1 -> bool [n_vec * 8]: element 8 v + 2 i keeps when the low half of word i of
    gen(seed, offset + v) is >= thresh16, element 8 v + 2 i + 1 when the high half is."""
    r = philox(seed, np.uint64(offset) + np.arange(n_vec, dtype=np.uint64))
    halves = np.stack([r & np.uint32(0xFFFF), r >> np.uint32(16)], -1)        # [n_vec, 4 words, 2 halves]
    return (halves >= thresh16).reshape(-1)


def topp_threshold(seed, counters, top_ps):
    """float32 thresholds u = uniform(seed, counter) * top_p, one per row, as the sampler forms them."""
    return uniform(seed, counters) * np.asarray(top_ps, dtype=np.float32)


def sorted_mass(probs):
    """float64 probs [R, V] -> (order [R, V], cum [R, V]): the tokens by descending probability, ties in ascending index order, and the
    cumulative mass through each of them."""
    p = torch.as_tensor(probs).to(torch.float64)
    order = torch.sort(-p, dim=-1, stable=True).indices
    return order, p.gather(-1, order).cumsum(-1)


def topp_expected(probs, top_p, u):
    """The top-p law (module docstring) for probs [R, V] (any float dtype, read exactly), top_p [R] and the uniform draws u [R] (float32).

    Returns (ids int64 [R], margin float64 [R]): the token the law picks and the distance from the threshold u * top_p to the nearer edge of
    that token's cumulative-mass interval.
    """
    p = torch.as_tensor(probs).to(torch.float64)
    thr = torch.as_tensor(np.asarray(u, dtype=np.float32) * np.asarray(top_p, dtype=np.float32)).to(p.device, torch.float64).reshape(-1, 1)
    thr = thr.expand(p.shape[0], 1).contiguous()
    order, cum = sorted_mass(p)
    V = p.shape[-1]
    k = torch.searchsorted(cum, thr).squeeze(-1)                  # first position with cum >= thr
    positive = p.gather(-1, order) > 0
    last = V - 1 - positive.flip(-1).int().argmax(-1)             # the last positive token in sorted order
    k = torch.where(k >= V, last, k)
    rows = torch.arange(p.shape[0], device=p.device)
    hi = cum[rows, k]
    lo = torch.where(k > 0, cum[rows, (k - 1).clamp(min=0)], torch.zeros_like(hi))
    t = thr.squeeze(-1)
    return order[rows, k], torch.minimum((t - lo).abs(), (hi - t).abs())


# ---------------------------------------------------------------------------------------------------------------- decode GEMV
def _dot_depth(K):
    """Longest fp32 rounding chain of one GEMV output: a lane's fma chain over its share of K (8 elements per 16-byte vector, one vector per
    32 lanes and step), 5 shuffle levels, up to 8 K-slices and the bias."""
    return 8 * math.ceil(K / 256) + 16


def gemv_ref(x, w, b=None, ln=None, res=None, act=None):
    """float64 reference and ``assert_close`` bound of ``gemv_fused`` (``act`` None, "gelu" or "swiglu"; ``ln = (gamma, beta, eps)``).

    The kernel's error before its output rounding, per output element:

    * LayerNorm prologue (two fp32 passes: a per-thread strided sum over K / 256 terms, 5 shuffle levels, 8 warp partials, an approximate
      division): the mean is off by at most delta = (ceil(K / 256) + 17) 2^-24 mean|x| and rstd by rho, half the variance's relative error
      plus rsqrt.approx's.  Both errors are common to a row, so their effect on output n is exact to first order: delta rstd |sum_k g_k w_nk|
      and rho |sum_k w_nk xhat_k g_k|.  The elementwise (x - mean) rstd g + b adds 3 2^-24 |xhat g| + 2^-24 |y| per input.
    * the dot product: ``_dot_depth(K)`` 2^-24 times the sum of |terms| (bias included).
    * the finish: GELU(tanh) moves by |gelu'(z)| dz plus tanh.approx's error (``TANH_APPROX``) times |z| / 2; SwiGLU as ``swiglu_refs``
      with the pre-activation errors propagated through its partial derivatives; a residual adds one fp32 rounding.

    Inputs offset far from zero make a one-pass variance (E[x^2] - E[x]^2 in fp32) cancel far beyond this bound.
    """
    u = R.FP32_U
    K = x.shape[-1]
    wd, xd = R._d(w), R._d(x)
    E = torch.zeros(x.shape[0], w.shape[0], dtype=torch.float64, device=xd.device)
    if ln is None:
        y = xd
    else:
        g, beta = R._d(ln[0]), R._d(ln[1])
        y, mean, rstd = R.layer_norm(x, ln[0], ln[1], ln[2])
        xg = (xd - mean[:, None]) * rstd[:, None] * g
        depth = math.ceil(K / 256) + 13
        delta = (depth + 4) * u * xd.abs().mean(-1)
        var = ((xd - mean[:, None]) ** 2).mean(-1)
        rel_var = (depth + 8) * u + delta ** 2 / var
        rho = 0.5 * rel_var * var / (var + ln[2]) + 2.0 ** -22 + u
        E = (delta * rstd)[:, None] * (wd @ g).abs()[None, :] + rho[:, None] * (xg @ wd.t()).abs() \
            + u * ((3 * xg.abs() + y.abs()) @ wd.abs().t())
    z = y @ wd.t() + (R._d(b) if b is not None else 0.0)
    terms = y.abs() @ wd.abs().t() + (R._d(b).abs() if b is not None else 0.0)
    dz = E + _dot_depth(K) * u * terms
    if act is None:
        h, E = z, dz
    elif act == "gelu":
        h = R.gelu(z, exact=False)
        E = R.gelu_grad(z, exact=False).abs() * dz + 0.5 * z.abs() * (R.TANH_APPROX + 4 * u) + 2 * u * h.abs()
    elif act == "swiglu":
        h = S.swiglu(z)
        a, bb = z[:, 0::2], z[:, 1::2]
        s = torch.sigmoid(a)
        # a moves h by |d h / d a| = |b s (1 + a (1 - s))|, b by |a s|
        E = S.swiglu_bound(z)["scale"] + (bb * s * (1 + a * (1 - s))).abs() * dz[:, 0::2] + (a * s).abs() * dz[:, 1::2]
    else:
        raise ValueError(f"act must be None, 'gelu' or 'swiglu', got {act!r}")
    if res is not None:
        h = h + R._d(res)
        E = E + u * h.abs()
    return h, dict(scale=E, approx=1.0)
