"""float64 references and error bounds for the SwiGLU kernels (``bias_swiglu`` forward / backward and the SwiGLU finish of the decode GEMV),
in the style of ``kernel_refs``: a reference takes the exact values the kernel was given and computes in float64, and a bound is the
``kernel_refs.assert_close`` arguments that cover the kernel's own error.

Layout: z [.., 2F] is pair-interleaved, column 2i the gate channel i and column 2i + 1 its up channel; the bias [2F] follows the same order.
With a = g + b_g, b = u + b_u and s = sigmoid(a):

    h  = a s b                          [.., F]
    dg = dh b s (1 + a (1 - s))         dz[.., 2i]
    du = dh a s                         dz[.., 2i + 1]

The kernels evaluate this in fp32 with s = 1 / (1 + __expf(-a)) under --use_fast_math (``1 / x`` is rcp.approx.ftz.f32, at most 1 ulp):

    a, b      one fp32 rounding each (2^-24 relative);
    s         __expf(-a): EXPF_ULP (2 + 1.173 |a|); the add 1 + e: 2^-24; the reciprocal: 1 ulp (EXPF_ULP).  An error de of e moves s by
              e / (1 + e) de <= de relatively.  The rounding of a itself moves s by (1 - s) |a| 2^-24 relatively.  Together
              rel_s <= EXPF_ULP (4 + 1.2 |a|) + 2^-24 |a|;
    h         the rounding of a moves a s by |1 + a (1 - s)| 2^-24 <= (1 + |a|) 2^-24, then s, b and two products:
              rel_h <= 2^-24 (4 + |a|) + EXPF_ULP (4 + 1.2 |a|);
    du        the same products as h with dh in place of b: rel_h;
    dg        t = 1 + a (1 - s): 1 - s is formed directly (no e s, which would be inf * 0 for a saturated gate), so its absolute error is
              s rel_s + 2^-24 (1 - s); a (1 - s) adds the roundings of a and the product, 1 + . one more.  Then |dh b s| (|t| (rel_s + 5 2^-24)
              + |a| (s rel_s + 3 2^-24)) bounds dg's error before the output rounding.

A saturated gate is exact in the limit: for a < -88 __expf(-a) overflows to inf and s = h = dz = 0, while float64 keeps e^a; that
difference is below 2^-122 (``FTZ_FLOOR``) wherever the result is a normal bf16 number.  Every bound is absolute (``approx = 1``: the
``_abs_bound`` form of ``kernel_refs``), so the elementwise test reads |got - ref| <= 4 (u (|ref| + tiny) + E + 2^-122).
"""
from __future__ import annotations

import torch

from kernel_refs import EXPF_ULP, FP32_U, _d

__all__ = ["split_pairs", "swiglu", "swiglu_grad", "swiglu_bound"]


def split_pairs(z, bias=None):
    """float64 (a, b) = (gate + b_g, up + b_u) of pair-interleaved z [.., 2F] and bias [2F]."""
    z = _d(z)
    if bias is not None:
        z = z + _d(bias)
    return z[..., 0::2], z[..., 1::2]


def swiglu(z, bias=None):
    """h [.., F] = silu(a) * b in float64."""
    a, b = split_pairs(z, bias)
    return a * torch.sigmoid(a) * b


def swiglu_grad(dh, z, bias=None):
    """dz [.., 2F] (pair-interleaved: dg at 2i, du at 2i + 1) of ``swiglu`` for the output gradient dh [.., F], in float64."""
    a, b = split_pairs(z, bias)
    s = torch.sigmoid(a)
    g = _d(dh)
    dz = torch.empty(*a.shape[:-1], 2 * a.shape[-1], dtype=torch.float64, device=a.device)
    dz[..., 0::2] = g * b * s * (1.0 + a * (1.0 - s))
    dz[..., 1::2] = g * a * s
    return dz


def _sigmoid_rel(a):
    return EXPF_ULP * (4 + 1.2 * a.abs()) + FP32_U * a.abs()


def swiglu_bound(z, bias=None, dh=None):
    """``assert_close`` arguments for ``swiglu`` (``dh`` None) or ``swiglu_grad`` (``dh`` given) of these kernel inputs (module docstring)."""
    a, b = split_pairs(z, bias)
    s = torch.sigmoid(a)
    aa = a.abs()
    rel_h = FP32_U * (4 + aa) + EXPF_ULP * (4 + 1.2 * aa)
    if dh is None:
        return dict(scale=(a * s * b).abs() * rel_h, approx=1.0)
    g = _d(dh).abs()
    rel_s = _sigmoid_rel(a)
    t = (1.0 + a * (1.0 - s)).abs()
    E = torch.empty(*a.shape[:-1], 2 * a.shape[-1], dtype=torch.float64, device=a.device)
    E[..., 0::2] = g * b.abs() * s * (t * (rel_s + 5 * FP32_U) + aa * (s * rel_s + 3 * FP32_U))
    E[..., 1::2] = g * aa * s * rel_h
    return dict(scale=E, approx=1.0)
