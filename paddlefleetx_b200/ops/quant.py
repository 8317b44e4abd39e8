"""Quantised linear layers on the 8-bit wgmma GEMMs.

``Int8Linear``  — W8A8 inference layer: int8 weights with per-output-channel scales (from QAT abs-max statistics or from
                  post-training SmoothQuant), activations quantised per token on the fly (``quantize_rows`` kernel, optional
                  SmoothQuant divisor), product dequantised in the GEMM epilogue.
``fp8_linear``  — fp8-e4m3 forward GEMM for tensor-parallel training layers; backward runs in bf16 (master path) — "fp8 on the TP GEMMs"
                  of BASELINE config #3.  Two recipes: ``mx`` (OCP MX block scaling: one E8M0 scale per 32 K-elements, applied by the
                  tensor core, ``kind::mxf8f6f4.block_scale``) and ``rowwise`` (per-token x per-channel fp32 scales in the epilogue).

CPU / no-native fallbacks emulate the same arithmetic with torch ops so exported models are testable anywhere.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import _native
from . import functional as OF


def quantize_weight_int8(w: torch.Tensor, smooth: Optional[torch.Tensor] = None):
    """w: [out, in] -> (int8 [out, in], scale fp32 [out]).  ``smooth`` [in] multiplies the weight columns (SmoothQuant)."""
    wf = w.detach().float()
    if smooth is not None:
        wf = wf * smooth.float().unsqueeze(0)
    scale = wf.abs().amax(1).clamp(min=1e-8) / 127.0
    q = torch.clamp(torch.round(wf / scale.unsqueeze(1)), -127, 127).to(torch.int8)
    return q, scale


def quantize_rows_reference(x: torch.Tensor, smooth: Optional[torch.Tensor], fp8: bool = False):
    xf = x.detach().float()
    if smooth is not None:
        xf = xf / smooth.float()
    qmax = 448.0 if fp8 else 127.0
    scale = xf.abs().amax(-1).clamp(min=1e-12) / qmax
    scaled = xf / scale.unsqueeze(-1)
    if fp8:
        return scaled.to(torch.float8_e4m3fn), scale
    return torch.clamp(torch.round(scaled), -127, 127).to(torch.int8), scale


class Int8Linear(nn.Module):
    def __init__(self, weight_q: torch.Tensor, weight_scale: torch.Tensor, bias: Optional[torch.Tensor] = None,
                 smooth: Optional[torch.Tensor] = None, act_scale: Optional[float] = None):
        super().__init__()
        self.register_buffer("weight_q", weight_q.contiguous())
        self.register_buffer("weight_scale", weight_scale.float().contiguous())
        self.register_buffer("bias", None if bias is None else bias.to(torch.bfloat16).contiguous())
        self.register_buffer("smooth", None if smooth is None else smooth.float().contiguous())
        self.act_scale = act_scale               # static activation scale from QAT (None = dynamic per token)
        self.out_features, self.in_features = weight_q.shape

    @classmethod
    def from_float(cls, weight: torch.Tensor, bias=None, smooth=None, act_scale=None) -> "Int8Linear":
        q, s = quantize_weight_int8(weight, smooth)
        return cls(q, s, bias, smooth, act_scale)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        shp = x.shape
        x2 = x.reshape(-1, shp[-1])
        if x2.is_cuda and _native.use_native(x2) and x2.dtype in (torch.bfloat16, torch.float16) and shp[-1] % 16 == 0 and self.out_features % 8 == 0:
            lib = _native.require()
            xq, xs = lib.quantize_rows(x2.contiguous(), self.smooth, False)
            if x2.shape[0] <= 8:          # decode: int8 weight stream on dp4a (csrc/gemv_skinny.cu)
                y = lib.gemv_w8a8(xq, self.weight_q, xs, self.weight_scale, self.bias)
            else:
                y = lib.gemm_lowp(xq, self.weight_q, xs, self.weight_scale, self.bias, 0)
            OF._count(2)
            return y.view(*shp[:-1], self.out_features).to(x.dtype)
        xq, xs = quantize_rows_reference(x2, self.smooth)
        y = (xq.float() @ self.weight_q.float().t()) * xs.unsqueeze(1) * self.weight_scale.unsqueeze(0)
        if self.bias is not None:
            y = y + self.bias.float()
        return y.to(x.dtype).view(*shp[:-1], self.out_features)


def quantize_tp_linears_int8(model: nn.Module, skip=("word_embeddings",)) -> int:
    """Serving-time W8A8 conversion of a (single-GPU) model built from the tensor-parallel linear layers: every
    ``ColumnParallelLinear`` / ``RowParallelLinear`` weight is replaced by an :class:`Int8Linear` (per-output-channel weight scales,
    dynamic per-token activation scales).  Returns the number of converted layers.  The tied LM head / embedding stays bf16."""
    from ..parallel.tp_layers import ColumnParallelLinear, RowParallelLinear

    n = 0
    for name, mod in model.named_modules():
        if isinstance(mod, (ColumnParallelLinear, RowParallelLinear)) and mod.world == 1 and getattr(mod, "int8", None) is None \
                and not any(s in name for s in skip) and mod.weight is not None:
            mod.int8 = Int8Linear.from_float(mod.weight.data, None)
            mod._parameters["weight"] = None        # free the bf16 copy
            n += 1
    return n


class _Fp8LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        lib = _native.require()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        xq, xs = lib.quantize_rows(x2, None, True)
        wq, ws = lib.quantize_rows(weight.contiguous(), None, True)
        y = lib.gemm_lowp(xq, wq, xs, ws, bias, 0)
        OF._count(3)
        ctx.save_for_backward(x2, weight)
        ctx.has_bias, ctx.shape = bias is not None, x.shape
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, gy):
        lib = _native.require()
        x2, weight = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1]).contiguous()
        gx = lib.gemm(g2, weight, None, None, True, False, 0, 0, 0).view(ctx.shape)
        gw = lib.gemm(g2, x2, None, None, False, False, 0, 0, 0)
        gb = lib.colsum(g2, False) if ctx.has_bias else None
        OF._count(4)
        return gx, gw, gb


def quantize_mx_reference(x: torch.Tensor) -> torch.Tensor:
    """OCP MX fp8 (e4m3 elements, one power-of-two scale per 32 consecutive elements of the last dim) — returns the DEQUANTISED tensor in
    fp32, i.e. what the block-scaled tensor-core GEMM multiplies.  The scale is the smallest power of two that brings the block's maximum
    inside the e4m3 range; ``csrc/quant_kernels.cu: quantize_mxfp8`` makes the same choice."""
    shape = x.shape
    blocks = x.float().reshape(-1, 32)
    amax = blocks.abs().amax(dim=1, keepdim=True)
    e = torch.where(amax > 0, torch.ceil(torch.log2(amax / 448.0)), torch.full_like(amax, -127.0)).clamp_(-127, 127)
    scale = torch.exp2(e)
    q = (blocks / scale).clamp_(-448.0, 448.0).to(torch.float8_e4m3fn).float()
    return (q * scale).reshape(shape)


class _MxFp8LinearFn(torch.autograd.Function):
    """Forward GEMM on MX block-scaled fp8 operands (scales applied by the tensor core); backward in bf16 on the saved high-precision
    operands, like the row-wise recipe."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        lib = _native.require()
        x2 = x.reshape(-1, x.shape[-1]).contiguous()
        xq, xs = lib.quantize_mxfp8(x2)
        wq, ws = lib.quantize_mxfp8(weight.contiguous())
        y = lib.gemm_mxfp8(xq, xs, wq, ws, bias)
        OF._count(3)
        ctx.save_for_backward(x2, weight)
        ctx.has_bias, ctx.shape = bias is not None, x.shape
        return y.view(*x.shape[:-1], weight.shape[0])

    backward = _Fp8LinearFn.backward


def fp8_linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None, recipe: str = "rowwise") -> torch.Tensor:
    native = x.is_cuda and x.dtype == torch.bfloat16 and _native.use_native(x)
    if recipe == "mx" and weight.shape[1] % 128 == 0 and weight.shape[0] % 8 == 0:
        if native:
            return _MxFp8LinearFn.apply(x, weight, bias)
        y = quantize_mx_reference(x.reshape(-1, x.shape[-1])) @ quantize_mx_reference(weight).t()
        y = y.to(x.dtype).view(*x.shape[:-1], weight.shape[0])
        exact = torch.nn.functional.linear(x, weight, bias)
        return exact + (y + (0 if bias is None else bias) - exact).detach()
    if native and weight.shape[1] % 16 == 0 and weight.shape[0] % 8 == 0:
        return _Fp8LinearFn.apply(x, weight, bias)
    xq, xs = quantize_rows_reference(x.reshape(-1, x.shape[-1]), None, True)
    wq, ws = quantize_rows_reference(weight, None, True)
    y = (xq.float() * xs.unsqueeze(1)) @ (wq.float() * ws.unsqueeze(1)).t()
    y = y.to(x.dtype).view(*x.shape[:-1], weight.shape[0])
    # straight-through: gradients flow as if the GEMM were exact
    exact = torch.nn.functional.linear(x, weight, bias)
    return exact + (y + (0 if bias is None else bias) - exact).detach()
