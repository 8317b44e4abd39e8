"""Attention front-end.

``attention(q, k, v)`` takes ``[b, s, heads, d]`` tensors (views are fine: the slices of a packed QKV projection, sequence-major
storage).  Path selection on CUDA / bf16:
  * training and inference at head_dim 128 or 64: our wgmma flash kernels — ``csrc/attention_fwd_sm90.cu`` and
    ``csrc/attention_bwd_sm90.cu`` — with in-kernel causal masking and counter-hash dropout (the backward regenerates the mask; nothing is
    stored).  ``flash_attention_packed`` is the same pair for the ``[b, s, heads, 3, d]`` output of a fused QKV projection: it reads q / k / v
    in place and writes ONE packed gradient, so no split / cat copies surround the kernels,
  * single-query decode steps over the static KV cache use ``csrc/attention_decode.cu`` (see models/.../gpt/model.py),
  * explicit masks, other head sizes (backward), fp16 and CPU tensors: PyTorch SDPA — a *library* call, reported as such by the launch
    accounting (it does not count towards ``gpu_launches``); ``PFX_NATIVE_ATTN=0`` forces it everywhere,
  * the unfused reference path (QK^T -> fused causal softmax -> PV) used when ``use_flash_attn=False`` — this mirrors reference
    ``core_attn`` (hybrid_model.py:303-346).
"""
from __future__ import annotations

from typing import Optional

import os

import torch
import torch.nn.functional as F

# 1 (default) = our kernels wherever they apply, 0 = library SDPA everywhere (A/B runs, debugging)
_NATIVE = int(os.environ.get("PFX_NATIVE_ATTN", "1"))
_MASK64 = (1 << 64) - 1


def _native_ok(q, k, v, attn_mask, causal, needs_grad: bool) -> bool:
    if not _NATIVE or attn_mask is not None or not q.is_cuda or q.dtype != torch.bfloat16 or k.dtype != q.dtype or v.dtype != q.dtype:
        return False
    d = q.shape[-1]
    if d not in (64, 128) or q.shape[1] < 1 or (causal and k.shape[1] < q.shape[1]):
        return False
    for t in (q, k, v):
        if t.dim() != 4 or t.stride(3) != 1 or any(t.stride(i) % 8 for i in range(3)) or t.data_ptr() % 16:
            return False
    from . import _native

    return _native.available()


def _dropout_seed(dropout_p: float, numel: int) -> int:
    if dropout_p <= 0.0:
        return 0
    from ..parallel.rng import get_rng_state_tracker

    seed, offset = get_rng_state_tracker().philox(numel)           # advances the active stream: recompute replays the same pair
    return ((int(seed) * 0x9E3779B97F4A7C15) ^ (int(offset) * 0xD1B54A32D192ED03 + 0x2545F4914F6CDD1D)) & 0x7FFFFFFFFFFFFFFF


def attn_keep_mask(seed: int, B: int, H: int, Sq: int, Sk: int, p: float, device) -> torch.Tensor:
    """The keep mask ``[B, H, Sq, Sk]`` (bool) our kernels generate for ``seed`` — a pure-PyTorch replica of csrc/pfx_attn.cuh used by
    the numerics tests (fp32 reference with the SAME dropout pattern)."""
    M = 0xFFFFFFFF

    def mix(x):
        x = x ^ (x >> 16); x = (x * 0x85EBCA6B) & M; x = x ^ (x >> 13); x = (x * 0xC2B2AE35) & M; x = x ^ (x >> 16)
        return x

    bh = torch.arange(B * H, device=device, dtype=torch.int64)
    key = mix(((seed & M) + 0x9E3779B9 * (bh + 1)) & M) ^ ((seed >> 32) & M)             # [BH]
    pairs = (Sk + 1) // 2
    q = torch.arange(Sq, device=device, dtype=torch.int64).view(1, Sq, 1)
    kp = torch.arange(pairs, device=device, dtype=torch.int64).view(1, 1, pairs)
    x = (q * pairs + kp) & M
    x = x ^ (x >> 16); x = (x * 0x85EBCA6B) & M
    x = x ^ key.view(-1, 1, 1)
    x = x ^ (x >> 13); x = (x * 0xC2B2AE35) & M; x = x ^ (x >> 16)
    thresh = int(p * 65536.0 + 0.5)
    even, odd = (x & 0xFFFF) >= thresh, (x >> 16) >= thresh
    keep = torch.stack([even, odd], dim=-1).reshape(B * H, Sq, 2 * pairs)[:, :, :Sk]
    return keep.view(B, H, Sq, Sk)


class _FlashAttnFn(torch.autograd.Function):
    """q / k / v ``[b, s, h, d]`` views -> ``[b, s, h, d]``.  ``packed`` = the three are slices of one ``[b, s, h, 3, d]`` tensor, which is
    then the single differentiable input (and the single gradient: dq / dk / dv are written straight into its three slices)."""

    @staticmethod
    def forward(ctx, packed, q, k, v, causal, scale, dropout_p, seed):
        from . import _native
        from . import functional as OF

        if packed is not None:
            q, k, v = packed.unbind(3)
        out, lse = _native.require().attention_fwd_v2(q, k, v, bool(causal), float(scale), float(dropout_p), int(seed))
        OF._count()
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.cfg = (packed is not None, bool(causal), float(scale), float(dropout_p), int(seed))
        return out

    @staticmethod
    def backward(ctx, dout):
        from . import _native
        from . import functional as OF

        q, k, v, out, lse = ctx.saved_tensors
        is_packed, causal, scale, dropout_p, seed = ctx.cfg
        if dout.stride(3) != 1 or any(dout.stride(i) % 8 for i in range(3)):
            dout = dout.contiguous()
        dmix = None
        if is_packed:
            b, s, h, d = q.shape
            dmix = torch.empty(b, s, h, 3, d, dtype=q.dtype, device=q.device)
            dq, dk, dv = dmix.unbind(3)
        else:
            dq, dk, dv = torch.empty_like(q, memory_format=torch.contiguous_format), torch.empty_like(k, memory_format=torch.contiguous_format), \
                torch.empty_like(v, memory_format=torch.contiguous_format)
        _native.require().attention_bwd(q, k, v, out, dout, lse, dq, dk, dv, causal, scale, dropout_p, seed)
        OF._count(4)           # memset is a driver call; prep + main + dq convert (+ the tensor-core kernel counted once more for its size)
        if is_packed:
            return dmix, None, None, None, None, None, None, None
        return None, dq, dk, dv, None, None, None, None


def flash_attention_packed(mix: torch.Tensor, causal: bool = True, dropout_p: float = 0.0, scale: Optional[float] = None) -> Optional[torch.Tensor]:
    """Attention on the ``[b, s, heads, 3, d]`` view of a fused QKV projection output (any batch / sequence strides).  Returns ``None`` when
    the native kernels do not apply (caller falls back to ``attention`` on the unbound slices)."""
    if mix.dim() != 5 or mix.shape[3] != 3:
        return None
    q, k, v = mix.unbind(3)
    needs_grad = torch.is_grad_enabled() and mix.requires_grad
    if not _native_ok(q, k, v, None, causal, needs_grad):
        return None
    sc = float(scale if scale is not None else q.shape[-1] ** -0.5)
    seed = _dropout_seed(dropout_p, q.shape[0] * q.shape[2] * q.shape[1] * k.shape[1])
    return _FlashAttnFn.apply(mix, None, None, None, causal, sc, dropout_p, seed)


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True, dropout_p: float = 0.0,
              scale: Optional[float] = None, attn_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    needs_grad = torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad)
    if _native_ok(q, k, v, attn_mask, causal, needs_grad):
        sc = float(scale if scale is not None else q.shape[-1] ** -0.5)
        seed = _dropout_seed(dropout_p, q.shape[0] * q.shape[2] * q.shape[1] * k.shape[1])
        return _FlashAttnFn.apply(None, q, k, v, causal, sc, dropout_p, seed)
    qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))           # [b, h, s, d]
    if attn_mask is not None:
        causal = False
    out = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=attn_mask, dropout_p=dropout_p, is_causal=causal, scale=scale)
    return out.transpose(1, 2)


def core_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, dropout_p: float, training: bool,
                   attn_mask: Optional[torch.Tensor] = None, causal: bool = True, rng_name: Optional[str] = "local_seed"
                   ) -> torch.Tensor:
    """Unfused attention: scores materialised as ``[b, heads, sq, sk]``."""
    from . import functional as OF

    qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
    scores = torch.matmul(qt, kt.transpose(-1, -2))
    if attn_mask is None and causal:
        probs = OF.causal_softmax(scores.contiguous(), scale)
    else:
        scores = scores.float() * scale
        if attn_mask is not None:
            scores = scores + attn_mask.float()
        probs = torch.softmax(scores, -1).to(q.dtype)
    probs = OF.dropout(probs, dropout_p, training, rng_name)
    return torch.matmul(probs, vt).transpose(1, 2)
