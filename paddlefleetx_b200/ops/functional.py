"""Functional op layer: every hot op of the model zoo goes through one of these.

On CUDA (bf16/fp16) the call lands in the hand-written sm_90a kernels of ``csrc/`` through an
``autograd.Function``; on CPU (and for fp32 debugging runs) the plain PyTorch expression next to it is used —
that expression is also the numerical reference in ``tests/``.  There is no runtime backend dispatch beyond
this device check: a CUDA tensor with a missing native library raises.

Reference call sites being replaced (SURVEY §2.6 L1-L15): ``FusedLinear`` / cuBLASLt epilogues, Paddle
LayerNorm, ``softmax_mask_fuse_upper_triangle``, ``c_softmax_with_cross_entropy``, dropout, fused AdamW,
``check_finite_and_unscale``, the custom ``topp_sampling`` op.
"""
from __future__ import annotations

import os
from typing import Optional, Tuple

import torch
import torch.nn.functional as F

from . import _native
from ..parallel.rng import get_rng_state_tracker

_LOWP = (torch.bfloat16, torch.float16)
_SMALLM = os.environ.get("PFX_SMALLM_GEMM", "1") == "1"
_GEMV_MAX_ROWS = 2 if _SMALLM else 8       # the swap-AB wgmma kernel serves 3 rows and up

# launch accounting for bench.py ("gpu_launches": kernels of OURS inside the timed region)
_launch_count = 0


def _count(n: int = 1) -> None:
    global _launch_count
    _launch_count += n


def native_launch_count() -> int:
    return _launch_count


def reset_launch_count() -> None:
    global _launch_count
    _launch_count = 0


def _native_ok(*ts) -> bool:
    t0 = next(t for t in ts if isinstance(t, torch.Tensor))
    return t0.is_cuda and t0.dtype in _LOWP and _native.use_native(*ts)


def _gemm_ok(x: torch.Tensor, *dims: int) -> bool:
    return x.is_cuda and x.dtype == torch.bfloat16 and all(d % 8 == 0 for d in dims) and _native.use_native(x)


# =============================================================================== linear
EPI_NONE, EPI_BIAS, EPI_BIAS_GELU, EPI_GELU = 0, 1, 2, 3


def _wgrad(lib, g2: torch.Tensor, x2: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
    """dW = g2^T x2.  With a flat gradient buffer behind the weight (``weight.main_grad``, set up by FusedAdamW) the GEMM stores or
    accumulates straight into it and a placeholder is handed to autograd (see optims/optimizer.py: direct gradient writes)."""
    main_grad = getattr(weight, "main_grad", None)
    if main_grad is not None:
        fresh = getattr(weight, "_grad_fresh", False)      # first touch since clear_grad: store, do not accumulate
        if main_grad.dtype == torch.float32:
            lib.gemm(g2, x2, None, main_grad, False, False, EPI_NONE, 1 if fresh else 2, 0)   # main_grad (+)= dY^T X
        elif fresh:
            lib.gemm(g2, x2, None, main_grad, False, False, EPI_NONE, 0, 0)
        else:
            main_grad.add_(lib.gemm(g2, x2, None, None, False, False, EPI_NONE, 0, 0))
        weight._grad_fresh = False
        # autograd still needs a tensor so that post-accumulate hooks (DP / ZeRO bucket readiness) fire; the optimizer's hook
        # drops ``weight.grad`` when this flag is set.
        weight.grad_added_to_main_grad = True
        gw = torch.empty_like(weight)
    else:
        gw = lib.gemm(g2, x2, None, None, False, False, EPI_NONE, 0, 0)
    _count()
    return gw


class _FusedFFNFn(torch.autograd.Function):
    """y = gelu(x W1^T + b1) W2^T with the elementwise work inside the GEMM epilogues: the FFN1 GEMM writes both the pre-activation
    (kept for the backward) and its GELU, the FFN2 dgrad GEMM multiplies by gelu'(pre-activation) on the way out.  Compared with
    linear -> bias_gelu -> linear this removes two full passes over the [tokens, 4h] activation in forward and three in backward
    (reference: FusedLinear + separate gelu kernel, hybrid_model.py:598-669; SURVEY L3 "GELU fusable in epilogue")."""

    @staticmethod
    def forward(ctx, x, w1, b1, w2, b2):
        lib = _native.require()
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        z, g = lib.gemm_bias_gelu_dual(x2, w1, b1)
        y = lib.gemm(g, w2, b2, None, True, True, EPI_BIAS if b2 is not None else EPI_NONE, 0, 0)
        _count(2)
        ctx.save_for_backward(x2, w1, w2, z, g)
        ctx.x_shape = x.shape
        ctx.has_b2 = b2 is not None
        return y.view(*x.shape[:-1], w2.shape[0])

    @staticmethod
    def backward(ctx, gy):
        lib = _native.require()
        x2, w1, w2, z, g = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1])
        if not g2.is_contiguous():
            g2 = g2.contiguous()
        dz = lib.gemm_dgelu(g2, w2, z)                      # (dy W2) * gelu'(z)
        _count()
        gw2 = _wgrad(lib, g2, g, w2) if ctx.needs_input_grad[3] else None
        gb1 = None
        if ctx.needs_input_grad[2]:
            gb1 = lib.colsum(dz, False)
            _count(2)
        gw1 = _wgrad(lib, dz, x2, w1) if ctx.needs_input_grad[1] else None
        gx = None
        if ctx.needs_input_grad[0]:
            gx = lib.gemm(dz, w1, None, None, True, False, EPI_NONE, 0, 0).view(ctx.x_shape)
            _count()
        gb2 = None
        if ctx.has_b2 and ctx.needs_input_grad[4]:
            gb2 = lib.colsum(g2, False)
            _count(2)
        return gx, gw1, gb1, gw2, gb2


_FUSED_FFN = os.environ.get("PFX_FUSED_FFN", "1") == "1"


def fused_ffn(x: torch.Tensor, w1: torch.Tensor, b1: torch.Tensor, w2: torch.Tensor, b2: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``gelu(x @ w1.T + b1) @ w2.T (+ b2)`` (tanh GELU).  The decoder layer passes ``b2 = None`` and folds that bias into its
    bias+dropout+residual kernel; expert FFNs pass it."""
    if (_FUSED_FFN and x.is_cuda and x.dtype == torch.bfloat16 and w1.dtype == torch.bfloat16 and w2.dtype == torch.bfloat16 and b1 is not None
            and b1.dtype == torch.bfloat16 and w1.is_contiguous() and w2.is_contiguous() and w1.shape[0] % 8 == 0 and w1.shape[1] % 8 == 0
            and w2.shape[0] % 8 == 0 and x.numel() // x.shape[-1] > 128 and (b2 is None or b2.dtype == torch.bfloat16) and _native.use_native(x)):
        return _FusedFFNFn.apply(x, w1, b1, w2, b2)
    return linear(bias_gelu(linear(x, w1, None), b1), w2, b2)


class _LinearFn(torch.autograd.Function):
    """y = x W^T (+ b).  fwd: TN wgmma GEMM with bias epilogue; dgrad: NN GEMM (B MN-major, no transpose
    copy); wgrad: TN GEMM with both operands MN-major, optionally accumulating straight into an fp32
    ``main_grad`` buffer (reference amp.py:44-63 does that with a separate elementwise hook)."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        lib = _native.require()
        x2 = x.reshape(-1, x.shape[-1])
        if not x2.is_contiguous():
            x2 = x2.contiguous()
        y = lib.gemm(x2, weight, bias, None, True, True, EPI_BIAS if bias is not None else EPI_NONE, 0, 0)
        _count()
        ctx.save_for_backward(x2, weight)
        ctx.has_bias = bias is not None
        ctx.x_shape = x.shape
        return y.view(*x.shape[:-1], weight.shape[0])

    @staticmethod
    def backward(ctx, gy):
        lib = _native.require()
        x2, weight = ctx.saved_tensors
        g2 = gy.reshape(-1, gy.shape[-1])
        if not g2.is_contiguous():
            g2 = g2.contiguous()
        gx = gw = gb = None
        if ctx.needs_input_grad[0]:
            gx = lib.gemm(g2, weight, None, None, True, False, EPI_NONE, 0, 0).view(ctx.x_shape)
            _count()
        if ctx.needs_input_grad[1]:
            gw = _wgrad(lib, g2, x2, weight)
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = lib.colsum(g2, False)
            _count(2)
        return gx, gw, gb


def linear(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor] = None) -> torch.Tensor:
    """weight is ``[out, in]``."""
    if (x.is_cuda and x.dtype == weight.dtype and x.dtype in (torch.bfloat16, torch.float16) and weight.is_contiguous()
            and x.numel() // x.shape[-1] <= _GEMV_MAX_ROWS and x.shape[-1] % 8 == 0 and not (torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad))
            and _native.available()):
        # token-by-token decoding: a weight stream, not a tensor-core problem (csrc/gemv_skinny.cu)
        _count()
        y = _native.require().gemv_skinny(x.reshape(-1, x.shape[-1]).contiguous(), weight, bias)
        return y.view(*x.shape[:-1], weight.shape[0])
    if (_SMALLM and x.is_cuda and x.dtype == torch.bfloat16 and weight.dtype == torch.bfloat16 and weight.is_contiguous()
            and x.numel() // x.shape[-1] <= 128 and x.shape[-1] % 8 == 0 and weight.shape[0] % 8 == 0
            and not (torch.is_grad_enabled() and (x.requires_grad or weight.requires_grad)) and _native.available()):
        # prefill / batched decode: swap-AB wgmma GEMM, split-K over a cluster (csrc/gemm_smallm_sm90.cu)
        _count()
        y = _native.require().gemm_smallm(x.reshape(-1, x.shape[-1]).contiguous(), weight, bias, 0)
        return y.view(*x.shape[:-1], weight.shape[0])
    if _gemm_ok(x, weight.shape[0], weight.shape[1]) and weight.dtype == torch.bfloat16 and weight.is_contiguous():
        return _LinearFn.apply(x, weight, bias)
    return F.linear(x, weight, bias)


def native_available() -> bool:
    return _native.available()


class _EmbeddingFn(torch.autograd.Function):
    """out = W[ids - vocab_start] (zero rows for ids of other vocab shards) (+ P[pos]).  Backward: deterministic sorted scatter-add
    (csrc/embedding.cu) straight into the flat optimizer's ``main_grad`` rows when present — the tied LM head has usually written that
    buffer already, so only the rows that occur are touched — or into a dense gradient otherwise."""

    @staticmethod
    def forward(ctx, ids, weight, vocab_start, pos_ids, pos_weight):
        lib = _native.require()
        ids_c = ids.contiguous()
        pos_c = pos_ids.contiguous() if pos_ids is not None else None
        out = lib.embedding_fwd(ids_c, weight, pos_c, pos_weight, int(vocab_start))
        _count()
        ctx.save_for_backward(ids_c, pos_c if pos_c is not None else ids_c)
        ctx.weights = (weight, pos_weight)
        ctx.vocab_start = int(vocab_start)
        return out

    @staticmethod
    def _scatter(lib, ids, dout2, weight, vocab_start):
        main_grad = getattr(weight, "main_grad", None)
        if main_grad is not None:
            if getattr(weight, "_grad_fresh", False):
                main_grad.zero_()
            target, ret = main_grad, torch.empty_like(weight)      # placeholder: the optimizer hook drops it (see _wgrad)
            weight._grad_fresh = False
            weight.grad_added_to_main_grad = True
        else:
            target = ret = torch.zeros_like(weight)
        flat = ids.reshape(-1)
        step = int(lib.embedding_bwd_max_tokens())
        for a in range(0, flat.numel(), step):                     # one sorted pass per <= 16 K tokens, in token order: deterministic
            lib.embedding_bwd_(flat[a:a + step], dout2[a:a + step], target, vocab_start, True)
            _count(2)
        return ret

    @staticmethod
    def backward(ctx, dout):
        lib = _native.require()
        ids, pos = ctx.saved_tensors
        weight, pos_weight = ctx.weights
        d2 = dout.reshape(-1, dout.shape[-1])
        if not d2.is_contiguous():
            d2 = d2.contiguous()
        gw = gp = None
        if ctx.needs_input_grad[1]:
            gw = _EmbeddingFn._scatter(lib, ids, d2, weight, ctx.vocab_start)
        if pos_weight is not None and ctx.needs_input_grad[4]:
            gp = _EmbeddingFn._scatter(lib, pos, d2, pos_weight, 0)
        return None, gw, None, None, gp


def embedding(ids: torch.Tensor, weight: torch.Tensor, vocab_start: int = 0, pos_ids: Optional[torch.Tensor] = None,
              pos_weight: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Word (+ position) embedding look-up; ``vocab_start`` selects this rank's rows of a vocabulary-parallel table (foreign ids give zero rows)."""
    if (weight.is_cuda and weight.dtype in (torch.bfloat16, torch.float16) and weight.shape[1] % 8 == 0 and weight.is_contiguous() and ids.dtype == torch.int64
            and (pos_weight is None or (pos_weight.dtype == weight.dtype and pos_weight.is_contiguous() and pos_ids is not None and pos_ids.dtype == torch.int64
                                        and pos_ids.shape == ids.shape)) and _native.use_native(weight)):
        return _EmbeddingFn.apply(ids, weight, vocab_start, pos_ids, pos_weight)
    local = ids - vocab_start
    if vocab_start != 0 or bool(((local < 0) | (local >= weight.shape[0])).any()):
        oob = (local < 0) | (local >= weight.shape[0])
        out = F.embedding(local.masked_fill(oob, 0), weight).masked_fill(oob.unsqueeze(-1), 0.0)
    else:
        out = F.embedding(ids, weight)
    if pos_weight is not None:
        out = out + F.embedding(pos_ids, pos_weight)
    return out


def gemv_max_rows() -> int:
    return _GEMV_MAX_ROWS


def gemv_fused(x: torch.Tensor, weight: torch.Tensor, bias=None, ln=None, residual=None, act: Optional[str] = None) -> torch.Tensor:
    """Decode-step linear with optional LayerNorm prologue (``ln = (gamma, beta, eps)``), GELU(tanh) and ``+ residual``:
    ``act((LN(x)) W^T + b) + residual`` for <= 8 rows in one weight-streaming kernel (csrc/gemv_skinny.cu)."""
    if x.is_cuda and _native.available():
        _count()
        lw, lb, eps = (ln[0], ln[1], float(ln[2])) if ln is not None else (None, None, 1e-5)
        return _native.require().gemv_fused(x.contiguous(), weight, bias, lw, lb, eps, None if residual is None else residual.contiguous(),
                                            1 if act == "gelu" else 0)
    h = x if ln is None else F.layer_norm(x.float(), (x.shape[-1],), ln[0].float(), ln[1].float(), ln[2]).to(x.dtype)
    y = F.linear(h, weight, bias)
    if act == "gelu":
        y = F.gelu(y, approximate="tanh")
    return y if residual is None else y + residual


def attention_decode_packed(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, additive_mask: torch.Tensor, write_idx: torch.Tensor,
                            scale: float) -> torch.Tensor:
    """``qkv`` [B,1,H,3,D]: append this token's K/V at ``write_idx`` and attend over the whole static cache (one kernel)."""
    if qkv.is_cuda and _native.available():
        _count()
        return _native.require().attention_decode_packed(qkv.contiguous(), k_cache, v_cache, additive_mask, write_idx, float(scale))
    q, k, v = qkv.unbind(3)
    k_cache.index_copy_(1, write_idx, k)
    v_cache.index_copy_(1, write_idx, v)
    return attention_decode(q, k_cache, v_cache, additive_mask, scale)


def attention_decode(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, additive_mask: torch.Tensor, scale: float) -> torch.Tensor:
    """q [B,1,H,D] against the whole static cache [B,Lmax,H,D]; ``additive_mask`` ([B,1,1,Lmax] or [B,Lmax]) hides padded and
    not-yet-written positions.  CPU / fallback: the plain softmax expression (also the numerical reference in the tests)."""
    if q.is_cuda and _native.available():
        _count()
        return _native.require().attention_decode(q.contiguous(), k_cache, v_cache, additive_mask, k_cache.shape[1], float(scale))
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k_cache.float()) * scale + additive_mask.reshape(q.shape[0], 1, 1, -1).float()
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v_cache.float()).to(q.dtype)


def matmul_nt(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """a[M,K] @ b[N,K]^T without autograd (used by fused comm paths and inference)."""
    if _gemm_ok(a, a.shape[-1], b.shape[0]):
        _count()
        return _native.require().gemm(a, b, None, None, True, True, EPI_NONE, 0, 0)
    return a @ b.t()


# =============================================================================== bias + gelu
class _BiasGeluFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias, exact=False):
        lib = _native.require()
        x = x.contiguous()
        ctx.save_for_backward(x, bias)
        ctx.exact = bool(exact)
        _count()
        return lib.bias_gelu_fwd(x, bias, ctx.exact)

    @staticmethod
    def backward(ctx, gy):
        lib = _native.require()
        x, bias = ctx.saved_tensors
        gx = lib.bias_gelu_bwd(gy.contiguous(), x, bias, ctx.exact)
        _count()
        gb = None
        if bias is not None and ctx.needs_input_grad[1]:
            gb = lib.colsum(gx.view(-1, gx.shape[-1]), False)
            _count(2)
        return gx, gb, None


def bias_gelu(x: torch.Tensor, bias: Optional[torch.Tensor] = None, exact: bool = False) -> torch.Tensor:
    """GELU of (x + bias): tanh approximation by default (reference GPT, hybrid_model.py:667 ``approximate=True``), exact erf form
    with ``exact=True`` (``nn.GELU`` default, used by the vision / multimodal models)."""
    if _native_ok(x) and x.shape[-1] % 8 == 0:
        if bias is not None and bias.dtype != x.dtype:        # O1 autocast: fp32 parameters next to bf16 activations
            bias = bias.to(x.dtype)
        return _BiasGeluFn.apply(x, bias, exact)
    return F.gelu(x if bias is None else x + bias, approximate="none" if exact else "tanh")


# =============================================================================== bias + dropout + residual
class _BiasDropoutAddFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, bias, residual, p, seed, offset):
        lib = _native.require()
        ctx.p, ctx.seed, ctx.offset = p, seed, offset
        ctx.has_bias, ctx.has_res = bias is not None, residual is not None
        _count()
        return lib.bias_dropout_add_fwd(x.contiguous(), bias, None if residual is None else residual.contiguous(), p, seed, offset)

    @staticmethod
    def backward(ctx, gy):
        lib = _native.require()
        gy = gy.contiguous()
        if ctx.p > 0:
            gx = lib.dropout_bwd(gy, ctx.p, ctx.seed, ctx.offset)   # mask regenerated from (seed, offset)
            _count()
        else:
            gx = gy
        gb = None
        if ctx.has_bias and ctx.needs_input_grad[1]:
            gb = lib.colsum(gx.view(-1, gx.shape[-1]), False)
            _count(2)
        return gx, gb, (gy if ctx.has_res else None), None, None, None


def bias_dropout_add(x: torch.Tensor, bias: Optional[torch.Tensor], residual: Optional[torch.Tensor], p: float,
                     training: bool, rng_name: Optional[str] = None) -> torch.Tensor:
    """``residual + dropout(x + bias)`` in one pass.  The CUDA path draws a Philox (seed, offset) from the
    named RNG stream and never materialises the mask."""
    p = float(p) if training else 0.0
    if _native_ok(x) and x.shape[-1] % 8 == 0:
        seed, offset = (0, 0)
        if p > 0:
            seed, offset = get_rng_state_tracker().philox(x.numel(), rng_name)
        if bias is not None and bias.dtype != x.dtype:        # the kernels read every operand in x's dtype
            bias = bias.to(x.dtype)
        if residual is not None and residual.dtype != x.dtype:
            residual = residual.to(x.dtype)
        return _BiasDropoutAddFn.apply(x, bias, residual, p, seed, offset)
    y = x if bias is None else x + bias
    if p > 0:
        if rng_name is not None:
            with get_rng_state_tracker().rng_state(rng_name):
                y = F.dropout(y, p, True)
        else:
            y = F.dropout(y, p, True)
    return y if residual is None else residual + y


def dropout(x: torch.Tensor, p: float, training: bool, rng_name: Optional[str] = None) -> torch.Tensor:
    if not training or p == 0:
        return x
    return bias_dropout_add(x, None, None, p, training, rng_name)


# =============================================================================== layer / rms norm
class _NormFn(torch.autograd.Function):
    """``with_res``: also hand the input back as a second output (an alias).  A pre-norm block takes its residual from THAT tensor, so
    the gradient of the residual branch arrives in this backward next to dy and the kernel writes ``norm_bwd(dy) + d_residual`` in one
    pass — otherwise autograd sums the two contributions with a separate full-size add (2 per transformer layer)."""

    @staticmethod
    def forward(ctx, x, weight, bias, eps, rms, with_res):
        lib = _native.require()
        x = x.contiguous()
        y, mean, rstd = lib.norm_fwd(x, weight, bias, eps, rms)
        _count()
        ctx.save_for_backward(x, weight, mean, rstd)
        ctx.rms, ctx.has_bias = rms, bias is not None
        if with_res:
            return y, x.view_as(x)
        return y

    @staticmethod
    def backward(ctx, gy, gres=None):
        lib = _native.require()
        x, weight, mean, rstd = ctx.saved_tensors
        if gy is None:            # only the residual alias was used
            return gres, None, None, None, None, None
        dx, dw, db = lib.norm_bwd(gy.contiguous(), x, weight, mean, rstd, ctx.rms, ctx.has_bias, None if gres is None else gres.contiguous())
        _count(3 if ctx.has_bias else 2)
        return dx, dw, (db if ctx.has_bias else None), None, None, None


def layer_norm(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], eps: float = 1e-5) -> torch.Tensor:
    if _native_ok(x, weight) and x.shape[-1] % 8 == 0 and x.shape[-1] <= 32768 and weight.dtype == x.dtype:
        return _NormFn.apply(x, weight, bias, eps, False, False)
    return F.layer_norm(x, (x.shape[-1],), weight, bias, eps)


def norm_with_residual(x: torch.Tensor, weight: torch.Tensor, bias: Optional[torch.Tensor], eps: float, rms: bool = False):
    """``(norm(x), x_res)`` for pre-norm blocks: use ``x_res`` (an alias of ``x``) as the residual operand and the backward adds the
    residual gradient inside the norm-backward kernel.  Falls back to ``(norm(x), x)`` off the native path."""
    if _native_ok(x, weight) and x.shape[-1] % 8 == 0 and x.shape[-1] <= 32768 and weight.dtype == x.dtype and torch.is_grad_enabled() and x.requires_grad:
        return _NormFn.apply(x, weight, bias, eps, rms, True)
    return (rms_norm(x, weight, eps) if rms else layer_norm(x, weight, bias, eps)), x


def rms_norm(x: torch.Tensor, weight: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    if _native_ok(x, weight) and x.shape[-1] % 8 == 0 and x.shape[-1] <= 32768 and weight.dtype == x.dtype:
        return _NormFn.apply(x, weight, None, eps, True, False)
    xf = x.float()
    return (xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + eps)).to(x.dtype) * weight


# =============================================================================== cross entropy
class _SoftmaxCEFn(torch.autograd.Function):
    """Per-token CE over (optionally vocab-sharded) logits.  fwd = one pass producing (max, sumexp, target);
    the three [tokens] vectors are all-reduced over the TP group; bwd rewrites the logits buffer in place."""

    @staticmethod
    def forward(ctx, logits, labels, group, vocab_start):
        import torch.distributed as dist

        lib = _native.require()
        l2 = logits.reshape(-1, logits.shape[-1])
        lab = labels.reshape(-1).contiguous()
        mx, sm, tg = lib.ce_stats(l2, lab, vocab_start)
        _count()
        pg = None if group is None else group.process_group
        if pg is not None and group.nranks > 1:
            gmx = mx.clone()
            dist.all_reduce(gmx, op=dist.ReduceOp.MAX, group=pg)
            sm = sm * torch.exp(mx - gmx)
            packed = torch.stack([sm, tg])
            dist.all_reduce(packed, group=pg)
            sm, tg, mx = packed[0], packed[1], gmx
        lse = mx + torch.log(sm)
        loss = lse - tg
        ctx.save_for_backward(l2, lab, lse)
        ctx.vocab_start = vocab_start
        ctx.shape = logits.shape
        return loss.view(labels.shape)

    @staticmethod
    def backward(ctx, gloss):
        lib = _native.require()
        l2, lab, lse = ctx.saved_tensors
        g = gloss.reshape(-1).float().contiguous()
        lib.ce_bwd_(l2, lab, lse, g, ctx.vocab_start)   # in place: logits buffer becomes dlogits
        _count()
        return l2.view(ctx.shape), None, None, None


def softmax_cross_entropy(logits: torch.Tensor, labels: torch.Tensor, group=None, vocab_start: int = 0) -> torch.Tensor:
    """Un-reduced CE, fp32, shape of ``labels``.  ``group``/``vocab_start`` describe a vocab-parallel shard
    (reference ParallelCrossEntropy, hybrid_model.py:951-996).  NOTE: the CUDA path consumes ``logits``
    (its storage is reused for the gradient)."""
    if _native_ok(logits) and logits.is_contiguous():
        return _SoftmaxCEFn.apply(logits, labels, group, vocab_start)
    return _softmax_ce_reference(logits, labels, group, vocab_start)


def _softmax_ce_reference(logits, labels, group, vocab_start):
    from ..parallel import comm_ops

    lf = logits.float()
    if group is None or group.nranks == 1:
        return F.cross_entropy(lf.reshape(-1, lf.shape[-1]), labels.reshape(-1), reduction="none").view(labels.shape)
    return _VocabParallelCEReference.apply(lf, labels, group, vocab_start)


class _VocabParallelCEReference(torch.autograd.Function):
    @staticmethod
    def forward(ctx, lf, labels, group, vocab_start):
        import torch.distributed as dist

        pg = group.process_group
        V = lf.shape[-1]
        mx = lf.max(-1).values
        dist.all_reduce(mx, op=dist.ReduceOp.MAX, group=pg)
        ex = torch.exp(lf - mx.unsqueeze(-1))
        sm = ex.sum(-1)
        dist.all_reduce(sm, group=pg)
        local = labels - vocab_start
        inside = (local >= 0) & (local < V)
        safe = local.clamp(0, V - 1)
        tg = torch.where(inside, lf.gather(-1, safe.unsqueeze(-1)).squeeze(-1), torch.zeros_like(mx))
        dist.all_reduce(tg, group=pg)
        lse = mx + sm.log()
        ctx.save_for_backward(ex / sm.unsqueeze(-1), safe, inside)
        return lse - tg

    @staticmethod
    def backward(ctx, g):
        probs, safe, inside = ctx.saved_tensors
        grad = probs.clone()
        grad.scatter_add_(-1, safe.unsqueeze(-1), -inside.to(grad.dtype).unsqueeze(-1))
        return grad * g.unsqueeze(-1), None, None, None


# =============================================================================== attention
def causal_softmax(scores: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    """softmax(scale * scores + causal mask) — reference ``softmax_mask_fuse_upper_triangle``."""
    if _native_ok(scores) and scores.is_contiguous():
        return _CausalSoftmaxFn.apply(scores, scale)
    sq, sk = scores.shape[-2:]
    mask = torch.ones(sq, sk, dtype=torch.bool, device=scores.device).triu(1 + sk - sq)
    return torch.softmax((scores.float() * scale).masked_fill(mask, float("-inf")), -1).to(scores.dtype)


class _CausalSoftmaxFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scores, scale):
        y = _native.require().causal_softmax_fwd(scores, scale)
        _count()
        ctx.save_for_backward(y)
        ctx.scale = scale
        return y

    @staticmethod
    def backward(ctx, gy):
        (y,) = ctx.saved_tensors
        _count()
        return _native.require().causal_softmax_bwd(gy.contiguous(), y, ctx.scale), None


def flash_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True, dropout_p: float = 0.0,
                    training: bool = True, scale: Optional[float] = None, attn_mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """q,k,v: [b, s, heads, d] -> [b, s, heads, d].  The fused kernel family lives in ops/attention.py; this
    wrapper picks it when available and otherwise calls the library SDPA (which counts as a library call)."""
    from . import attention as _attn

    return _attn.attention(q, k, v, causal=causal, dropout_p=dropout_p if training else 0.0, scale=scale, attn_mask=attn_mask)


# =============================================================================== rotary
class _RopeFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, positions, seq_len, base):
        ctx.save_for_backward(positions) if positions is not None else None
        ctx.has_pos, ctx.seq_len, ctx.base = positions is not None, seq_len, base
        _count()
        return _native.require().rope(x.contiguous(), positions, seq_len, base, False)

    @staticmethod
    def backward(ctx, gy):
        pos = ctx.saved_tensors[0] if ctx.has_pos else None
        _count()
        return _native.require().rope(gy.contiguous(), pos, ctx.seq_len, ctx.base, True), None, None, None


def rope(x: torch.Tensor, positions: Optional[torch.Tensor] = None, base: float = 10000.0) -> torch.Tensor:
    """NeoX-style rotary embedding on ``[b, s, heads, d]`` (new capability; the reference GPT uses learned
    absolute positions only)."""
    b, s, h, d = x.shape
    if x.is_cuda and _native.use_native(x):
        return _RopeFn.apply(x, positions, s, base)
    pos = (positions.reshape(b, s).float() if positions is not None else
           torch.arange(s, device=x.device, dtype=torch.float32).expand(b, s))
    inv = base ** (-torch.arange(0, d, 2, device=x.device, dtype=torch.float32) / d)
    ang = pos[..., None] * inv
    cs, sn = ang.cos()[:, :, None, :], ang.sin()[:, :, None, :]
    xf = x.float()
    x1, x2 = xf[..., : d // 2], xf[..., d // 2:]
    return torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], -1).to(x.dtype)


# =============================================================================== sampling
def topp_sampling(probs: torch.Tensor, top_ps: torch.Tensor, seed: int = -1, offset: Optional[int] = None
                  ) -> Tuple[torch.Tensor, torch.Tensor]:
    """Nucleus sampling: returns (prob[bs,1], id[bs,1]).  Semantics of the reference custom op
    (ppfleetx/ops/topp_sampling.cu:620-663): draw u ~ U(0,1) * top_p per row, walk the descending-sorted
    cumulative sum, first index with cumsum >= u wins."""
    bs = probs.shape[0]
    if probs.is_cuda and _native.use_native(probs):
        if seed < 0 or offset is None:
            seed, offset = get_rng_state_tracker().philox(bs * 4)
        _count()
        return tuple(_native.require().topp_sampling(probs.contiguous(), top_ps.reshape(-1), int(seed), int(offset)))
    gen = None
    if seed >= 0:
        gen = torch.Generator(device=probs.device)
        gen.manual_seed(int(seed) + int(offset or 0))
    sp, si = probs.float().sort(-1, descending=True)
    cum = sp.cumsum(-1)
    u = torch.rand(bs, 1, generator=gen, device=probs.device) * top_ps.reshape(-1, 1).float()
    pos = (cum >= u).float().argmax(-1, keepdim=True)
    return sp.gather(-1, pos).to(probs.dtype), si.gather(-1, pos)
