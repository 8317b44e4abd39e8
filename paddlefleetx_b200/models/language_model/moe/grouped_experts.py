"""Grouped expert FFN: every local expert's ``h -> 4h -> GELU -> h`` (or SwiGLU: ``h -> 2F gate / up pairs -> F -> h``) in FOUR kernel
launches forward (tile table, FFN1 with the dual pre-activation / activation epilogue, FFN2) and seven backward, for any number of experts
and any routing — no per-expert loop, no host round trip.

The reference runs its experts as a Python loop over ``fwd_expert_count.numpy()`` slices (moe/moe_layer.py:195-208), i.e. one
device->host copy per MoE layer per pass plus ``num_expert`` small GEMM launches.  Here the dispatch kernel leaves the routed tokens
expert-major in a fixed-capacity buffer together with a segment table IN DEVICE MEMORY; ``moe_tile_table`` turns that table into a
per-row-block expert index, and the tcgen05 GEMM (``gemm_sm100.cu``, ``GemmGroup``) picks its B slice (the stacked expert weights),
its bias slice, or — for the weight gradient — its K range from the table while it runs.  Row blocks past the routed rows are skipped
by the tile loop itself.

The experts' weights live in four stacked parameters (``GroupedExperts``) so that the kernel sees ``[E, out, in]`` behind one tensor
map; the expert modules keep working on slices of them and checkpoints keep the per-expert names.
"""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

from ....ops import _native

EPI_NONE, EPI_BIAS, EPI_BIAS_GELU_DUAL, EPI_DGELU, EPI_BIAS_SWIGLU_DUAL, EPI_DSWIGLU = 0, 1, 4, 5, 6, 7


class GroupedExperts(nn.Module):
    """Owns the parameters of ``E`` structurally identical expert FFNs as four stacked tensors ``w1 [E, 4h, h]``, ``b1 [E, 4h]``,
    ``w2 [E, h, 4h]``, ``b2 [E, h]`` (SwiGLU experts: ``w1 [E, 2F, h]``, ``b1 [E, 2F]``, ``w2 [E, h, F]``) — what the grouped GEMM
    addresses with one tensor map.  The expert modules it was built from lose
    their own parameters and see slices of the stacks instead (``bind_views``), so ``experts[e](x)`` keeps working (fallback loop,
    tests) and gradients of either path land in the same stacked ``.grad``.  Checkpoints keep the per-expert names
    (``experts.{e}.htoh4.weight`` ...) through the state-dict hooks of :class:`MoELayer`."""

    NAMES = (("w1", "htoh4", "weight"), ("b1", "htoh4", "bias"), ("w2", "h4toh", "weight"), ("b2", "h4toh", "bias"))

    def __init__(self, experts: List[nn.Module]):
        super().__init__()
        assert self.supported(experts)
        self.activation = getattr(experts[0], "activation", "gelu")
        for stacked, lin, attr in self.NAMES:
            t = torch.stack([getattr(getattr(ex, lin), attr).data for ex in experts]).contiguous()
            par = nn.Parameter(t)
            par.is_expert = True
            par.no_sync = True
            if attr == "bias":
                par.no_weight_decay = True      # a stacked bias is 2-D and is not called "...bias": keep it out of weight decay like the per-expert biases
            setattr(self, stacked, par)
        for ex in experts:                      # the stacks are the parameters now
            for _, lin, attr in self.NAMES:
                del getattr(ex, lin)._parameters[attr]
        object.__setattr__(self, "_experts", list(experts))      # not a submodule: MoELayer.experts already registers them
        self.bind_views()

    @staticmethod
    def supported(experts) -> bool:
        if not experts:
            return False
        for ex in experts:
            if not (isinstance(getattr(ex, "htoh4", None), nn.Linear) and isinstance(getattr(ex, "h4toh", None), nn.Linear)):
                return False
            if ex.htoh4._parameters.get("bias") is None or ex.h4toh._parameters.get("bias") is None or ex.htoh4._parameters.get("weight") is None:
                return False
        a = experts[0]
        act = getattr(a, "activation", "gelu")
        same = all(ex.htoh4.weight.shape == a.htoh4.weight.shape and ex.h4toh.weight.shape == a.h4toh.weight.shape
                   and ex.htoh4.weight.dtype == a.htoh4.weight.dtype and getattr(ex, "activation", "gelu") == act for ex in experts)
        d_hidden, d_model = a.htoh4.weight.shape
        if act == "swiglu":      # htoh4 [2F, h] of gate / up pairs, h4toh [h, F]
            ffn = a.h4toh.weight.shape[1]
            return same and d_model % 128 == 0 and ffn % 128 == 0 and d_hidden == 2 * ffn
        return same and act == "gelu" and d_model % 128 == 0 and d_hidden % 128 == 0

    def bind_views(self):
        """(Re-)attach differentiable slices of the stacks to the expert modules (cheap; call before using ``experts[e]`` directly)."""
        for e, ex in enumerate(self._experts):
            for stacked, lin, attr in self.NAMES:
                object.__setattr__(getattr(ex, lin), attr, getattr(self, stacked)[e])

    @property
    def num_expert(self) -> int:
        return self.w1.shape[0]

    # ---- checkpoint names stay per expert (reference layout: experts.{e}.htoh4.weight, ...)
    def split_state(self, state_dict, prefix: str, experts_prefix: str):
        for stacked, lin, attr in self.NAMES:
            t = state_dict.pop(prefix + stacked)
            for e in range(t.shape[0]):
                state_dict[f"{experts_prefix}{e}.{lin}.{attr}"] = t[e]

    def merge_state(self, state_dict, prefix: str, experts_prefix: str):
        for stacked, lin, attr in self.NAMES:
            keys = [f"{experts_prefix}{e}.{lin}.{attr}" for e in range(self.num_expert)]
            if all(k in state_dict for k in keys):
                state_dict[prefix + stacked] = torch.stack([state_dict.pop(k) for k in keys])


class GroupedFFN(torch.autograd.Function):
    """``ys[rows of e] = act(xs W1[e]^T + b1[e]) W2[e]^T + b2[e]`` over an expert-major, block-aligned row buffer, with ``act`` the tanh GELU
    or the SwiGLU of the pair-interleaved FFN1 output (``activation``).  Either way FFN1 saves its pre-activation ``pre`` for the backward.

    ``xs`` is the whole fixed-capacity buffer; ``tile_group`` / ``seg2`` (device tensors) say which blocks carry rows.  Rows of ``pre``,
    ``h`` and the outputs in blocks no expert owns are never written, and padded rows inside an expert's block are never read downstream."""

    @staticmethod
    def forward(ctx, xs, tile_group, seg2, w1, b1, w2, b2, staging, row_align, recompute_h, activation="gelu"):
        lib = _native.require()
        swiglu = activation == "swiglu"
        rows, ffn1 = xs.shape[0], w1.shape[1]
        pre = torch.empty(rows, ffn1, dtype=xs.dtype, device=xs.device)
        h = torch.empty(rows, w2.shape[2], dtype=xs.dtype, device=xs.device)
        lib.gemm_grouped(xs, w1, b1, tile_group, pre, True, EPI_BIAS_SWIGLU_DUAL if swiglu else EPI_BIAS_GELU_DUAL, h, None, row_align)
        # ``staging`` (a MoEDispatcher or None): its ``stage_out`` buffer is where the combine kernel's peers pull from, so FFN2 (and dX in
        # the backward) write there directly; a fresh view object keeps autograd's bookkeeping off the persistent tensor
        ys = staging.stage_out[:rows] if staging is not None else torch.empty_like(xs)
        lib.gemm_grouped(h, w2, b2, tile_group, ys, True, EPI_BIAS, None, None, row_align)
        ctx.row_align, ctx.staging, ctx.recompute_h, ctx.swiglu = row_align, staging, recompute_h, swiglu
        ctx.save_for_backward(xs, tile_group, seg2, pre, h if not recompute_h else pre.new_empty(0), w1, w2)
        return ys

    @staticmethod
    def backward(ctx, g_ys):
        lib = _native.require()
        align = ctx.row_align
        xs, tile_group, seg2, pre, h, w1, w2 = ctx.saved_tensors
        E = w1.shape[0]
        g_ys = g_ys.contiguous()
        if ctx.recompute_h:          # trade the [rows, F] activation for one elementwise pass
            h = lib.bias_swiglu_fwd(pre, None) if ctx.swiglu else torch.nn.functional.gelu(pre, approximate="tanh")
        # FFN2: dW2[e] = dY_e^T H_e, db2[e] = colsum(dY_e), dPre = act'(pre) applied to dY W2[e]
        dw2 = torch.empty_like(w2)
        lib.gemm_grouped_wgrad(g_ys, h, seg2, dw2)
        db2 = lib.grouped_colsum(g_ys, seg2, E)
        dpre = torch.empty_like(pre)
        lib.gemm_grouped(g_ys, w2, None, tile_group, dpre, False, EPI_DSWIGLU if ctx.swiglu else EPI_DGELU, None, pre, align)
        del h
        # FFN1: dW1[e] = dPre_e^T X_e, db1[e] = colsum(dPre_e), dX = dPre W1[e]
        dw1 = torch.empty_like(w1)
        lib.gemm_grouped_wgrad(dpre, xs, seg2, dw1)
        db1 = lib.grouped_colsum(dpre, seg2, E)
        dxs = None
        if ctx.needs_input_grad[0]:
            dxs = ctx.staging.stage_out[:xs.shape[0]] if ctx.staging is not None else torch.empty_like(xs)
            lib.gemm_grouped(dpre, w1, None, tile_group, dxs, False, EPI_NONE, None, None, align)
        return dxs, None, None, dw1, db1, dw2, db2, None, None, None, None


def grouped_ffn(xs, tile_group, seg2, ge: GroupedExperts, staging=None, row_align: int = 128, recompute_h: bool = False):
    return GroupedFFN.apply(xs, tile_group, seg2, ge.w1, ge.b1, ge.w2, ge.b2, staging, row_align, recompute_h, ge.activation)


def reference_grouped_ffn(xs, seg2_host, ge: GroupedExperts):
    """Plain per-expert loop over the same layout (tests), in fp32 or, for float64 inputs, in float64: rows outside the segments stay zero."""
    F = torch.nn.functional
    dt = torch.float64 if xs.dtype == torch.float64 else torch.float32
    out = torch.zeros_like(xs, dtype=dt)
    for e in range(ge.num_expert):
        s, n = seg2_host[2 * e], seg2_host[2 * e + 1]
        if n:
            pre = F.linear(xs[s:s + n].to(dt), ge.w1[e].to(dt), ge.b1[e].to(dt))
            if ge.activation == "swiglu":      # column 2i gate channel i, 2i + 1 its up channel
                hcur = F.silu(pre[:, 0::2]) * pre[:, 1::2]
            else:
                hcur = F.gelu(pre, approximate="tanh")
            out[s:s + n] = F.linear(hcur, ge.w2[e].to(dt), ge.b2[e].to(dt))
    return out
