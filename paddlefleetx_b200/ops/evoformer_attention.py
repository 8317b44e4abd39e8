"""Evoformer gated attention (AlphaFold2 / HelixFold ``Attention``; reference ppfleetx/models/protein_folding/attentions.py:35-180).

    out[g, q, h, :] = softmax_k(scale * q.k + mask_bias[g, k] + pair_bias[g // groups_per_pair, h, q, k]) @ v * sigmoid(gate)

Forward: one wgmma kernel (``csrc/evoformer_attn_sm90.cu``) — logits, both biases, softmax, P V and the gate never leave the chip; only the
output and two row statistics (the row maximum and log2 of the row sum, kept apart so that rows whose keys all carry the -1e9 padding bias
keep their 1 / Sk probabilities) are written.  Backward: a second wgmma kernel recomputes the probabilities per tile from (q, k, biases,
statistics) and produces dq / dk / dv / dgate and the pair-bias gradient (fp32 reductions over the groups that share a bias); nothing of size
[g, h, q, k] is ever stored (the reference keeps logits, probabilities and the gated average of all 48 blocks x 6 attentions alive).
``PFX_EVO_BWD=torch`` selects the older chunked recomputation with library matmuls (also used when the mask bias needs a gradient).

CPU / unsupported shapes fall back to the plain PyTorch expression, which is also the numerics reference of the tests.
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from . import _native

_CHUNK_ELEMS = 1 << 27          # probabilities materialised per backward chunk (fp32 elements)
_BWD = os.environ.get("PFX_EVO_BWD", "native")      # "native" = wgmma backward kernel, "torch" = chunked recomputation with library matmuls


def reference(q, k, v, mask_bias, pair_bias, gate, groups_per_pair: int, scale: float):
    """The plain expression over [G, S, H, D] operands (any device), in fp32 — or in the inputs' own precision when that is wider."""
    G, Sq, H, D = q.shape
    ct = torch.promote_types(q.dtype, torch.float32)
    logits = torch.einsum("gqhd,gkhd->ghqk", q.to(ct), k.to(ct)) * scale
    if mask_bias is not None:
        logits = logits + mask_bias.to(ct).view(G, 1, 1, -1)
    if pair_bias is not None:
        logits = logits + pair_bias.to(ct).repeat_interleave(groups_per_pair, dim=0)
    p = torch.softmax(logits, dim=-1)
    o = torch.einsum("ghqk,gkhd->gqhd", p, v.to(ct))
    if gate is not None:
        o = o * torch.sigmoid(gate.to(ct))
    return o


def supported(q: torch.Tensor, k: torch.Tensor) -> bool:
    return (q.is_cuda and q.dtype == torch.bfloat16 and q.dim() == 4 and q.shape[-1] == 32 and q.shape[2] % 2 == 0
            and _native.use_native(q) and k.shape[1] >= 1)


class _EvoAttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, mask_bias, pair_bias, gate, groups_per_pair, scale):
        lib = _native.require()
        q, k, v = q.contiguous(), k.contiguous(), v.contiguous()
        mb = None if mask_bias is None else mask_bias.float().contiguous()
        pb = None if pair_bias is None else pair_bias.to(torch.bfloat16).contiguous()
        gt = None if gate is None else gate.contiguous()
        out, stats = lib.evoformer_attention_fwd(q, k, v, mb, pb, gt, groups_per_pair, scale)
        ctx.save_for_backward(q, k, v, mb if mb is not None else q.new_empty(0), pb if pb is not None else q.new_empty(0),
                              gt if gt is not None else q.new_empty(0), stats, out)
        ctx.flags = (mask_bias is not None, pair_bias is not None, gate is not None)
        ctx.gpp, ctx.scale = groups_per_pair, scale
        ctx.bias_dtypes = (None if mask_bias is None else mask_bias.dtype, None if pair_bias is None else pair_bias.dtype)
        return out

    @staticmethod
    def backward(ctx, dout):
        """Gradients of the gated attention w.r.t. q / k / v, the two additive biases and the gate: the native kernel recomputes the probabilities
        from the saved row statistics tile by tile (dK / dV in tensor memory, dQ through an fp32 workspace); bias gradients are reduced over the axes
        the biases were broadcast along."""
        q, k, v, mb, pb, gt, stats = ctx.saved_tensors[:7]
        has_mb, has_pb, has_gate = ctx.flags
        gpp, scale = ctx.gpp, ctx.scale
        G, Sq, H, D = q.shape
        Sk = k.shape[1]
        dout = dout.contiguous()
        need_mb = has_mb and ctx.needs_input_grad[3]
        if _BWD == "native" and q.is_cuda and len(ctx.saved_tensors) == 8 and not need_mb:
            # one wgmma kernel (csrc/evoformer_attn_sm90.cu): five products per (group, head, key tile), pair-bias gradient by fp32 reds
            lib = _native.require()
            out = ctx.saved_tensors[7]
            need_pb = has_pb and ctx.needs_input_grad[4]
            dq, dk, dv, dgate, dpair = lib.evoformer_attention_bwd(q, k, v, out, dout, stats, mb if has_mb else None, pb if has_pb else None,
                                                                   gt if has_gate else None, gpp, scale, need_pb)
            mb_dt, pb_dt = ctx.bias_dtypes
            return (dq, dk, dv, None, dpair.to(pb_dt) if need_pb else None, dgate if has_gate else None, None, None)
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        dgate = torch.empty_like(gt) if has_gate else None
        need_pb = has_pb and ctx.needs_input_grad[4]
        need_mb = has_mb and ctx.needs_input_grad[3]
        dpb = torch.zeros(G // gpp, H, Sq, Sk, dtype=torch.float32, device=q.device) if need_pb else None
        dmb = torch.zeros(G, Sk, dtype=torch.float32, device=q.device) if need_mb else None
        # chunks of whole pair-bias groups: the bias gradient of a chunk is a plain sum over its groups
        per_group = H * Sq * Sk
        groups = max(_CHUNK_ELEMS // max(per_group, 1), 1)
        step = max(groups // gpp, 1) * gpp if groups >= gpp else groups
        if step < gpp:
            while gpp % step:
                step -= 1
        for g0 in range(0, G, step):
            g1 = min(g0 + step, G)
            sl = slice(g0, g1)
            qc, kc, vc = q[sl], k[sl], v[sl]
            # fp32 products: a 16-bit q.k rounds every logit by 2^-8 relative, which exp() turns into a probability error of about 1 %
            logits = torch.einsum("gqhd,gkhd->ghqk", qc.float(), kc.float()) * scale
            if has_mb:
                logits += mb[sl].view(g1 - g0, 1, 1, Sk)
            if has_pb:
                idx = torch.arange(g0, g1, device=q.device) // gpp
                logits += pb.index_select(0, idx).float()
            # softmax of the recomputed logits, not exp(logits - lse): on a row whose keys all carry -1e9 the fp32 logits are all equal and
            # their log-sum-exp loses log(Sk) to rounding
            p = torch.softmax(logits, -1)                                       # [g, h, q, k] fp32, rows sum to 1
            del logits
            pb16 = p.to(q.dtype)                                                # matmul operands in the activations' dtype
            do = dout[sl]
            if has_gate:
                o = torch.einsum("ghqk,gkhd->gqhd", pb16, vc).float()
                sig = torch.sigmoid(gt[sl].float())
                dgate[sl] = (do.float() * o * sig * (1 - sig)).to(dgate.dtype)
                do = (do.float() * sig).to(q.dtype)
                del o, sig
            dv[sl] = torch.einsum("ghqk,gqhd->gkhd", pb16, do)
            dp = torch.einsum("gqhd,gkhd->ghqk", do, vc).float()
            ds = p * (dp - (dp * p).sum(-1, keepdim=True))
            del dp, p, pb16
            if need_pb:
                if step >= gpp:
                    dpb[g0 // gpp:(g1 + gpp - 1) // gpp] += ds.view(-1, gpp, H, Sq, Sk).sum(1)
                else:
                    dpb[g0 // gpp] += ds.sum(0)
            if need_mb:
                dmb[sl] = ds.sum((1, 2))
            ds16 = (ds * scale).to(q.dtype)
            del ds
            dq[sl] = torch.einsum("ghqk,gkhd->gqhd", ds16, kc)
            dk[sl] = torch.einsum("ghqk,gqhd->gkhd", ds16, qc)
        mb_dt, pb_dt = ctx.bias_dtypes
        return (dq, dk, dv, None if dmb is None else dmb.to(mb_dt), None if dpb is None else dpb.to(pb_dt), dgate, None, None)


def evoformer_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, mask_bias: Optional[torch.Tensor] = None,
                        pair_bias: Optional[torch.Tensor] = None, gate: Optional[torch.Tensor] = None, groups_per_pair: int = 1,
                        scale: Optional[float] = None) -> torch.Tensor:
    """``q`` [G, Sq, H, D], ``k`` / ``v`` [G, Sk, H, D]; ``mask_bias`` [G, Sk]; ``pair_bias`` [G // groups_per_pair, H, Sq, Sk];
    ``gate`` [G, Sq, H, D] (pre-sigmoid).  Returns [G, Sq, H, D] in ``q``'s dtype."""
    scale = float(q.shape[-1]) ** -0.5 if scale is None else float(scale)
    if supported(q, k):
        return _EvoAttnFn.apply(q, k, v, mask_bias, pair_bias, gate, int(groups_per_pair), scale)
    return reference(q, k, v, mask_bias, pair_bias, gate, int(groups_per_pair), scale).to(q.dtype)
