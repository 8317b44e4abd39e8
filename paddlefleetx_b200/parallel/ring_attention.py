"""Ring attention: context parallelism without a head-count limit (``Distributed.cp_mode: ring``).

Beyond the reference (SURVEY 2.3 lists CP / ring attention as absent, F4).  Ulysses (``comm_ops.seq_head_all_to_all``) trades sequence shards
for head shards and therefore stops at ``cp <= heads / mp``; the ring keeps every head on every rank and passes K / V blocks round the
context-parallel group instead, so the context length scales with the number of ranks whatever the head count.

Layout.  The sequence is cut into ``2c`` chunks and rank ``r`` holds chunks ``r`` and ``2c - 1 - r`` (``zigzag_slice``).  Under a causal mask
every rank then does the same amount of work at every ring step — with contiguous slices the last rank would attend to ``c`` blocks while the
first attends to one, and the step time is the maximum:

  * step 0 (own K / V):          ordinary causal attention over the local ``s / c`` positions (the two chunks are in ascending order);
  * block from a rank ``j < r``: all local queries see its FIRST chunk, none see its second  ->  ``q x k[:half]``, unmasked;
  * block from a rank ``j > r``: only the local SECOND chunk sees it, and sees all of it     ->  ``q[half:] x k``, unmasked.

Every block is one call of the flash kernels (``csrc/attention_fwd_sm90.cu`` returns the row log-sum-exp, ``attention_bwd_sm90.cu`` takes
the FINAL log-sum-exp and output, which is all a block's backward needs: ``P = exp(S - lse)``, ``delta = rowsum(dO o O)``); partial outputs
are merged with the usual online-softmax rescaling in fp32.  The transfer of the next block is posted before the current block is computed
(``batch_isend_irecv``: NCCL p2p on its own internal stream on CUDA, gloo on CPU), so the exchange hides behind the attention math.  In the
backward the ``dK / dV`` accumulators (fp32) travel with their K / V block and arrive home after ``c`` steps.

CPU tensors, other dtypes and head sizes run the same schedule on a plain PyTorch block (used by the gloo parity tests).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.distributed as dist

from ..ops import attention as ATT


def zigzag_slice(t: torch.Tensor, c: int, r: int, dim: int = 1) -> torch.Tensor:
    """Chunks ``r`` and ``2c - 1 - r`` of ``t`` cut into ``2c`` pieces along ``dim`` — this rank's part of the sequence."""
    assert t.shape[dim] % (2 * c) == 0, f"sequence length {t.shape[dim]} must be a multiple of 2 x cp_degree = {2 * c}"
    parts = t.chunk(2 * c, dim=dim)
    return torch.cat([parts[r], parts[2 * c - 1 - r]], dim=dim)


def local_positions(s_local: int, c: int, r: int, mode: str, device=None) -> torch.Tensor:
    """Global positions ``[s_local]`` of rank ``r``'s sequence shard when the data carries the default ``0 .. s-1`` position ids: a contiguous
    slice (Ulysses) or the two zigzag chunks (ring).  Used where position ids do not travel with the activations (pipeline stages > 0)."""
    if mode == "ring":
        half = s_local // 2
        a = torch.arange(half, device=device)
        return torch.cat([r * half + a, (2 * c - 1 - r) * half + a])
    return r * s_local + torch.arange(s_local, device=device)


def zigzag_merge(parts, dim: int = 1) -> torch.Tensor:
    """Inverse of ``zigzag_slice`` over the rank-ordered list of local tensors."""
    c = len(parts)
    halves = [p.chunk(2, dim=dim) for p in parts]
    return torch.cat([h[0] for h in halves] + [halves[c - 1 - i][1] for i in range(c)], dim=dim)


# ---------------------------------------------------------------------------------------------------------------------------------------
# one block: (out, lse) forward, (dq, dk, dv) backward
def _keep_mask(seed: int, q: torch.Tensor, k: torch.Tensor, p: float):
    return ATT.attn_keep_mask(seed, q.shape[0], q.shape[2], q.shape[1], k.shape[1], p, q.device)


def _math_dtype(t: torch.Tensor) -> torch.dtype:
    return torch.float64 if t.dtype == torch.float64 else torch.float32


def _block_fwd(q, k, v, causal: bool, scale: float, dropout_p: float, seed: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """``[b, sq, h, d] x [b, sk, h, d]`` -> output ``[b, sq, h, d]`` (math dtype on the fallback, bf16 from the kernels) and the natural
    log-sum-exp of the scaled scores ``[b, h, sq]``."""
    if ATT._native_ok(q, k, v, None, causal, False):
        from ..ops import _native
        from ..ops import functional as OF

        out, lse = _native.require().attention_fwd_v2(q, k, v, bool(causal), float(scale), float(dropout_p), int(seed))
        OF._count()
        return out, lse
    md = _math_dtype(q)
    s = torch.einsum("bqhd,bkhd->bhqk", q.to(md), k.to(md)) * scale
    if causal:
        sq, sk = s.shape[-2:]
        s = s.masked_fill(torch.ones(sq, sk, dtype=torch.bool, device=s.device).triu(1 + sk - sq), float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - lse.unsqueeze(-1))
    if dropout_p > 0:
        p = p * _keep_mask(seed, q, k, dropout_p).to(md) / (1.0 - dropout_p)
    return torch.einsum("bhqk,bkhd->bqhd", p, v.to(md)), lse


def _block_bwd(q, k, v, out, dout, lse, causal: bool, scale: float, dropout_p: float, seed: int):
    """Gradients of one block given the FINAL output / log-sum-exp of its query rows."""
    if ATT._native_ok(q, k, v, None, causal, True) and out.dtype == q.dtype:
        from ..ops import _native
        from ..ops import functional as OF

        if dout.stride(3) != 1 or any(dout.stride(i) % 8 for i in range(3)):
            dout = dout.contiguous()
        dq, dk, dv = (torch.empty_like(t, memory_format=torch.contiguous_format) for t in (q, k, v))
        _native.require().attention_bwd(q, k, v, out, dout, lse.contiguous(), dq, dk, dv, bool(causal), float(scale), float(dropout_p), int(seed))
        OF._count(4)
        return dq, dk, dv
    md = _math_dtype(q)
    qf, kf, vf, of, do = (t.to(md) for t in (q, k, v, out, dout))
    s = torch.einsum("bqhd,bkhd->bhqk", qf, kf) * scale
    if causal:
        sq, sk = s.shape[-2:]
        s = s.masked_fill(torch.ones(sq, sk, dtype=torch.bool, device=s.device).triu(1 + sk - sq), float("-inf"))
    p = torch.exp(s - lse.to(md).unsqueeze(-1))                      # probabilities against the GLOBAL normaliser
    dp = torch.einsum("bqhd,bkhd->bhqk", do, vf)
    if dropout_p > 0:
        keep = _keep_mask(seed, q, k, dropout_p).to(md) / (1.0 - dropout_p)
        dv = torch.einsum("bhqk,bqhd->bkhd", p * keep, do)
        dp = dp * keep
    else:
        dv = torch.einsum("bhqk,bqhd->bkhd", p, do)
    delta = (do * of).sum(-1).permute(0, 2, 1).unsqueeze(-1)         # [b, h, sq, 1]
    ds = p * (dp - delta) * scale
    return torch.einsum("bhqk,bkhd->bqhd", ds, kf), torch.einsum("bhqk,bqhd->bkhd", ds, qf), dv


def _merge(acc_out, acc_lse, out, lse):
    """Online-softmax merge of a new partial result into the accumulator (both over the same query rows); fp32 / fp64 state."""
    if acc_out is None:
        return out.to(_math_dtype(out)), lse.clone()
    new = torch.logaddexp(acc_lse, lse)
    wa = torch.exp(acc_lse - new).permute(0, 2, 1).unsqueeze(-1)      # [b, sq, h, 1]
    wb = torch.exp(lse - new).permute(0, 2, 1).unsqueeze(-1)
    return acc_out * wa + out.to(acc_out.dtype) * wb, new


# ---------------------------------------------------------------------------------------------------------------------------------------
class _Ring:
    """Neighbour exchange inside a ``_Group``: ``post`` starts sending ``tensors`` to the next rank and receiving the previous rank's into
    fresh buffers, ``wait`` returns those buffers.  Send buffers stay referenced until ``wait``."""

    def __init__(self, group):
        self.pg = group.process_group
        self.next = group.ranks[(group.rank + 1) % group.nranks]
        self.prev = group.ranks[(group.rank - 1) % group.nranks]
        self._pending = None

    def post(self, tensors):
        send = [t.contiguous() for t in tensors]
        recv = [torch.empty_like(t) for t in send]
        ops = [dist.P2POp(dist.isend, t, self.next, self.pg) for t in send] + [dist.P2POp(dist.irecv, t, self.prev, self.pg) for t in recv]
        self._pending = (dist.batch_isend_irecv(ops), send, recv)

    def wait(self):
        reqs, _send, recv = self._pending
        for r in reqs:
            r.wait()
        self._pending = None
        return recv


def _block_plan(causal: bool, r: int, src: int, half: int):
    """Which query rows meet which key rows when rank ``r`` holds the block of rank ``src``: ``(q_slice, k_slice, causal_in_block)`` or ``None``
    for the unmasked non-causal case handled by the caller."""
    if not causal or src == r:
        return slice(None), slice(None), causal
    if src < r:
        return slice(None), slice(0, half), False
    return slice(half, None), slice(None), False


def _block_seed(seed: int, r: int, src: int) -> int:
    """A distinct dropout stream per (query rank, key rank) pair, the same in forward and backward."""
    return (seed + 0x632BE59BD9B4E019 * (1 + r * 64 + src)) & 0x7FFFFFFFFFFFFFFF if seed else 0


class _RingAttnFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, q, k, v, group, causal, scale, dropout_p, seed):
        c, r = group.nranks, group.rank
        half = q.shape[1] // 2
        ring = _Ring(group)
        out = lse = None
        kv = (k, v)
        for step in range(c):
            src = (r - step) % c                                       # whose K / V we hold at this step
            if step + 1 < c:
                ring.post(kv)
            qs, ks, blk_causal = _block_plan(causal, r, src, half)
            o_b, l_b = _block_fwd(q[:, qs], kv[0][:, ks], kv[1][:, ks], blk_causal, scale, dropout_p, _block_seed(seed, r, src))
            if qs == slice(None):
                out, lse = _merge(out, lse, o_b, l_b)
            else:                                                      # only the second local chunk sees this block (never at step 0)
                o2, l2 = _merge(out[:, qs], lse[:, :, qs], o_b, l_b)
                out = torch.cat([out[:, :half], o2], dim=1)
                lse = torch.cat([lse[:, :, :half], l2], dim=2)
            if step + 1 < c:
                kv = ring.wait()
        out = out.to(q.dtype)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.cfg = (group, causal, scale, dropout_p, seed)
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        group, causal, scale, dropout_p, seed = ctx.cfg
        c, r = group.nranks, group.rank
        half = q.shape[1] // 2
        md = _math_dtype(q)
        ring_kv, ring_d = _Ring(group), _Ring(group)                   # every rank posts in the same order (kv, d, kv, d, ...): pairs match up
        dq = torch.zeros(q.shape, dtype=md, device=q.device)
        kv = (k, v)
        dkv = (torch.zeros(k.shape, dtype=md, device=k.device), torch.zeros(v.shape, dtype=md, device=v.device))
        for step in range(c):
            src = (r - step) % c
            if step + 1 < c:
                ring_kv.post(kv)                                       # the NEXT block's K / V travel while this block's gradients are computed
            qs, ks, blk_causal = _block_plan(causal, r, src, half)
            g_q, g_k, g_v = _block_bwd(q[:, qs], kv[0][:, ks], kv[1][:, ks], out[:, qs], dout[:, qs], lse[:, :, qs], blk_causal, scale, dropout_p,
                                       _block_seed(seed, r, src))
            if step > 0:
                dkv = tuple(ring_d.wait())                             # this block's accumulator, sent by the previous rank after ITS last step
            dq[:, qs] += g_q.to(md)
            dkv[0][:, ks] += g_k.to(md)
            dkv[1][:, ks] += g_v.to(md)
            if step + 1 < c:
                kv = ring_kv.wait()
            ring_d.post(dkv)                                           # the accumulators follow their block; the last hop brings them home
        dkv = ring_d.wait()
        return dq.to(q.dtype), dkv[0].to(k.dtype), dkv[1].to(v.dtype), None, None, None, None, None


def ring_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, group, causal: bool = True, dropout_p: float = 0.0,
                   scale: Optional[float] = None) -> torch.Tensor:
    """Attention over a sequence sharded across ``group`` in the zigzag layout: ``q / k / v`` are this rank's ``[b, s / c, heads, d]``."""
    sc = float(scale if scale is not None else q.shape[-1] ** -0.5)
    if group is None or group.nranks == 1:
        return ATT.attention(q, k, v, causal=causal, dropout_p=dropout_p, scale=sc)
    assert q.shape[1] % 2 == 0 and q.shape == k.shape == v.shape, "ring attention takes equally sized zigzag shards of q, k and v"
    seed = ATT._dropout_seed(dropout_p, q.shape[0] * q.shape[2] * q.shape[1] * k.shape[1])
    return _RingAttnFn.apply(q, k, v, group, bool(causal), sc, float(dropout_p), seed)
