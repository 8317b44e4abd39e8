"""GPT model family: one implementation for single-card, tensor-parallel, sequence-parallel and MoE runs.

Capabilities mirrored from the reference (single-card ``gpt/dygraph/single_model.py:56-1419`` and hybrid
``gpt/dygraph/hybrid_model.py:90-1000``):
  * pre-LN decoder, fused or split QKV, tanh-GELU FFN, learned absolute positions, tied LM head,
  * ``scale_qk_by_layer_num`` (scores computed as (q/(L*sqrt(d))) k^T then *L — hybrid_model.py:310-315),
  * flash attention or unfused ``QK^T -> fused causal softmax -> PV`` core attention,
  * recompute granularities ``full | full_attn | core_attn`` and ``no_recompute_layers``,
  * Megatron TP (+ sequence parallel in ``[s, b, h]`` layout) through ``parallel/tp_layers.py``,
  * KV cache for generation, sequence-classification head, masked-mean pre-training criterion,
  * optional MoE FFN per layer (``moe_configs``).

State-dict keys keep the reference's structured names (SURVEY §5.4), e.g.
``gpt.decoder.layers.3.self_attn.qkv_proj.weight``; linear weights are stored ``[out, in]`` (torch) instead
of Paddle's ``[in, out]`` — ``utils/ckpt_convert.py`` transposes when importing genuine Paddle checkpoints.
The fused-QKV output dimension is laid out ``[heads, 3, head_dim]`` like the reference.  With grouped-query attention
(``num_key_value_heads`` = Hkv < heads, G = heads / Hkv query heads per K/V head) it is ``[Hkv, G + 2, head_dim]``: the G query heads of
a group, then its key, then its value.  G = 1 is the ``[heads, 3, head_dim]`` layout, and because the layout splits by whole groups
along the output rows, tensor parallelism shards it like any column-parallel weight when ``Hkv % mp == 0``.
With ``ffn_activation="swiglu"`` the FFN is h = silu(x W_g + b_g) * (x W_u + b_u) of width F = ``ffn_hidden_size``, and ``linear1`` is
``[2F, H]`` with pair-interleaved rows: row 2i is gate channel i, row 2i + 1 its up channel (the bias likewise).  A contiguous
column-parallel shard then holds whole pairs, so tensor parallelism and checkpoint resharding split ``linear1`` as before.
With ``reset_attention_mask`` a sample packed from several documents attends within each document only: ``GPTModel.forward`` builds
one ``DocumentMask`` from the position ids (which restart at 0 at each document start) and every layer receives it as ``attn_mask``.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import torch
import torch.nn as nn

from ....ops import attention as ATT
from ....ops import functional as OF
from ....parallel import comm_ops as C
from ....parallel.recompute import recompute
from ....parallel.rng import get_rng_state_tracker
from ....parallel.tp_layers import _OPTIONS as _TP_OPTIONS
from ....parallel.tp_layers import (ColumnParallelLinear, ColumnSequenceParallelLinear, ParallelCrossEntropy,
                                    RowParallelLinear, RowSequenceParallelLinear, VocabParallelEmbedding,
                                    mark_as_sequence_parallel_parameter, parallel_matmul)


class LayerNorm(nn.Module):
    def __init__(self, hidden: int, eps: float = 1e-5, sequence_parallel: bool = False, dtype=None, device=None):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden, dtype=dtype, device=device))
        self.bias = nn.Parameter(torch.zeros(hidden, dtype=dtype, device=device))
        self.eps = eps
        if sequence_parallel:
            mark_as_sequence_parallel_parameter(self.weight)
            mark_as_sequence_parallel_parameter(self.bias)

    def forward(self, x):
        return OF.layer_norm(x, self.weight, self.bias, self.eps)

    def forward_res(self, x):
        """(norm(x), residual alias of x): see ``OF.norm_with_residual``."""
        return OF.norm_with_residual(x, self.weight, self.bias, self.eps, False)


class RMSNorm(nn.Module):
    """``Model.normalization: rmsnorm`` — x / rms(x) * weight, no mean subtraction, no bias (Zhang & Sennrich 2019); runs the fused
    sm_100a norm kernel (``OF.rms_norm``).  Not in the reference (SURVEY §2.6 "demanded by the north-star")."""

    def __init__(self, hidden: int, eps: float = 1e-6, sequence_parallel: bool = False, dtype=None, device=None):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(hidden, dtype=dtype, device=device))
        self.bias = None
        self.eps = eps
        if sequence_parallel:
            mark_as_sequence_parallel_parameter(self.weight)

    def forward(self, x):
        return OF.rms_norm(x, self.weight, self.eps)

    def forward_res(self, x):
        return OF.norm_with_residual(x, self.weight, None, self.eps, True)


FFN_ACTIVATIONS = ("gelu", "swiglu")


def swiglu_ffn_size(hidden: int) -> int:
    """Default SwiGLU width: 8h/3 rounded up to a multiple of 256 (5632 at h = 2048), which keeps the FFN's parameter count near that of
    a 4h GELU FFN."""
    return -(-8 * hidden // (3 * 256)) * 256


def make_norm(kind: Optional[str], hidden: int, sequence_parallel: bool = False, dtype=None, device=None) -> nn.Module:
    kind = (kind or "layernorm").lower()
    if kind in ("layernorm", "layer_norm", "ln"):
        return LayerNorm(hidden, 1e-5, sequence_parallel, dtype, device)
    if kind in ("rmsnorm", "rms_norm", "rms"):
        return RMSNorm(hidden, 1e-6, sequence_parallel, dtype, device)
    raise ValueError(f"Model.normalization must be layernorm or rmsnorm, got {kind!r}")


class KVCache:
    """Pre-allocated static KV cache: in-place writes, no per-step concat/re-allocation (the reference grows
    its cache with ``concat`` every token, hybrid_model.py:198-214).  ``heads`` are the K/V heads (fewer than the query heads under
    grouped-query attention)."""

    def __init__(self, batch: int, max_len: int, heads: int, head_dim: int, dtype, device):
        self.k = torch.zeros(batch, max_len, heads, head_dim, dtype=dtype, device=device)
        self.v = torch.zeros_like(self.k)
        self.length = 0
        # graph mode: the write position is a device tensor and the whole buffer is attended (invalid keys are masked), so a
        # decode step has static shapes and can be replayed from a CUDA graph
        self.static_index: Optional[torch.Tensor] = None

    def reset(self) -> None:
        self.length = 0
        self.static_index = None

    def append(self, k: torch.Tensor, v: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        if self.static_index is not None:
            self.k.index_copy_(1, self.static_index, k)
            self.v.index_copy_(1, self.static_index, v)
            return self.k, self.v
        n = k.shape[1]
        self.k[:, self.length:self.length + n] = k
        self.v[:, self.length:self.length + n] = v
        self.length += n
        return self.k[:, :self.length], self.v[:, :self.length]


class MultiHeadAttention(nn.Module):
    def __init__(self, hidden: int, num_heads: int, attn_dropout: float = 0.0, fuse_attn_qkv: bool = True, scale_qk_coeff: float = 1.0,
                 use_flash_attn: bool = True, fused_softmax_with_triangular: bool = True, sequence_parallel: bool = False,
                 mp_group=None, init_std: float = 0.02, out_init_std: float = 0.02, recompute_core: bool = False,
                 fused_tp_comm: bool = False, use_rope: bool = False, num_key_value_heads: Optional[int] = None, dtype=None, device=None):
        super().__init__()
        self.hidden, self.num_heads = hidden, num_heads
        self.head_dim = hidden // num_heads
        assert self.head_dim * num_heads == hidden
        self.num_kv_heads = num_key_value_heads or num_heads
        assert num_heads % self.num_kv_heads == 0, f"heads {num_heads} % num_key_value_heads {self.num_kv_heads}"
        self.group = num_heads // self.num_kv_heads            # query heads per K/V head
        self.world = C.group_size(mp_group)
        assert num_heads % self.world == 0, f"heads {num_heads} % mp {self.world}"
        assert self.num_kv_heads % self.world == 0, f"num_key_value_heads {self.num_kv_heads} % mp {self.world}"
        self.local_heads = num_heads // self.world
        self.local_kv_heads = self.num_kv_heads // self.world
        self.attn_dropout = attn_dropout
        self.fuse_attn_qkv = fuse_attn_qkv
        self.scale_qk_coeff = scale_qk_coeff
        self.use_flash_attn = use_flash_attn
        self.fused_softmax_with_triangular = fused_softmax_with_triangular
        self.sequence_parallel = sequence_parallel
        self.recompute_core = recompute_core
        self.use_rope = use_rope
        kw = dict(mp_group=mp_group, dtype=dtype, device=device)
        Col = ColumnSequenceParallelLinear if sequence_parallel else ColumnParallelLinear
        Row = RowSequenceParallelLinear if sequence_parallel else RowParallelLinear
        ckw = dict(kw, gather_output=False, init_std=init_std)
        rkw = dict(kw, input_is_parallel=True, init_std=out_init_std, skip_bias_add=True)
        if sequence_parallel:
            ckw["fused_comm"] = fused_tp_comm
            rkw["fused_comm"] = fused_tp_comm
        kv_width = self.num_kv_heads * self.head_dim
        if fuse_attn_qkv:
            self.qkv_proj = Col(hidden, hidden + 2 * kv_width, **ckw)
        else:
            self.q_proj = Col(hidden, hidden, **ckw)
            self.k_proj = Col(hidden, kv_width, **ckw)
            self.v_proj = Col(hidden, kv_width, **ckw)
        self.out_proj = Row(hidden, hidden, **rkw)
        # context parallelism (``Distributed.cp_degree`` > 1): the group comes from the process topology, not from a constructor argument,
        # because to every other part of the model the members of a cp group are ordinary data-parallel ranks
        self.cp_group, self.cp_mode = None, "ulysses"
        from ....distributed.apis import env as _env

        hcg = getattr(_env, "_hcg", None)           # only an already-built topology counts (get_hcg() would build a default one)
        if hcg is not None and getattr(hcg, "cp", 1) > 1:
            if self.group > 1:
                raise ValueError("num_key_value_heads < num_attention_heads is not supported with context parallelism (Distributed.cp_degree > 1)")
            self.cp_group = hcg.get_context_parallel_group()
            self.cp_mode = getattr(hcg, "cp_mode", "ulysses")
            assert self.cp_mode == "ring" or self.local_heads % self.cp_group.nranks == 0, \
                f"local heads {self.local_heads} % cp {self.cp_group.nranks} (Ulysses shards heads; cp_mode: ring has no such limit)"

    # -- projections -------------------------------------------------------------------------
    def _packed_view(self, mix: torch.Tensor) -> torch.Tensor:
        """fused projection output -> ``[.., local_kv_heads, G + 2, d]`` (``[.., local_heads, 3, d]`` without grouping)."""
        return mix.view(*mix.shape[:-1], self.local_kv_heads, self.group + 2, self.head_dim)

    def _split_packed(self, mix: torch.Tensor):
        """q ``[.., local_heads, d]``, k / v ``[.., local_kv_heads, d]`` from the packed view."""
        if self.group == 1:
            return mix.unbind(-2)
        g = self.group
        return mix[..., :g, :].flatten(-3, -2), mix[..., g, :], mix[..., g + 1, :]

    def _qkv(self, x: torch.Tensor):
        """returns q as ``[b, s, local_heads, d]`` and k, v as ``[b, s, local_kv_heads, d]``."""
        if self.fuse_attn_qkv:
            q, k, v = self._split_packed(self._packed_view(self.qkv_proj(x)))
        else:
            lead = x.shape[:-1] if not self.sequence_parallel else (-1, x.shape[1])
            q, k, v = (p(x).view(*lead, n, self.head_dim)
                       for p, n in ((self.q_proj, self.local_heads), (self.k_proj, self.local_kv_heads), (self.v_proj, self.local_kv_heads)))
        if self.sequence_parallel:      # [s, b, heads, d] -> [b, s, heads, d]
            q, k, v = (t.transpose(0, 1) for t in (q, k, v))
        return q, k, v

    def _core(self, q, k, v, attn_mask):
        scale = 1.0 / math.sqrt(self.head_dim)
        p = self.attn_dropout if self.training else 0.0
        if isinstance(attn_mask, ATT.DocumentMask):
            if self.use_flash_attn:
                if p > 0:
                    with get_rng_state_tracker().rng_state("local_seed"):
                        return ATT.attention(q, k, v, dropout_p=p, scale=scale, attn_mask=attn_mask)
                return ATT.attention(q, k, v, dropout_p=0.0, scale=scale, attn_mask=attn_mask)
            attn_mask = attn_mask.additive()
        if (q.shape[1] == 1 and p == 0.0 and q.is_cuda and not torch.is_grad_enabled() and attn_mask is not None and attn_mask.dtype == q.dtype
                and attn_mask.shape[-1] == k.shape[1] and attn_mask.numel() == q.shape[0] * k.shape[1] and k.is_contiguous() and v.is_contiguous()
                and self.head_dim in (64, 128) and q.dtype in (torch.bfloat16, torch.float16) and OF.native_available()):
            # decode step over the static KV cache: one streaming kernel instead of a library attention call
            return OF.attention_decode(q, k, v, attn_mask, scale)
        if self.use_flash_attn:
            if attn_mask is not None:
                m = attn_mask if attn_mask.dtype == torch.bool else attn_mask.to(q.dtype)
                return ATT.attention(q, k, v, causal=False, dropout_p=p, scale=scale, attn_mask=m)
            if p > 0:
                with get_rng_state_tracker().rng_state("local_seed"):
                    return ATT.attention(q, k, v, causal=True, dropout_p=p, scale=scale)
            return ATT.attention(q, k, v, causal=q.shape[1] > 1, dropout_p=0.0, scale=scale)
        if self.scale_qk_coeff != 1.0:
            # overflow trick for fp16: scores = (q / (coeff * sqrt(d))) k^T, softmax input multiplied back by coeff
            q = q / self.scale_qk_coeff
            scale = scale * self.scale_qk_coeff
        causal = attn_mask is None and self.fused_softmax_with_triangular
        if attn_mask is None and not causal:
            sq, sk = q.shape[1], k.shape[1]
            attn_mask = torch.full((sq, sk), -1e4, device=q.device, dtype=torch.float32).triu(1 + sk - sq)
        return ATT.core_attention(q, k, v, scale, p, self.training, attn_mask=attn_mask, causal=causal)

    def _forward_context_parallel(self, x, attn_mask, positions):
        """Ulysses context parallelism: this rank holds ``s / c`` positions of every head; one all-to-all turns that into every position
        of ``H / c`` heads for the attention itself (causal over the FULL sequence), a second one turns it back.
        Ring mode (``Distributed.cp_mode: ring``): every head stays here, K / V blocks travel (parallel/ring_attention.py)."""
        q, k, v = self._qkv(x)                                                   # [b, s/c, H, d]
        if self.use_rope:
            if positions is None:     # pipeline stages > 0 receive activations only: the shard's positions follow from the layout (default ids)
                from ....parallel.ring_attention import local_positions

                positions = local_positions(q.shape[1], self.cp_group.nranks, self.cp_group.rank, self.cp_mode, q.device).expand(q.shape[0], -1)
            q, k = OF.rope(q.contiguous(), positions), OF.rope(k.contiguous(), positions)      # ``positions`` are global (sliced with the tokens)
        if self.cp_mode == "ring":
            assert attn_mask is None, "ring attention builds the causal mask from the zigzag layout; explicit masks are not sharded"
            from ....parallel.ring_attention import ring_attention

            p = self.attn_dropout if self.training else 0.0
            if p > 0:
                with get_rng_state_tracker().rng_state("local_seed"):
                    out = ring_attention(q, k, v, self.cp_group, True, p, self.head_dim ** -0.5)
            else:
                out = ring_attention(q, k, v, self.cp_group, True, 0.0, self.head_dim ** -0.5)
            return self._project_out(out)
        q, k, v = (C.seq_head_all_to_all(t, self.cp_group, 2, 1) for t in (q, k, v))           # [b, s, H/c, d]
        out = recompute(self._core, q, k, v, attn_mask) if (self.recompute_core and self.training) else self._core(q, k, v, attn_mask)
        out = C.seq_head_all_to_all(out, self.cp_group, 1, 2)                    # [b, s/c, H, d]
        return self._project_out(out)

    def _project_out(self, out):
        """``[b, s, heads, d]`` -> output projection; Megatron sequence parallelism wants ``[s, b, h / n]`` (GEMM -> reduce-scatter along s)."""
        out = out.reshape(out.shape[0], out.shape[1], self.local_heads * self.head_dim)
        if self.sequence_parallel:
            out = out.transpose(0, 1).contiguous()
        return self.out_proj(out)

    def forward(self, x: torch.Tensor, attn_mask: Optional[torch.Tensor] = None, cache: Optional[KVCache] = None,
                positions: Optional[torch.Tensor] = None):
        if self.cp_group is not None and cache is None:
            return self._forward_context_parallel(x, attn_mask, positions)
        doc = attn_mask if isinstance(attn_mask, ATT.DocumentMask) else None
        if (self.fuse_attn_qkv and self.use_flash_attn and not self.use_rope and cache is None and (attn_mask is None or doc is not None)
                and x.is_cuda and not (self.recompute_core and self.training)):
            # fused projection output [.., heads, 3, d] goes to the flash kernels as it is: q / k / v are read in place (TMA views), the
            # backward writes one packed gradient — no unbind / transpose / cat copies around the attention
            mix = self._packed_view(self.qkv_proj(x))
            if self.sequence_parallel:
                mix = mix.transpose(0, 1)
            if mix.shape[1] > 1:
                p = self.attn_dropout if self.training else 0.0
                scale = 1.0 / math.sqrt(self.head_dim)
                if p > 0:
                    with get_rng_state_tracker().rng_state("local_seed"):
                        out = ATT.flash_attention_packed(mix, causal=True, dropout_p=p, scale=scale, doc=doc)
                else:
                    out = ATT.flash_attention_packed(mix, causal=True, dropout_p=0.0, scale=scale, doc=doc)
            else:
                out = None
            if out is None:
                q, k, v = self._split_packed(mix)
                out = self._core(q, k, v, doc)
            out = out.reshape(out.shape[0], out.shape[1], self.local_heads * self.head_dim)
            if self.sequence_parallel:
                out = out.transpose(0, 1).contiguous()
            return self.out_proj(out)
        q, k, v = self._qkv(x)
        if self.use_rope:
            pos = positions
            if pos is None and cache is not None and cache.length > 0:
                pos = torch.arange(cache.length, cache.length + q.shape[1], device=q.device).expand(q.shape[0], -1)
            q, k = OF.rope(q.contiguous(), pos), OF.rope(k.contiguous(), pos)
        if cache is not None:
            k, v = cache.append(k, v)
        if self.recompute_core and self.training:
            out = recompute(self._core, q, k, v, attn_mask)
        else:
            out = self._core(q, k, v, attn_mask)
        out = out.reshape(out.shape[0], out.shape[1], self.local_heads * self.head_dim)
        if self.sequence_parallel:
            out = out.transpose(0, 1).contiguous()
        return self.out_proj(out)          # (y, bias): bias is folded into the following dropout+residual kernel


class TransformerDecoderLayer(nn.Module):
    def __init__(self, hidden: int, num_heads: int, ffn_hidden: int, hidden_dropout: float = 0.1, attn_dropout: float = 0.1,
                 num_layers: int = 1, sequence_parallel: bool = False, mp_group=None, init_std: float = 0.02,
                 recompute_attn: bool = False, recompute_core: bool = False, moe_layer: Optional[nn.Module] = None,
                 fused_tp_comm: bool = False, normalization: Optional[str] = None, ffn_activation: str = "gelu", dtype=None, device=None,
                 **attn_kwargs):
        super().__init__()
        if ffn_activation not in FFN_ACTIVATIONS:
            raise ValueError(f"Model.ffn_activation must be one of {', '.join(FFN_ACTIVATIONS)}, got {ffn_activation!r}")
        if ffn_activation == "swiglu" and moe_layer is not None:
            raise ValueError("ffn_activation: swiglu is not supported with MoE layers (moe_configs); the experts keep GELU")
        self.ffn_activation = ffn_activation
        out_std = init_std / math.sqrt(2.0 * num_layers)
        self.sequence_parallel = sequence_parallel
        self.hidden_dropout = hidden_dropout
        self.recompute_attn = recompute_attn
        self.norm1 = make_norm(normalization, hidden, sequence_parallel, dtype, device)
        self.self_attn = MultiHeadAttention(hidden, num_heads, attn_dropout, sequence_parallel=sequence_parallel, mp_group=mp_group,
                                            init_std=init_std, out_init_std=out_std, recompute_core=recompute_core,
                                            fused_tp_comm=fused_tp_comm, dtype=dtype, device=device, **attn_kwargs)
        self.norm2 = make_norm(normalization, hidden, sequence_parallel, dtype, device)
        self.moe_mlp = moe_layer
        if moe_layer is None:
            Col = ColumnSequenceParallelLinear if sequence_parallel else ColumnParallelLinear
            Row = RowSequenceParallelLinear if sequence_parallel else RowParallelLinear
            kw = dict(mp_group=mp_group, dtype=dtype, device=device)
            extra = dict(fused_comm=fused_tp_comm) if sequence_parallel else {}
            ffn1_width = 2 * ffn_hidden if ffn_activation == "swiglu" else ffn_hidden      # gate / up pairs, interleaved
            self.linear1 = Col(hidden, ffn1_width, gather_output=False, init_std=init_std, has_bias=True, **kw, **extra)
            self.linear2 = Row(ffn_hidden, hidden, input_is_parallel=True, init_std=out_std, skip_bias_add=True, **kw, **extra)
        # hidden dropout stream: identical inside the TP group without SP, distinct under SP
        self.rng_name = "local_seed" if sequence_parallel else "global_seed"

    def _attn_block(self, x, attn_mask, cache, positions):
        h, x = self.norm1.forward_res(x)
        y, b = self.self_attn(h, attn_mask, cache, positions)
        return OF.bias_dropout_add(y, b, x, self.hidden_dropout, self.training, self.rng_name)

    def _ffn(self, h):
        l1, l2 = self.linear1, self.linear2
        if self.ffn_activation == "swiglu":
            return l2(OF.bias_swiglu(l1(h, skip_bias=True), l1.bias))
        if (getattr(l1, "world", 1) == 1 and not self.self_attn.sequence_parallel and getattr(l1, "int8", None) is None and l1.weight is not None
                and not getattr(l1, "needs_forward", False) and not getattr(l2, "needs_forward", False)
                and l1.bias is not None and getattr(l2, "skip_bias_add", False) and not _TP_OPTIONS["fp8_tp_gemm"]):
            # single tensor-parallel rank: both GEMMs in one autograd node with GELU / GELU' inside their epilogues
            return OF.fused_ffn(h, l1.weight, l1.bias, l2.weight), l2.bias
        z = l1(h, skip_bias=True)                # GEMM only; bias rides in the fused bias+GELU kernel
        return l2(OF.bias_gelu(z, l1.bias))

    def _decode_fast_ok(self, x, attn_mask, cache) -> bool:
        a = self.self_attn
        forced = getattr(self, "_force_decode_fast", False)          # tests: run the fused-step composition through the CPU expressions
        hw = forced or (x.is_cuda and x.shape[0] <= OF.gemv_max_rows() and a.head_dim in (64, 128) and x.dtype in (torch.bfloat16, torch.float16)
                        and OF.native_available())
        return (hw and isinstance(self.norm1, LayerNorm) and cache is not None and cache.static_index is not None and x.shape[1] == 1
                and not self.training and not torch.is_grad_enabled() and self.moe_mlp is None and a.world == 1 and not a.sequence_parallel
                and a.fuse_attn_qkv and not a.use_rope and a.use_flash_attn
                and attn_mask is not None and attn_mask.dtype == x.dtype and attn_mask.numel() == x.shape[0] * cache.k.shape[1]
                and getattr(a.qkv_proj, "int8", None) is None and a.qkv_proj.weight is not None
                and not any(getattr(m, "needs_forward", False) for m in (a.qkv_proj, a.out_proj, self.linear1, self.linear2)))

    def _decode_fast(self, x, attn_mask, cache):
        """One decode token through the layer in five launches: LN1+QKV GEMV, cache-append + attention, out-proj GEMV + bias + residual,
        LN2+FFN1 GEMV + bias + GELU / SwiGLU, FFN2 GEMV + bias + residual (the generic path takes thirteen)."""
        a = self.self_attn
        b = x.shape[0]
        x2 = x.reshape(b, -1)
        qkv = OF.gemv_fused(x2, a.qkv_proj.weight, a.qkv_proj.bias, ln=(self.norm1.weight, self.norm1.bias, self.norm1.eps))
        o = OF.attention_decode_packed(qkv.view(b, 1, a.local_kv_heads, a.group + 2, a.head_dim), cache.k, cache.v, attn_mask, cache.static_index,
                                       1.0 / math.sqrt(a.head_dim))
        x2 = OF.gemv_fused(o.view(b, -1), a.out_proj.weight, a.out_proj.bias, residual=x2)
        h = OF.gemv_fused(x2, self.linear1.weight, self.linear1.bias, ln=(self.norm2.weight, self.norm2.bias, self.norm2.eps),
                          act=self.ffn_activation)
        x2 = OF.gemv_fused(h, self.linear2.weight, self.linear2.bias, residual=x2)
        return x2.view_as(x)

    def forward(self, x: torch.Tensor, attn_mask: Optional[torch.Tensor] = None, cache: Optional[KVCache] = None,
                positions: Optional[torch.Tensor] = None) -> torch.Tensor:
        if self._decode_fast_ok(x, attn_mask, cache):
            return self._decode_fast(x, attn_mask, cache)
        if self.recompute_attn and self.training and cache is None:
            x = recompute(self._attn_block, x, attn_mask, None, positions)
        else:
            x = self._attn_block(x, attn_mask, cache, positions)
        h, x = self.norm2.forward_res(x)
        if self.moe_mlp is not None:
            y = self.moe_mlp(h)
            return OF.bias_dropout_add(y, None, x, self.hidden_dropout, self.training, self.rng_name)
        y, b = self._ffn(h)
        return OF.bias_dropout_add(y, b, x, self.hidden_dropout, self.training, self.rng_name)


class TransformerDecoder(nn.Module):
    def __init__(self, layers: List[nn.Module], hidden: int, use_recompute: bool = False, recompute_granularity: str = "full",
                 no_recompute_layers: Optional[List[int]] = None, sequence_parallel: bool = False, dtype=None, device=None,
                 normalization: Optional[str] = None):
        super().__init__()
        self.layers = nn.ModuleList(layers)
        self.norm = make_norm(normalization, hidden, sequence_parallel, dtype, device)
        self.use_recompute = use_recompute
        self.recompute_granularity = recompute_granularity
        self.no_recompute_layers = set(no_recompute_layers or [])

    def forward(self, x, attn_mask=None, caches: Optional[List[KVCache]] = None, positions=None):
        for i, layer in enumerate(self.layers):
            cache = caches[i] if caches is not None else None
            if (self.use_recompute and self.recompute_granularity == "full" and self.training and cache is None
                    and i not in self.no_recompute_layers):
                x = recompute(layer, x, attn_mask, None, positions)
            else:
                x = layer(x, attn_mask, cache, positions)
        return self.norm(x)


class GPTEmbeddings(nn.Module):
    def __init__(self, vocab_size: int, hidden: int, max_position: int, hidden_dropout: float, init_std: float, sequence_parallel: bool,
                 mp_group=None, use_rope: bool = False, dtype=None, device=None):
        super().__init__()
        self.word_embeddings = VocabParallelEmbedding(vocab_size, hidden, mp_group, init_std, dtype, device)
        self.use_rope = use_rope
        if not use_rope:
            self.position_embeddings = nn.Embedding(max_position, hidden, dtype=dtype, device=device)
            with torch.no_grad():
                self.position_embeddings.weight.normal_(0.0, init_std)
        self.hidden_dropout = hidden_dropout
        self.sequence_parallel = sequence_parallel
        self.group = mp_group

    def forward(self, input_ids: torch.Tensor, position_ids: Optional[torch.Tensor] = None) -> torch.Tensor:
        if not self.use_rope and position_ids is None:
            position_ids = torch.arange(input_ids.shape[1], device=input_ids.device).unsqueeze(0).expand_as(input_ids)
        if not self.use_rope and self.word_embeddings.world == 1:
            # word + position look-up and their sum in one kernel (csrc/embedding.cu); backward scatters into both tables deterministically
            x = self.word_embeddings(input_ids, position_ids.contiguous(), self.position_embeddings.weight)
        else:
            x = self.word_embeddings(input_ids)
            if not self.use_rope:
                x = x + self.position_embeddings(position_ids)
        if self.sequence_parallel:
            x = C.scatter_seq(x.transpose(0, 1).contiguous(), self.group)     # [s/n, b, h]
            return OF.dropout(x, self.hidden_dropout, self.training, "local_seed")
        return OF.dropout(x, self.hidden_dropout, self.training, "global_seed")


class GPTModel(nn.Module):
    def __init__(self, vocab_size: int = 50304, hidden_size: int = 768, num_layers: int = 12, num_attention_heads: int = 12,
                 ffn_hidden_size: Optional[int] = None, hidden_dropout_prob: float = 0.1, attention_probs_dropout_prob: float = 0.1,
                 max_position_embeddings: int = 1024, type_vocab_size: int = 16, initializer_range: float = 0.02,
                 use_recompute: bool = False, recompute_granularity: Optional[str] = "full", no_recompute_layers=None,
                 fused_linear: bool = False, fuse_attn_qkv: bool = True, scale_qk_by_layer_num: bool = True,
                 sequence_parallel: bool = False, use_flash_attn: bool = True, fused_softmax_with_triangular: bool = True,
                 mp_group=None, moe_configs: Optional[dict] = None, fused_tp_comm: bool = False, use_rope: bool = False,
                 normalization: Optional[str] = None, num_key_value_heads: Optional[int] = None, ffn_activation: str = "gelu",
                 reset_attention_mask: bool = False, dtype=None, device=None, **unused):
        super().__init__()
        ffn_hidden_size = ffn_hidden_size or (swiglu_ffn_size(hidden_size) if ffn_activation == "swiglu" else 4 * hidden_size)
        recompute_granularity = recompute_granularity or "full"
        self.hidden_size, self.vocab_size, self.num_layers = hidden_size, vocab_size, num_layers
        self.initializer_range = initializer_range
        self.mp_group = mp_group
        self.reset_attention_mask = reset_attention_mask
        self.sequence_parallel = sequence_parallel and C.group_size(mp_group) > 1
        sp = self.sequence_parallel
        self.embeddings = GPTEmbeddings(vocab_size, hidden_size, max_position_embeddings, hidden_dropout_prob, initializer_range,
                                        sp, mp_group, use_rope, dtype, device)
        layers = []
        for i in range(num_layers):
            moe = None
            if moe_configs and moe_configs.get("expert_mode", False):
                from ..moe.moe_layer import build_moe_layer

                moe = build_moe_layer(hidden_size, ffn_hidden_size, moe_configs, num_layers, initializer_range, mp_group, dtype, device, i)
            layers.append(TransformerDecoderLayer(
                hidden_size, num_attention_heads, ffn_hidden_size, hidden_dropout_prob, attention_probs_dropout_prob, num_layers,
                sequence_parallel=sp, mp_group=mp_group, init_std=initializer_range,
                recompute_attn=use_recompute and recompute_granularity == "full_attn",
                recompute_core=use_recompute and recompute_granularity == "core_attn", moe_layer=moe, fused_tp_comm=fused_tp_comm,
                dtype=dtype, device=device, fuse_attn_qkv=fuse_attn_qkv,
                scale_qk_coeff=float(num_layers) if scale_qk_by_layer_num else 1.0, use_flash_attn=use_flash_attn,
                fused_softmax_with_triangular=fused_softmax_with_triangular, use_rope=use_rope, normalization=normalization,
                num_key_value_heads=num_key_value_heads, ffn_activation=ffn_activation))
        self.decoder = TransformerDecoder(layers, hidden_size, use_recompute, recompute_granularity, no_recompute_layers, sp, dtype, device,
                                          normalization=normalization)

    def new_caches(self, batch: int, max_len: int) -> List[KVCache]:
        p = self.decoder.norm.weight
        lh, hd = self.decoder.layers[0].self_attn.local_kv_heads, self.decoder.layers[0].self_attn.head_dim
        return [KVCache(batch, max_len, lh, hd, p.dtype, p.device) for _ in self.decoder.layers]

    def forward(self, input_ids, position_ids=None, attention_mask=None, caches: Optional[List[KVCache]] = None):
        if position_ids is None and caches is not None and caches[0].length > 0:
            past = caches[0].length
            position_ids = torch.arange(past, past + input_ids.shape[1], device=input_ids.device).unsqueeze(0).expand_as(input_ids)
        if self.reset_attention_mask and attention_mask is None and position_ids is not None and caches is None:
            # one mask for every layer: on CUDA one launch derives the per-row key bounds and their per-tile min / max
            attention_mask = ATT.DocumentMask.from_positions(position_ids)
        x = self.embeddings(input_ids, position_ids)
        x = self.decoder(x, attention_mask, caches, position_ids)
        if self.sequence_parallel:
            x = C.gather_seq(x, self.mp_group).transpose(0, 1).contiguous()      # back to [b, s, h]
        return x


GPTModelHybrid = GPTModel


class GPTForPretraining(nn.Module):
    """LM head tied to the (vocab-parallel) word embedding."""

    def __init__(self, gpt: GPTModel, parallel_output: bool = True):
        super().__init__()
        self.gpt = gpt
        self.parallel_output = parallel_output

    def forward(self, input_ids, position_ids=None, attention_mask=None, caches=None):
        h = self.gpt(input_ids, position_ids, attention_mask, caches)
        return parallel_matmul(h, self.gpt.embeddings.word_embeddings.weight, self.gpt.mp_group, self.parallel_output)


GPTForPretrainingHybrid = GPTForPretraining


class GPTPretrainingCriterion(nn.Module):
    """loss = sum(CE * mask) / sum(mask) (reference hybrid_model.py:955-996)."""

    def __init__(self, mp_group=None):
        super().__init__()
        self.ce = ParallelCrossEntropy(mp_group)

    def forward(self, logits: torch.Tensor, labels: torch.Tensor, loss_mask: torch.Tensor, denominator: Optional[torch.Tensor] = None) -> torch.Tensor:
        """``denominator`` (per-sample live-token counts) replaces ``sum(mask)`` when the mask seen here is only a shard of the sequences
        (context parallelism under the pipeline schedule: language_module.GPTModule.pretreating_batch)."""
        per_tok = self.ce(logits, labels)
        mask = loss_mask.reshape(-1).float()
        return (per_tok.reshape(-1) * mask).sum() / (mask.sum() if denominator is None else denominator.float().sum())


GPTPretrainingCriterionHybird = GPTPretrainingCriterion  # (sic) name used by the reference module layer


class GPTForSequenceClassification(nn.Module):
    """Pooled logit = hidden state of the last non-pad token -> ``score`` (reference single_model.py:856-895)."""

    def __init__(self, gpt: GPTModel, num_classes: int = 2, pad_token_id: int = 0):
        super().__init__()
        self.gpt = gpt
        p = gpt.decoder.norm.weight
        self.score = nn.Linear(gpt.hidden_size, num_classes, bias=False, dtype=p.dtype, device=p.device)
        with torch.no_grad():
            self.score.weight.normal_(0.0, gpt.initializer_range)
        self.pad_token_id = pad_token_id

    def forward(self, input_ids, position_ids=None, attention_mask=None):
        h = self.gpt(input_ids, position_ids, attention_mask)
        logits = self.score(h)
        eos = (input_ids != self.pad_token_id).to(torch.int64).sum(-1) - 1
        return logits[torch.arange(input_ids.shape[0], device=input_ids.device), eos.clamp_min(0)]


def vocab_size_with_padding(vocab_size: int, div_unit: int, mp_degree: int) -> int:
    """Pad the vocabulary to a multiple of ``div_unit * mp`` (reference language_module.py:62-70)."""
    mult = div_unit * mp_degree
    return ((vocab_size + mult - 1) // mult) * mult


# ---------------------------------------------------------------------------------------------------------------------------------------
# Names of the reference's split files (gpt/dygraph/{single,hybrid}_model.py, gpt/auto/auto_model.py) that resolve to this module.
def get_attr(layer, name):
    """Attribute lookup through wrapper layers (``._layer`` / ``._layers``), reference hybrid_model.py:59-63."""
    while layer is not None:
        value = getattr(layer, name, None)
        if value is not None:
            return value
        layer = getattr(layer, "_layer", None) or getattr(layer, "_layers", None)
    raise AttributeError(name)


def get_triangle_upper_mask(x: torch.Tensor, mask: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Additive causal mask shaped like the score tensor ``x`` (``-inf`` above the diagonal) unless one is given
    (reference hybrid_model.py:1681-1688; the training path never builds it: the flash kernels mask by tile)."""
    if mask is not None:
        return mask
    return torch.full_like(x, float("-inf")).triu(1)


class ConcatSoftmaxInput(torch.autograd.Function):
    """All-gather vocabulary-parallel logits along the last axis; backward keeps this rank's slice (reference hybrid_model.py:1691-1708,
    used by ``GPTForGenerationHybrid`` to sample from the full distribution)."""

    @staticmethod
    def forward(ctx, inp, group=None):
        ctx.group = group
        if C.group_size(group) == 1:
            return inp.view_as(inp)
        return C.all_gather_dim(inp.contiguous(), group, inp.dim() - 1)

    @staticmethod
    def backward(ctx, grad):
        if C.group_size(ctx.group) == 1:
            return grad, None
        return C.split_dim(grad, ctx.group, grad.dim() - 1), None


# the auto-parallel variants are the same classes: the sharding the reference annotates with ``auto.shard_tensor`` lives in the layers
GPTModelAuto = GPTModel
GPTForPretrainingAuto = GPTForPretraining
GPTPretrainingCriterionAuto = GPTPretrainingCriterion

from ....utils.lazy import lazy_exports  # noqa: E402

__getattr__ = lazy_exports(__name__, {
    "GPTForPretrainingPipe": ".pipe", "GPTPretrainingCriterionPipe": ".pipe", "EmbeddingPipe": ".pipe", "LayerNormPipe": ".pipe",
    "GPTForGeneration": ".generation", "GPTForGenerationHybrid": ".generation", "GPTForGenerationAuto": ".generation:GPTForGeneration",
    "ExpertLayer": "..moe.moe_layer",
})
