"""Pipeline-parallel GPT: a ``PipelineLayer`` built from layer descriptors.

Stage layout (reference gpt/dygraph/hybrid_model.py:1002-1206): ``SharedLayerDesc('embed')`` (word+position
embedding) -> L x ``TransformerDecoderLayer`` -> final LayerNorm (+ sequence-parallel gather) ->
``SharedLayerDesc('embed', forward_func=logits)`` (tied LM head) with ``GPTPretrainingCriterionPipe`` as the loss on
the last stage; ``seg_method = layer:TransformerDecoderLayer`` (uniform fallback), ``virtual_pp_degree`` and
``pp_recompute_interval`` supported.
"""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from ....parallel import comm_ops as C
from ....parallel.pipeline import LayerDesc, PipelineLayer, SharedLayerDesc
from ....parallel.tp_layers import parallel_matmul
from . import model as gpt


class EmbeddingPipe(gpt.GPTEmbeddings):
    """Embedding stage; also owns the tied LM-head weight on the last stage."""

    @property
    def embedding_weight(self):
        return self.word_embeddings.weight

    def forward(self, tokens, position_ids=None):
        return super().forward(tokens, position_ids)


class LayerNormPipe(nn.Module):
    def __init__(self, hidden: int, sequence_parallel: bool, mp_group=None, dtype=None, device=None, normalization=None):
        super().__init__()
        self.norm = gpt.make_norm(normalization, hidden, sequence_parallel, dtype, device)
        self.sequence_parallel = sequence_parallel
        self.group = mp_group

    def forward(self, x):
        x = self.norm(x)
        if self.sequence_parallel:
            x = C.gather_seq(x, self.group).transpose(0, 1).contiguous()
        return x


def _logits_helper(embedding: EmbeddingPipe, hidden: torch.Tensor) -> torch.Tensor:
    return parallel_matmul(hidden, embedding.embedding_weight, embedding.group, parallel_output=True)


class GPTPretrainingCriterionPipe(gpt.GPTPretrainingCriterion):
    """Same masked-mean CE; signature ``(logits, labels, loss_mask)`` as called by the pipeline runtime."""


class GPTForPretrainingPipe(PipelineLayer):
    def __init__(self, hcg, mp_group=None, vocab_size: int = 50304, hidden_size: int = 768, num_layers: int = 12,
                 num_attention_heads: int = 12, ffn_hidden_size: Optional[int] = None, hidden_dropout_prob: float = 0.1,
                 attention_probs_dropout_prob: float = 0.1, max_position_embeddings: int = 1024, initializer_range: float = 0.02,
                 use_recompute: bool = False, recompute_granularity: Optional[str] = "full", no_recompute_layers=None,
                 fuse_attn_qkv: bool = True, scale_qk_by_layer_num: bool = True, sequence_parallel: bool = False,
                 use_flash_attn: bool = True, fused_softmax_with_triangular: bool = True, virtual_pp_degree: int = 1,
                 pp_recompute_interval: int = 1, fused_tp_comm: bool = False, use_rope: bool = False, normalization=None,
                 num_key_value_heads: Optional[int] = None, ffn_activation: str = "gelu", dtype=None, device=None, **unused):
        ffn_hidden_size = ffn_hidden_size or (gpt.swiglu_ffn_size(hidden_size) if ffn_activation == "swiglu" else 4 * hidden_size)
        recompute_granularity = recompute_granularity or "full"
        sp = sequence_parallel and C.group_size(mp_group) > 1
        embed_args = dict(vocab_size=vocab_size, hidden=hidden_size, max_position=max_position_embeddings,
                          hidden_dropout=hidden_dropout_prob, init_std=initializer_range, sequence_parallel=sp, mp_group=mp_group,
                          use_rope=use_rope, dtype=dtype, device=device)
        descs = [SharedLayerDesc("embed", EmbeddingPipe, shared_weight_attr="embedding_weight", **embed_args)]
        for _ in range(num_layers):
            descs.append(LayerDesc(
                gpt.TransformerDecoderLayer, hidden_size, num_attention_heads, ffn_hidden_size, hidden_dropout_prob,
                attention_probs_dropout_prob, num_layers, sequence_parallel=sp, mp_group=mp_group, init_std=initializer_range,
                recompute_attn=use_recompute and recompute_granularity == "full_attn",
                recompute_core=use_recompute and recompute_granularity == "core_attn", fused_tp_comm=fused_tp_comm, dtype=dtype,
                device=device, fuse_attn_qkv=fuse_attn_qkv, scale_qk_coeff=float(num_layers) if scale_qk_by_layer_num else 1.0,
                use_flash_attn=use_flash_attn, fused_softmax_with_triangular=fused_softmax_with_triangular, use_rope=use_rope,
                normalization=normalization, num_key_value_heads=num_key_value_heads, ffn_activation=ffn_activation))
        descs.append(LayerDesc(LayerNormPipe, hidden_size, sp, mp_group, dtype, device, normalization))
        descs.append(SharedLayerDesc("embed", EmbeddingPipe, forward_func=_logits_helper, shared_weight_attr="embedding_weight", **embed_args))
        interval = pp_recompute_interval if (use_recompute and recompute_granularity == "full") else 0
        super().__init__(layers=descs, loss_fn=GPTPretrainingCriterionPipe(mp_group), hcg=hcg, seg_method="layer:TransformerDecoderLayer",
                         recompute_interval=interval, recompute_ctx=None,
                         num_virtual_pipeline_stages=virtual_pp_degree if virtual_pp_degree and virtual_pp_degree > 1 else 1)
        self.mp_group = mp_group
        self.hidden_size, self.vocab_size, self.num_layers = hidden_size, vocab_size, num_layers
