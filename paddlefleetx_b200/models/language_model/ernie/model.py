"""ERNIE: bidirectional encoder with MLM + sentence-order heads (single card, tensor parallel, pipeline).

Reference: ppfleetx/models/language_model/ernie/dygraph/{single_model.py:34-765, hybrid_model.py:40-992} and
ernie/layers/*.  Kept: word / position / token-type / task embeddings, post-LN encoder (``normalize_before`` switch),
tanh pooler, MLM transform (dense + act + LN) with a decoder tied to the word embedding, SOP head, masked-position
gather before the MLM head, ``ignore_index = -1`` criterion, sequence-classification head.

Beyond the reference (needed for BASELINE config #3, ERNIE-10B mp4 + ZeRO-3): the MLM decoder is vocabulary-parallel
and the loss uses the vocab-parallel CE kernel (the reference leaves both replicated — SURVEY §2.7); attention runs the
fused flash path with a padding mask: ``ErnieModel.forward`` builds one ``KeyPaddingMask`` per forward pass from the 2-D mask or the
pad tokens, and every layer hands it to the key-padding flash kernels (the explicit-mask paths add its ``[b, 1, 1, s]`` form).
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from ....ops import attention as ATT
from ....ops import functional as OF
from ....parallel import comm_ops as C
from ....parallel.recompute import recompute
from ....parallel.rng import get_rng_state_tracker
from ....parallel.tp_layers import (ColumnParallelLinear, ColumnSequenceParallelLinear, ParallelCrossEntropy, RowParallelLinear,
                                    RowSequenceParallelLinear, VocabParallelEmbedding, _tp_linear, parallel_matmul)
from ..gpt.model import LayerNorm

_ACT = {"gelu": lambda x: F.gelu(x, approximate="none"), "relu": F.relu, "tanh": torch.tanh}


class ErnieEmbeddings(nn.Module):
    def __init__(self, vocab_size, hidden, hidden_dropout=0.1, max_position=512, type_vocab_size=2, task_type_vocab_size=3, task_id=0,
                 use_task_id=False, init_std=0.02, mp_group=None, dtype=None, device=None):
        super().__init__()
        kw = dict(dtype=dtype, device=device)
        self.word_embeddings = VocabParallelEmbedding(vocab_size, hidden, mp_group, init_std, dtype, device)
        self.position_embeddings = nn.Embedding(max_position, hidden, **kw)
        self.token_type_embeddings = nn.Embedding(type_vocab_size, hidden, **kw)
        self.use_task_id, self.task_id = use_task_id, task_id
        if use_task_id:
            self.task_type_embeddings = nn.Embedding(task_type_vocab_size, hidden, **kw)
        for e in (self.position_embeddings, self.token_type_embeddings, getattr(self, "task_type_embeddings", None)):
            if e is not None:
                with torch.no_grad():
                    e.weight.normal_(0.0, init_std)
        self.layer_norm = LayerNorm(hidden, 1e-12, False, dtype, device)
        self.dropout_p = hidden_dropout

    def forward(self, input_ids, token_type_ids=None, position_ids=None, task_type_ids=None, inputs_embeds=None, past_key_values_length=None):
        """``inputs_embeds`` replaces the word-embedding lookup; ``past_key_values_length`` offsets the default positions when the caller
        feeds only the new tokens of an incrementally extended sequence (reference single_model.py:71-112)."""
        words = self.word_embeddings(input_ids) if input_ids is not None else inputs_embeds
        b, s = words.shape[:2]
        if position_ids is None:
            position_ids = (torch.arange(s, device=words.device) + int(past_key_values_length or 0)).unsqueeze(0).expand(b, s)
        if token_type_ids is None:
            token_type_ids = torch.zeros(b, s, dtype=torch.long, device=words.device)
        x = words + self.position_embeddings(position_ids) + self.token_type_embeddings(token_type_ids)
        if self.use_task_id:
            if task_type_ids is None:
                task_type_ids = torch.full((b, s), self.task_id, dtype=torch.long, device=words.device)
            x = x + self.task_type_embeddings(task_type_ids)
        return OF.dropout(self.layer_norm(x), self.dropout_p, self.training, "global_seed")


class ErnieSelfAttention(nn.Module):
    """Separate q/k/v column-parallel projections like the reference hybrid model (no fused QKV), row-parallel output."""

    def __init__(self, hidden, heads, attn_dropout, mp_group=None, init_std=0.02, dtype=None, device=None, use_flash_attn=True,
                 sequence_parallel=False, fused_tp_comm=False):
        super().__init__()
        self.heads, self.head_dim = heads, hidden // heads
        self.local_heads = heads // C.group_size(mp_group)
        self.group, self.sequence_parallel = mp_group, sequence_parallel
        kw = dict(mp_group=mp_group, init_std=init_std, dtype=dtype, device=device)
        # the three projections stay separate modules (checkpoint keys of the reference); under sequence parallelism they share ONE
        # all-gather of the sequence shards (see forward) instead of gathering three times
        self.q_proj = ColumnParallelLinear(hidden, hidden, gather_output=False, **kw)
        self.k_proj = ColumnParallelLinear(hidden, hidden, gather_output=False, **kw)
        self.v_proj = ColumnParallelLinear(hidden, hidden, gather_output=False, **kw)
        if sequence_parallel:
            self.out_proj = RowSequenceParallelLinear(hidden, hidden, input_is_parallel=True, fused_comm=fused_tp_comm, **kw)
        else:
            self.out_proj = RowParallelLinear(hidden, hidden, input_is_parallel=True, **kw)
        self.attn_dropout = attn_dropout
        self.use_flash_attn = use_flash_attn

    def forward_detailed(self, x, attn_mask=None, cache=None, need_weights=False):
        """The inspection / incremental path (reference layers/transformer.py:346-436): explicit softmax so that the attention probabilities
        can be returned, and an optional ``(k, v)`` cache of [b, heads, s_past, d] that the new keys / values are appended to.  Returns
        ``(out, weights or None, new_cache or None)``.  Not used by training (that is ``forward``: flash kernels, no materialised scores)."""
        assert not self.sequence_parallel, "attention weights / caches are not available on sequence-parallel activations"
        b, s, _ = x.shape
        q, k, v = (p(x).view(b, s, self.local_heads, self.head_dim).transpose(1, 2) for p in (self.q_proj, self.k_proj, self.v_proj))
        new_cache = None
        if cache is not None:
            k, v = torch.cat([cache[0], k], dim=2), torch.cat([cache[1], v], dim=2)
            new_cache = (k, v)
        scores = torch.matmul(q * self.head_dim ** -0.5, k.transpose(-1, -2))
        if attn_mask is not None:
            scores = scores + attn_mask.to(scores.dtype)
        weights = torch.softmax(scores.float(), dim=-1).to(q.dtype)
        probs = weights
        if self.training and self.attn_dropout > 0:
            with get_rng_state_tracker().rng_state("local_seed"):
                probs = F.dropout(weights, self.attn_dropout, True)
        o = torch.matmul(probs, v).transpose(1, 2).reshape(b, s, self.local_heads * self.head_dim)
        return self.out_proj(o), (probs if need_weights else None), new_cache

    def gen_cache(self, x):
        """Empty ``(k, v)`` cache for a batch shaped like ``x`` (reference ``MultiHeadAttention.gen_cache``)."""
        z = x.new_zeros(x.shape[0], self.local_heads, 0, self.head_dim)
        return (z, z.clone())

    def forward(self, x, attn_mask=None):
        """``attn_mask``: a ``KeyPaddingMask`` (the flash kernels read it as it is, also on the gathered ``[s, b, ...]`` views of sequence
        parallelism) or an additive tensor."""
        if self.sequence_parallel:
            # x: [s/n, b, h] -> one all-gather (backward: reduce-scatter) -> [s, b, h]; the column-parallel GEMMs then run on the gathered
            # tensor directly (no identity/all-reduce pair: the gather's backward already sums the partial input gradients)
            xg = C.all_gather_seq(x, self.group)
            s, b, _ = xg.shape
            q, k, v = (_tp_linear(xg, p.weight, p.bias, p).view(s, b, self.local_heads, self.head_dim).transpose(0, 1)
                       for p in (self.q_proj, self.k_proj, self.v_proj))
        else:
            b, s, _ = x.shape
            q, k, v = (p(x).view(b, s, self.local_heads, self.head_dim) for p in (self.q_proj, self.k_proj, self.v_proj))
        p = self.attn_dropout if self.training else 0.0
        scale = self.head_dim ** -0.5
        if self.use_flash_attn:
            m = attn_mask if attn_mask is None or isinstance(attn_mask, ATT.KeyPaddingMask) else attn_mask.to(q.dtype)
            if p > 0:
                with get_rng_state_tracker().rng_state("local_seed"):
                    o = ATT.attention(q, k, v, causal=False, dropout_p=p, scale=scale, attn_mask=m)
            else:
                o = ATT.attention(q, k, v, causal=False, dropout_p=0.0, scale=scale, attn_mask=m)
        else:
            o = ATT.core_attention(q, k, v, scale, p, self.training, attn_mask=attn_mask, causal=False)
        o = o.reshape(b, s, self.local_heads * self.head_dim)
        if self.sequence_parallel:
            o = o.transpose(0, 1).contiguous()               # [s, b, h/n] -> GEMM -> reduce-scatter along s -> [s/n, b, h]
        return self.out_proj(o)


class TransformerEncoderLayer(nn.Module):
    def __init__(self, hidden, heads, ffn, dropout=0.1, activation="gelu", attn_dropout=None, act_dropout=None, normalize_before=False,
                 mp_group=None, init_std=0.02, dtype=None, device=None, use_flash_attn=True, sequence_parallel=False, fused_tp_comm=False):
        super().__init__()
        self.normalize_before = normalize_before
        sp = sequence_parallel
        self.self_attn = ErnieSelfAttention(hidden, heads, dropout if attn_dropout is None else attn_dropout, mp_group, init_std, dtype, device,
                                            use_flash_attn, sp, fused_tp_comm)
        kw = dict(mp_group=mp_group, init_std=init_std, dtype=dtype, device=device)
        if sp:          # all-gather -> GEMM and GEMM -> reduce-scatter pairs (single fused kernels with Fused.tp_comm)
            self.linear1 = ColumnSequenceParallelLinear(hidden, ffn, gather_output=False, fused_comm=fused_tp_comm, **kw)
            self.linear2 = RowSequenceParallelLinear(ffn, hidden, input_is_parallel=True, fused_comm=fused_tp_comm, **kw)
        else:
            self.linear1 = ColumnParallelLinear(hidden, ffn, gather_output=False, **kw)
            self.linear2 = RowParallelLinear(ffn, hidden, input_is_parallel=True, **kw)
        self.norm1 = LayerNorm(hidden, 1e-12, sp, dtype, device)
        self.norm2 = LayerNorm(hidden, 1e-12, sp, dtype, device)
        # hidden dropout: the same mask on every TP rank for replicated activations, per-rank masks on sequence shards
        self.rng_name = "local_seed" if sp else "global_seed"
        self.dropout_p = dropout
        self.act_dropout_p = dropout if act_dropout is None else act_dropout
        self.activation = activation

    def forward(self, x, attn_mask=None, cache=None, output_attentions=False):
        """Plain call: the layer output.  With a ``cache`` and / or ``output_attentions`` the result is a tuple
        ``(output[, new_cache][, attention_probs])`` like the reference layer (layers/transformer.py:544-620)."""
        detailed = cache is not None or output_attentions
        res = x
        if self.normalize_before:
            x = self.norm1(x)
        if detailed:
            attn, weights, new_cache = self.self_attn.forward_detailed(x, attn_mask, cache, output_attentions)
        else:
            attn = self.self_attn(x, attn_mask)
        x = res + OF.dropout(attn, self.dropout_p, self.training, self.rng_name)
        if not self.normalize_before:
            x = self.norm1(x)
        res = x
        if self.normalize_before:
            x = self.norm2(x)
        h = _ACT[self.activation](self.linear1(x))
        h = OF.dropout(h, self.act_dropout_p, self.training, "local_seed" if self.rng_name == "local_seed" else "global_seed")
        x = res + OF.dropout(self.linear2(h), self.dropout_p, self.training, self.rng_name)
        if not self.normalize_before:
            x = self.norm2(x)
        if not detailed:
            return x
        return (x,) + ((new_cache,) if cache is not None else ()) + ((weights,) if output_attentions else ())

    def gen_cache(self, x):
        return self.self_attn.gen_cache(x)


class TransformerEncoder(nn.Module):
    def __init__(self, layers: List[nn.Module], norm: Optional[nn.Module] = None, use_recompute: bool = False):
        super().__init__()
        self.layers = nn.ModuleList(layers)
        self.norm = norm
        self.use_recompute = use_recompute

    def forward(self, x, attn_mask=None, cache=None, output_attentions=False, output_hidden_states=False, return_dict=False):
        """Default call: the final hidden states (fast path, flash attention).  ``return_dict=True`` returns a
        ``BaseModelOutputWithPastAndCrossAttentions`` with whatever of caches / per-layer hidden states (embedding output first) / attention
        probabilities was asked for; as in the reference (layers/transformer.py:669-760) a non-dict call returns the hidden states only."""
        use_cache = getattr(self, "_use_cache", None)
        if cache is None and use_cache:
            cache = [self.layers[0].gen_cache(x) for _ in self.layers]
        if cache is None and not output_attentions and not output_hidden_states and not return_dict:
            for layer in self.layers:
                if self.use_recompute and self.training:
                    x = recompute(layer, x, attn_mask)
                else:
                    x = layer(x, attn_mask)
            return x if self.norm is None else self.norm(x)
        new_caches = [] if cache is not None and (use_cache is None or use_cache) else None
        attentions = [] if output_attentions else None
        hidden = [x] if output_hidden_states else None
        for i, layer in enumerate(self.layers):
            out = layer(x, attn_mask, None if cache is None else tuple(cache[i]), output_attentions)
            x, extras = (out[0], out[1:]) if isinstance(out, tuple) else (out, ())
            if hidden is not None:
                hidden.append(x)
            if attentions is not None:
                attentions.append(extras[-1])
            if new_caches is not None:
                new_caches.append(tuple(extras[0]))
        if self.norm is not None:
            x = self.norm(x)
            if hidden is not None:
                hidden[-1] = x
        if not return_dict:
            return x
        from .model_outputs import BaseModelOutputWithPastAndCrossAttentions

        return BaseModelOutputWithPastAndCrossAttentions(last_hidden_state=x, past_key_values=new_caches, hidden_states=hidden, attentions=attentions)

    def gen_cache(self, x):
        return [layer.gen_cache(x) for layer in self.layers]


class ErniePooler(nn.Module):
    def __init__(self, hidden, init_std=0.02, dtype=None, device=None):
        super().__init__()
        self.dense = nn.Linear(hidden, hidden, dtype=dtype, device=device)
        with torch.no_grad():
            self.dense.weight.normal_(0.0, init_std); self.dense.bias.zero_()

    def forward(self, hidden_states):
        return torch.tanh(self.dense(hidden_states[:, 0]))


class ErnieModel(nn.Module):
    def __init__(self, vocab_size=40000, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, ffn_hidden_size=None,
                 intermediate_size=None, hidden_act="gelu", hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1,
                 max_position_embeddings=512, type_vocab_size=2, task_type_vocab_size=3, task_id=0, use_task_id=False,
                 initializer_range=0.02, pad_token_id=0, use_recompute=False, mp_group=None, use_flash_attn=True, dtype=None, device=None,
                 num_layers=None, sequence_parallel=False, fused_tp_comm=False, **unused):
        super().__init__()
        # Megatron sequence parallelism over the tensor-parallel group (not in the reference's ERNIE): activations between the GEMM pairs
        # live as [s/n, b, h] shards, so LayerNorm / dropout / residual work and memory drop by n and every TP collective becomes an
        # all-gather or reduce-scatter that the fused compute+collective kernels can absorb (Fused.tp_comm)
        self.sequence_parallel = bool(sequence_parallel) and C.group_size(mp_group) > 1
        sp = self.sequence_parallel
        num_hidden_layers = num_layers or num_hidden_layers
        ffn = ffn_hidden_size or intermediate_size or 4 * hidden_size
        self.pad_token_id, self.initializer_range, self.hidden_size, self.mp_group = pad_token_id, initializer_range, hidden_size, mp_group
        self.vocab_size, self.hidden_act = vocab_size, hidden_act            # read by the heads, as in the reference (single_model.py:464-480)
        self.hidden_dropout_prob = hidden_dropout_prob
        self.embeddings = ErnieEmbeddings(vocab_size, hidden_size, hidden_dropout_prob, max_position_embeddings, type_vocab_size,
                                          task_type_vocab_size, task_id, use_task_id, initializer_range, mp_group, dtype, device)
        layers = [TransformerEncoderLayer(hidden_size, num_attention_heads, ffn, hidden_dropout_prob, hidden_act, attention_probs_dropout_prob,
                                          0, False, mp_group, initializer_range, dtype, device, use_flash_attn, sp, fused_tp_comm)
                  for _ in range(num_hidden_layers)]
        self.encoder = TransformerEncoder(layers, None, use_recompute)
        self.pooler = ErniePooler(hidden_size, initializer_range, dtype, device)

    def get_input_embeddings(self):
        return self.embeddings.word_embeddings

    def set_input_embeddings(self, value):
        self.embeddings.word_embeddings = value

    def forward(self, input_ids=None, token_type_ids=None, position_ids=None, attention_mask=None, task_type_ids=None, past_key_values=None,
                inputs_embeds=None, use_cache=None, output_hidden_states=False, output_attentions=False, return_dict=False):
        """``(sequence_output, pooled_output)``; with ``return_dict=True`` a ``BaseModelOutputWithPoolingAndCrossAttentions`` that also carries
        the requested ``past_key_values`` / ``hidden_states`` / ``attentions`` (argument list of the reference, single_model.py:241-375).
        The training recipes use the first five arguments only and stay on the flash-attention path."""
        if (input_ids is None) == (inputs_embeds is None):
            raise ValueError("You cannot specify both input_ids and inputs_embeds at the same time." if input_ids is not None
                             else "You have to specify either input_ids or inputs_embeds")
        dtype = self.pooler.dense.weight.dtype
        past_len = past_key_values[0][0].shape[2] if past_key_values is not None else None
        detailed = past_key_values is not None or bool(use_cache) or output_hidden_states or output_attentions or return_dict
        if not detailed and attention_mask is None and input_ids is not None:
            attention_mask = ATT.KeyPaddingMask.from_ids(input_ids, self.pad_token_id, dtype)
        elif not detailed and attention_mask is not None and attention_mask.dim() == 2:
            attention_mask = ATT.KeyPaddingMask.from_valid(attention_mask, dtype)
        elif attention_mask is None:
            if input_ids is not None:
                pad = (input_ids == self.pad_token_id)
                attention_mask = pad[:, None, None, :].to(dtype) * -1e4
                if past_len is not None:          # everything already cached is visible
                    attention_mask = torch.cat([attention_mask.new_zeros(attention_mask.shape[0], 1, 1, past_len), attention_mask], dim=-1)
        elif attention_mask.dim() == 2:
            attention_mask = (1.0 - attention_mask[:, None, None, :].to(dtype)) * -1e4
        x = self.embeddings(input_ids, token_type_ids, position_ids, task_type_ids, inputs_embeds, past_len)
        if not detailed:
            if self.sequence_parallel:
                assert x.shape[1] % C.group_size(self.mp_group) == 0, "sequence length must divide by the tensor-parallel degree under sequence parallelism"
                x = C.scatter_seq(x.transpose(0, 1).contiguous(), self.mp_group)          # [b, s, h] -> [s/n, b, h]
            seq = self.encoder(x, attention_mask)
            if self.sequence_parallel:
                seq = C.gather_seq(seq, self.mp_group).transpose(0, 1).contiguous()       # heads and pooler run replicated on the full sequence
            return seq, self.pooler(seq)
        assert not self.sequence_parallel, "caches / per-layer outputs are not available with sequence parallelism"
        self.encoder._use_cache = use_cache
        try:
            enc = self.encoder(x, attention_mask, past_key_values, output_attentions, output_hidden_states, return_dict)
        finally:
            self.encoder._use_cache = None
        if isinstance(enc, torch.Tensor):
            return enc, self.pooler(enc)
        from .model_outputs import BaseModelOutputWithPoolingAndCrossAttentions

        seq = enc[0]
        return BaseModelOutputWithPoolingAndCrossAttentions(last_hidden_state=seq, pooler_output=self.pooler(seq), past_key_values=enc.past_key_values,
                                                            hidden_states=enc.hidden_states, attentions=enc.attentions)


class ErnieLMPredictionHead(nn.Module):
    def __init__(self, hidden, vocab_size, activation="gelu", embedding_weights: Optional[nn.Parameter] = None, mp_group=None, init_std=0.02,
                 dtype=None, device=None):
        super().__init__()
        self.transform = nn.Linear(hidden, hidden, dtype=dtype, device=device)
        with torch.no_grad():
            self.transform.weight.normal_(0.0, init_std); self.transform.bias.zero_()
        self.activation = activation
        self.layer_norm = LayerNorm(hidden, 1e-12, False, dtype, device)
        self.mp_group = mp_group
        world = C.group_size(mp_group)
        self.decoder_weight = embedding_weights if embedding_weights is not None else nn.Parameter(
            torch.empty(vocab_size // world, hidden, dtype=dtype, device=device).normal_(0.0, init_std))
        self.decoder_bias = nn.Parameter(torch.zeros(vocab_size // world, dtype=dtype, device=device))
        self.decoder_bias.tp_sharded = world > 1
        self.decoder_bias.split_axis = 0

    def forward(self, hidden_states, masked_positions=None):
        if masked_positions is not None:
            hidden_states = hidden_states.reshape(-1, hidden_states.shape[-1]).index_select(0, masked_positions.reshape(-1).long())
        h = self.layer_norm(_ACT[self.activation](self.transform(hidden_states)))
        return parallel_matmul(h, self.decoder_weight, self.mp_group, parallel_output=True) + self.decoder_bias


class ErniePretrainingHeads(nn.Module):
    def __init__(self, hidden, vocab_size, activation, embedding_weights=None, mp_group=None, init_std=0.02, binary_head=True, dtype=None,
                 device=None):
        super().__init__()
        self.predictions = ErnieLMPredictionHead(hidden, vocab_size, activation, embedding_weights, mp_group, init_std, dtype, device)
        self.seq_relationship = nn.Linear(hidden, 2, dtype=dtype, device=device) if binary_head else None

    def forward(self, sequence_output, pooled_output, masked_positions=None):
        scores = self.predictions(sequence_output, masked_positions)
        rel = self.seq_relationship(pooled_output) if self.seq_relationship is not None else None
        return scores, rel


class ErnieForPretraining(nn.Module):
    def __init__(self, ernie: ErnieModel, vocab_size: Optional[int] = None, hidden_act: Optional[str] = None, binary_head: bool = True):
        super().__init__()
        self.ernie = ernie
        vocab_size = vocab_size or ernie.vocab_size                  # reference signature: ErnieForPretraining(ernie)
        hidden_act = hidden_act or ernie.hidden_act
        p = ernie.pooler.dense.weight
        self.cls = ErniePretrainingHeads(ernie.hidden_size, vocab_size, hidden_act, ernie.embeddings.word_embeddings.weight, ernie.mp_group,
                                         ernie.initializer_range, binary_head, p.dtype, p.device)

    def forward(self, input_ids=None, token_type_ids=None, position_ids=None, attention_mask=None, masked_positions=None, inputs_embeds=None,
                labels=None, next_sentence_label=None, output_hidden_states=False, output_attentions=False, return_dict=False):
        """``(prediction_scores, seq_relationship_score)`` — what the training module consumes.  With ``labels`` and ``next_sentence_label``
        the summed MLM + sentence-order loss is prepended; ``return_dict=True`` gives an ``ErnieForPreTrainingOutput``
        (reference single_model.py:486-560)."""
        if inputs_embeds is None and labels is None and not (output_hidden_states or output_attentions or return_dict):
            seq, pooled = self.ernie(input_ids, token_type_ids, position_ids, attention_mask)
            return self.cls(seq, pooled, masked_positions)
        outputs = self.ernie(input_ids, token_type_ids, position_ids, attention_mask, inputs_embeds=inputs_embeds,
                             output_hidden_states=output_hidden_states, output_attentions=output_attentions, return_dict=return_dict)
        scores, rel = self.cls(outputs[0], outputs[1], masked_positions)
        loss = None
        if labels is not None and next_sentence_label is not None:
            full = C.gather_last_dim(scores, self.ernie.mp_group) if C.group_size(self.ernie.mp_group) > 1 else scores
            loss = F.cross_entropy(full.reshape(-1, full.shape[-1]).float(), labels.reshape(-1).long()) \
                + F.cross_entropy(rel.reshape(-1, 2).float(), next_sentence_label.reshape(-1).long())
        if not return_dict:
            out = (scores, rel) + tuple(outputs[2:])
            return ((loss,) + out) if loss is not None else out
        from .model_outputs import ErnieForPreTrainingOutput

        return ErnieForPreTrainingOutput(loss=loss, prediction_logits=scores, seq_relationship_logits=rel, hidden_states=outputs.hidden_states,
                                         attentions=outputs.attentions)


ErnieForPretrainingHybrid = ErnieForPretraining
ErnieModelHybrid = ErnieModel


class ErniePretrainingCriterion(nn.Module):
    """MLM loss (mean over labels != -1, vocab-parallel CE) + optional SOP loss."""

    def __init__(self, with_nsp_loss: bool = True, mp_group=None):
        super().__init__()
        self.with_nsp_loss = with_nsp_loss
        self.ce = ParallelCrossEntropy(mp_group)

    def forward(self, prediction_scores, seq_relationship_score, masked_lm_labels, next_sentence_labels=None):
        labels = masked_lm_labels.reshape(-1).long()
        valid = labels >= 0
        per_tok = self.ce(prediction_scores.reshape(-1, prediction_scores.shape[-1]).contiguous(), labels.clamp(min=0))
        mlm = (per_tok * valid.float()).sum() / valid.float().sum().clamp(min=1.0)
        if not self.with_nsp_loss or seq_relationship_score is None or next_sentence_labels is None:
            return mlm
        sop = F.cross_entropy(seq_relationship_score.float(), next_sentence_labels.reshape(-1).long())
        return mlm + sop, mlm, sop


class ErnieForSequenceClassification(nn.Module):
    def __init__(self, ernie: ErnieModel, num_classes: int = 2, dropout: Optional[float] = None):
        super().__init__()
        self.ernie = ernie
        p = ernie.pooler.dense.weight
        self.dropout_p = getattr(ernie, "hidden_dropout_prob", 0.1) if dropout is None else dropout      # reference single_model.py:664-666
        self.num_classes = num_classes
        self.classifier = nn.Linear(ernie.hidden_size, num_classes, dtype=p.dtype, device=p.device)
        with torch.no_grad():
            self.classifier.weight.normal_(0.0, ernie.initializer_range); self.classifier.bias.zero_()

    def forward(self, input_ids=None, token_type_ids=None, position_ids=None, attention_mask=None, inputs_embeds=None, labels=None,
                output_hidden_states=False, output_attentions=False, return_dict=False):
        """The logits; ``labels`` adds the loss in front (MSE for one class, cross entropy for integer labels, BCE-with-logits for float
        multi-label targets) and ``return_dict=True`` gives a ``SequenceClassifierOutput`` (reference single_model.py:672-735)."""
        outputs = self.ernie(input_ids, token_type_ids, position_ids, attention_mask, inputs_embeds=inputs_embeds,
                             output_hidden_states=output_hidden_states, output_attentions=output_attentions, return_dict=return_dict)
        logits = self.classifier(OF.dropout(outputs[1], self.dropout_p, self.training, "global_seed"))
        loss = None
        if labels is not None:
            if self.num_classes == 1:
                loss = F.mse_loss(logits.float(), labels.to(torch.float32))
            elif labels.dtype in (torch.int64, torch.int32):
                loss = F.cross_entropy(logits.reshape(-1, self.num_classes).float(), labels.reshape(-1).long())
            else:
                loss = F.binary_cross_entropy_with_logits(logits.float(), labels.to(torch.float32))
        if not return_dict:
            out = (logits,) + tuple(outputs[2:])
            return ((loss,) + out) if loss is not None else (out[0] if len(out) == 1 else out)
        from .model_outputs import SequenceClassifierOutput

        return SequenceClassifierOutput(loss=loss, logits=logits, hidden_states=outputs.hidden_states, attentions=outputs.attentions)


# ---------------------------------------------------------------------------------------------------------------------------------------
# Names of the reference's split files (ernie/dygraph/hybrid_model.py, ernie/auto/auto_model.py, ernie/layers/*transformer.py) that resolve
# to this module: the tensor-parallel / auto-parallel variants are the same classes (the layers are topology-aware).
ErniePretrainingCriterionHybrid = ErniePretrainingCriterion
ErnieForSequenceClassificationHybrid = ErnieForSequenceClassification
ErnieModelAuto = ErnieModel
ErnieForPretrainingAuto = ErnieForPretraining
ErniePretrainingCriterionAuto = ErniePretrainingCriterion
ErnieForSequenceClassificationAuto = ErnieForSequenceClassification
MultiHeadAttention = ErnieSelfAttention


class Embedding(nn.Embedding):
    """Embedding table with the reference constructor (ernie/auto/auto_model.py:37-95: ``padding_idx`` may be negative, ``sparse`` gradients,
    validated sizes); the row of ``padding_idx`` stays zero and receives no gradient."""

    def __init__(self, num_embeddings, embedding_dim, padding_idx=None, sparse=False, weight_attr=None, name=None, dtype=None, device=None):
        if num_embeddings <= 0:
            raise ValueError("num_embeddings must be gather than 0")
        if embedding_dim <= 0:
            raise ValueError("embedding_dim must be gather than 0")
        if padding_idx is not None and not -num_embeddings <= padding_idx < num_embeddings:
            raise ValueError(f"padding_idx must be within [-{num_embeddings}, {num_embeddings})")
        super().__init__(num_embeddings, embedding_dim, padding_idx=padding_idx, sparse=bool(sparse), dtype=dtype, device=device)


class LayerNormPipe(LayerNorm):
    """Final norm as a pipeline stage entry (reference hybrid_model.py:761-765): takes and returns the hidden states only."""

    def forward(self, x, *rest):
        return super().forward(x)


class ErniePoolerPipe(ErniePooler):
    """Pooler as a pipeline stage entry (reference hybrid_model.py:768-772): ``hidden -> (hidden, pooled)``."""

    def forward(self, hidden_states, *rest):
        return hidden_states, super().forward(hidden_states)


from ....utils.lazy import lazy_exports  # noqa: E402

__getattr__ = lazy_exports(__name__, {
    "EmbeddingsPipe": ".pipe", "TransformerEncoderLayerPipe": ".pipe", "ErniePretrainingCriterionPipe": ".pipe", "ErnieForPretrainingPipe": ".pipe",
})
