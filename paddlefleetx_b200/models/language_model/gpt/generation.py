"""``GPTForGeneration`` — sampling / greedy decoding with a static KV cache.

Semantics follow the reference's ``sample`` loop (gpt/dygraph/hybrid_model.py:1453-1678, single_model.py:1139-1419):
left-padded prompts, logits processors -> temperature -> top-k filter -> top-p -> multinomial, per-sequence
``unfinished`` flags, pad emitted after EOS, score = mean log-prob of the chosen tokens, ``max_dec_len`` budget.

B200-first changes: the cache is pre-allocated (no per-token concat), top-p sampling runs in the fused ``topp_sampling``
kernel (no vocabulary sort), the "all sequences finished?" host check is amortised over ``sync_every`` steps, and
the single-token decode step is CUDA-graph capturable (``ops/decode_graph.py``).
"""
from __future__ import annotations

from typing import Optional, Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from ....ops import attention as ATT
from ....ops import functional as OF
from ....parallel.tp_layers import parallel_matmul
from . import model as gpt
from .processor import (ForcedBOSTokenLogitsProcessor, ForcedEOSTokenLogitsProcessor, HammingDiversityLogitsProcessor,
                        LogitsProcessorList, MinLengthLogitsProcessor, RepetitionPenaltyLogitsProcessor)


def top_k_filter(probs: torch.Tensor, top_k: int, min_tokens_to_keep: int = 1) -> torch.Tensor:
    k = min(max(int(top_k), min_tokens_to_keep), probs.shape[-1])
    kth = torch.topk(probs, k, dim=-1).values[:, -1:]
    return torch.where(probs >= kth, probs, torch.zeros_like(probs))


def top_p_filter(probs: torch.Tensor, top_p: float, min_tokens_to_keep: int = 1) -> torch.Tensor:
    sp, si = probs.sort(-1, descending=True)
    remove = sp.cumsum(-1) > top_p
    if min_tokens_to_keep > 1:
        remove[:, :min_tokens_to_keep - 1] = False
    remove[:, 1:] = remove[:, :-1].clone()
    remove[:, 0] = False
    mask = torch.zeros_like(remove).scatter(1, si, remove)
    return torch.where(mask, torch.zeros_like(probs), probs)


class GPTForGeneration(nn.Module):
    def __init__(self, gpt_model: gpt.GPTModel, configs=None, **overrides):
        super().__init__()
        self.gpt = gpt_model
        cfg = dict(configs or {})
        cfg.update(overrides)
        self.max_length = int(cfg.get("max_dec_len", 20))
        self.min_length = int(cfg.get("min_dec_len", 0))
        self.decode_strategy = cfg.get("decode_strategy", "sampling")
        self.temperature = float(cfg.get("temperature", 1.0))
        self.top_k = int(cfg.get("top_k", 0) or 0)
        self.top_p = float(cfg.get("top_p", 1.0) or 1.0)
        self.repetition_penalty = float(cfg.get("repetition_penalty", 1.0))
        self.num_beams = int(cfg.get("num_beams", 1))
        self.num_beam_groups = int(cfg.get("num_beam_groups", 1))
        self.length_penalty = float(cfg.get("length_penalty", 0.0))
        self.early_stopping = bool(cfg.get("early_stopping", False))
        self.bos_token_id = cfg.get("bos_token_id")
        self.eos_token_id = cfg.get("eos_token_id", 50256)
        self.pad_token_id = cfg.get("pad_token_id", self.eos_token_id)
        self.num_return_sequences = int(cfg.get("num_return_sequences", 1))
        self.diversity_rate = float(cfg.get("diversity_rate", 0.0))
        self.forced_bos_token_id = cfg.get("forced_bos_token_id")
        self.forced_eos_token_id = cfg.get("forced_eos_token_id")
        self.use_topp_sampling = bool(cfg.get("use_topp_sampling", True))
        self.sync_every = int(cfg.get("sync_every", 8))
        self.max_dec_len_limit = int(cfg.get("max_dec_len_limit", 512))
        # decode steps replayed from a CUDA graph (static KV cache + masked full-length attention); reference decodes eagerly
        self.use_cuda_graph = bool(cfg.get("use_cuda_graph", True))
        self._graphs = {}
        self._force_static = bool(cfg.get("force_static_decode", False))   # exercise the static-cache step without a GPU (tests)
        if self.decode_strategy not in ("sampling", "greedy_search"):
            raise ValueError(f"decode_strategy {self.decode_strategy!r} is not implemented (sampling | greedy_search); "
                             "the reference accepts beam_search in its validator and then rejects it as well")

    # -------------------------------------------------------------------------------------------------
    def get_logits_processor(self, min_length, max_length, eos_token_id, forced_bos_token_id=None, forced_eos_token_id=None,
                             num_beams=1, num_beam_groups=1, diversity_rate=0.0, repetition_penalty=None) -> LogitsProcessorList:
        procs = LogitsProcessorList()
        if min_length is not None and eos_token_id is not None and min_length > -1:
            procs.append(MinLengthLogitsProcessor(min_length, eos_token_id))
        if num_beam_groups > 1 and diversity_rate > 0.0:
            procs.append(HammingDiversityLogitsProcessor(diversity_rate, num_beams, num_beam_groups))
        if repetition_penalty is not None and repetition_penalty != 1.0:
            procs.append(RepetitionPenaltyLogitsProcessor(repetition_penalty))
        if forced_bos_token_id is not None:
            procs.append(ForcedBOSTokenLogitsProcessor(forced_bos_token_id))
        if forced_eos_token_id is not None:
            procs.append(ForcedEOSTokenLogitsProcessor(max_length, forced_eos_token_id))
        return procs

    def _lm_logits(self, hidden_last: torch.Tensor) -> torch.Tensor:
        return parallel_matmul(hidden_last, self.gpt.embeddings.word_embeddings.weight, self.gpt.mp_group, parallel_output=False)

    @staticmethod
    def _prompt_masks(input_ids: torch.Tensor, pad_token_id, attention_mask: Optional[torch.Tensor]):
        b, s = input_ids.shape
        if attention_mask is None:
            valid = (input_ids != pad_token_id) if pad_token_id is not None else torch.ones_like(input_ids, dtype=torch.bool)
            if pad_token_id is not None and bool((input_ids[:, -1] == pad_token_id).any()):
                valid = torch.ones_like(input_ids, dtype=torch.bool)      # right-padded / eos-as-pad prompts: attend to everything
        else:
            valid = attention_mask.reshape(b, -1)[:, -s:].bool()
        position_ids = (valid.long().cumsum(-1) - 1).clamp(min=0)
        return valid, position_ids

    @torch.no_grad()
    def forward(self, input_ids: torch.Tensor, attention_mask: Optional[torch.Tensor] = None, position_ids: Optional[torch.Tensor] = None,
                seed: Optional[int] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        return self.generate(input_ids, attention_mask, position_ids, seed)

    @torch.no_grad()
    def generate(self, input_ids, attention_mask=None, position_ids=None, seed: Optional[int] = None):
        """Decode ``max_length`` new tokens for a batch of (left-padded) prompts: prefill once into the static KV cache, then one token per step —
        logits processors (min length, repetition penalty, forced BOS / EOS), temperature, top-k / top-p sampling (native radix-descent sampler on
        CUDA) or greedy search; the single-token step is replayed from a CUDA graph when enabled.  Returns ``(generated ids, scores)``
        (reference single_model.py:898-1320)."""
        self.gpt.eval()
        if self.num_return_sequences > 1:
            input_ids = input_ids.repeat_interleave(self.num_return_sequences, 0)
            attention_mask = attention_mask.repeat_interleave(self.num_return_sequences, 0) if attention_mask is not None else None
        b, prompt_len = input_ids.shape
        dev = input_ids.device
        max_new = min(self.max_length, self.max_dec_len_limit)
        total_len = prompt_len + max_new
        procs = self.get_logits_processor(self.min_length + prompt_len if self.min_length else None, total_len, self.eos_token_id,
                                          self.forced_bos_token_id, self.forced_eos_token_id, self.num_beams, self.num_beam_groups,
                                          self.diversity_rate, self.repetition_penalty)
        valid, pos = self._prompt_masks(input_ids, self.pad_token_id, attention_mask)
        if position_ids is not None:
            pos = position_ids
        graph_state = self._graph_state(b, total_len, dev) if (self.use_cuda_graph and (dev.type == "cuda" or self._force_static) and self.gpt.mp_group is None) else None
        if graph_state is not None:
            caches = graph_state["caches"]
            for c in caches:
                c.reset()
        else:
            caches = self.gpt.new_caches(b, total_len)
        key_valid = torch.zeros(b, total_len, dtype=torch.bool, device=dev)
        key_valid[:, :prompt_len] = valid
        # prefill: causal + padding mask
        causal = torch.ones(prompt_len, prompt_len, dtype=torch.bool, device=dev).tril()
        mask = (causal.unsqueeze(0) & valid.unsqueeze(1)).unsqueeze(1)                 # [b,1,s,s] bool (True = attend)
        mask = mask | torch.eye(prompt_len, dtype=torch.bool, device=dev)              # padded rows still need one key
        # unpadded prompts (the common serving case) need no explicit mask: plain causal attention runs on the native flash kernel;
        # left-padded ones run it too, under a document mask (see _left_padded_mask)
        prefill_mask = None
        if not (attention_mask is None and bool(valid.all())):
            prefill_mask = _left_padded_mask(valid)
            if prefill_mask is None:
                prefill_mask = _to_additive(mask, hidden_dtype(self.gpt))
        hidden = self.gpt(input_ids, pos, prefill_mask, caches)
        logits = self._lm_logits(hidden[:, -1:, :])[:, 0, :].float()

        out_ids = torch.full((b, max_new), int(self.pad_token_id if self.pad_token_id is not None else 0), dtype=torch.long, device=dev)
        unfinished = torch.ones(b, 1, dtype=torch.bool, device=dev)
        scores = torch.zeros(b, 1, dtype=torch.float32, device=dev)
        all_ids = input_ids
        next_pos = pos[:, -1:] + 1
        gen = None
        if seed is not None:
            gen = torch.Generator(device=dev)
            gen.manual_seed(int(seed))
        steps_done = 0
        for step in range(max_new):
            logits = procs(all_ids, logits)
            logp = F.log_softmax(logits, -1)
            if self.decode_strategy == "greedy_search":
                next_tok = logits.argmax(-1, keepdim=True)
            else:
                scaled = logits / self.temperature if self.temperature != 1.0 else logits
                probs = F.softmax(scaled, -1)
                if self.top_k:
                    probs = top_k_filter(probs, self.top_k)
                if self.top_p < 1.0 and self.use_topp_sampling:
                    probs = probs / probs.sum(-1, keepdim=True)
                    tp = torch.full((b,), self.top_p, device=dev)
                    _, next_tok = OF.topp_sampling(probs, tp, seed=-1 if seed is None else int(seed), offset=None if seed is None else step * b)
                else:
                    if self.top_p < 1.0:
                        probs = top_p_filter(probs, self.top_p)
                    next_tok = torch.multinomial(probs, 1, generator=gen)
            next_score = logp.gather(1, next_tok)
            if self.eos_token_id is not None:
                next_tok = torch.where(unfinished, next_tok, torch.full_like(next_tok, int(self.pad_token_id)))
            scores = torch.where(unfinished, (scores * step + next_score) / (step + 1), scores)
            out_ids[:, step:step + 1] = next_tok
            all_ids = torch.cat([all_ids, next_tok], 1)
            if self.eos_token_id is not None:
                unfinished = unfinished & (next_tok != self.eos_token_id)
            steps_done = step + 1
            if step == max_new - 1:
                break
            if (step + 1) % self.sync_every == 0 and not bool(unfinished.any()):     # amortised host check
                break
            key_valid[:, prompt_len + step] = True
            cur = prompt_len + step + 1
            if graph_state is not None:
                logits = self._graph_decode(graph_state, next_tok, next_pos, key_valid, prompt_len + step)
            else:
                dmask = _to_additive(key_valid[:, :cur].view(b, 1, 1, cur), hidden_dtype(self.gpt))
                hidden = self.gpt(next_tok, next_pos, dmask, caches)
                logits = self._lm_logits(hidden)[:, 0, :].float()
            next_pos = next_pos + 1
        return out_ids[:, :steps_done], scores


def _graph_methods():
    """CUDA-graph decode: one captured step = embeddings + all layers (KV written at a device-side index, attention over the whole
    static cache with an additive validity mask) + LM head.  Captured lazily per (batch, total_len); replays cost one launch."""

    def _graph_state(self, b: int, total_len: int, dev):
        key = (b, total_len)
        st = self._graphs.get(key)
        if st is None:
            dt = hidden_dtype(self.gpt)
            st = {"caches": self.gpt.new_caches(b, total_len), "graph": None,
                  "tok": torch.zeros(b, 1, dtype=torch.long, device=dev), "pos": torch.zeros(b, 1, dtype=torch.long, device=dev),
                  "idx": torch.zeros(1, dtype=torch.long, device=dev), "mask": torch.zeros(b, 1, 1, total_len, dtype=dt, device=dev),
                  "logits": None}
            if len(self._graphs) >= 4:                      # bound the memory held by stale shapes
                self._graphs.pop(next(iter(self._graphs)))
            self._graphs[key] = st
        return st

    def _decode_static(self, st):
        hidden = self.gpt(st["tok"], st["pos"], st["mask"], st["caches"])
        return self._lm_logits(hidden)[:, 0, :].float()

    def _graph_decode(self, st, next_tok, next_pos, key_valid, write_index: int):
        st["tok"].copy_(next_tok)
        st["pos"].copy_(next_pos)
        st["idx"].fill_(write_index)
        st["mask"].copy_(_to_additive(key_valid.view(key_valid.shape[0], 1, 1, -1), st["mask"].dtype))
        for c in st["caches"]:
            c.static_index = st["idx"]
        if st["tok"].device.type != "cuda":
            return self._decode_static(st)
        if st["graph"] is None:
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):                    # warm-up outside capture (lazy inits, autotune-free but allocates)
                self._decode_static(st)
            torch.cuda.current_stream().wait_stream(side)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                st["logits"] = self._decode_static(st)
            st["graph"] = g
        st["graph"].replay()
        return st["logits"]

    return _graph_state, _decode_static, _graph_decode


GPTForGeneration._graph_state, GPTForGeneration._decode_static, GPTForGeneration._graph_decode = _graph_methods()


def hidden_dtype(model: gpt.GPTModel):
    return model.decoder.norm.weight.dtype


def _left_padded_mask(valid: torch.Tensor) -> Optional[ATT.DocumentMask]:
    """The prefill mask ``causal & valid | eye`` of a LEFT-padded batch as a document mask: a valid query attends from its row's first
    valid key, a padding query only itself (key_start = i).  ``None`` for any other validity pattern (right or interior padding)."""
    s = valid.shape[1]
    if s > 1 and not bool((valid[:, 1:] >= valid[:, :-1]).all()):
        return None
    i = torch.arange(s, device=valid.device)
    first = s - valid.sum(-1, keepdim=True)
    return ATT.DocumentMask.from_key_start(torch.where(valid, first, i))


def _to_additive(bool_mask: torch.Tensor, dtype) -> torch.Tensor:
    return torch.zeros(bool_mask.shape, dtype=dtype, device=bool_mask.device).masked_fill(~bool_mask, -1e4)


GPTForGenerationHybrid = GPTForGeneration
