"""Language-model task modules: ``GPTModule`` (pre-training), ``GPTFinetuneModule`` (GLUE sequence
classification), ``GPTGenerationModule``, ``GPTEvalModule`` (WikiText ppl / LAMBADA cloze) and ``MoEModule``.

Behaviour reference: ppfleetx/models/language_model/language_module.py:73-830 and utils.py:39-180 (config
post-processing: ``ffn = 4h``, recompute defaults, ``decay_steps *= global_batch_size``, ``num_samples`` baked
into the dataset block, ``multi_precision = amp.enable``).  The canonical ``[train] ... ips_total: N tokens/s``
log line is kept verbatim because the TIPC-style harness greps it.
"""
from __future__ import annotations

import copy
from typing import Optional

import torch

from ...core.module.basic_module import BasicModule
from ...distributed.apis import env
from ...parallel.tp_layers import register_sequence_parallel_allreduce_hooks
from ...utils.log import logger
from .gpt import model as gpt


# ------------------------------------------------------------------------------------ config post-processing
def is_fused_matmul_bias_supported() -> bool:
    """The reference probes for cuBLASLt's fused GEMM epilogue (language_model/utils.py); here bias / GELU epilogues are part of the native
    tcgen05 GEMM, so the answer is whether the native library is usable on this machine."""
    from ...ops import functional as OF

    return bool(OF.native_available())


def process_data_configs(config) -> None:
    g, eng = config.Global, config.Engine
    eval_freq = eng.eval_freq if eng.eval_freq and eng.eval_freq > 0 else max(eng.max_steps, 1)
    n = {"Train": g.global_batch_size * eng.max_steps,
         "Eval": g.global_batch_size * (eng.max_steps // eval_freq + 1) * eng.eval_iters,
         "Test": g.global_batch_size * eng.test_iters}
    for mode in ("Train", "Eval", "Test"):
        if mode in config.get("Data", {}):
            ds = config.Data[mode].dataset
            ds["num_samples"] = n[mode]
            ds["mode"] = mode
            ds["seed"] = g.seed
            ds["model_type"] = config.Model.get("name", "GPT")
            if ds.get("name") == "SyntheticGPTDataset":
                ds.setdefault("vocab_size", config.Model.get("vocab_size", 50304))
            config.Data[mode].sampler["batch_size"] = g.local_batch_size


def process_model_configs(config) -> None:
    m = config.Model
    if m.get("ffn_hidden_size") is None:
        m["ffn_hidden_size"] = gpt.swiglu_ffn_size(m["hidden_size"]) if m.get("ffn_activation") == "swiglu" else 4 * m["hidden_size"]
    if m.get("use_recompute"):
        if not m.get("recompute_granularity"):
            m["recompute_granularity"] = "full"
        nrl = m.get("no_recompute_layers") or []
        assert isinstance(nrl, list) and all(isinstance(i, int) for i in nrl), "no_recompute_layers should be a list of ints"
        if nrl:
            assert min(nrl) >= 0 and max(nrl) < m["num_layers"], "no_recompute_layers out of range"
        m["no_recompute_layers"] = sorted(set(nrl))
    pp = config.Distributed.pp_degree
    if pp > 1:
        vpp = m.get("virtual_pp_degree") or 1
        m["virtual_pp_degree"] = vpp
        if m["num_layers"] % (vpp * pp) != 0:
            assert vpp == 1, "virtual pp doesn't support uneven layer split."
            logger.warning(f"num_layers {m['num_layers']} is not divisible by pp_degree {pp}")
        if vpp > 1:
            acc = config.Global.local_batch_size // config.Global.micro_batch_size
            assert acc % pp == 0, f"num of microbatches {acc} should be divisible of pp_degree {pp} when using interleave pipeline"
    elif m.get("virtual_pp_degree"):
        logger.warning("virtual_pp_degree is unuseful.")


def process_optim_configs(config) -> None:
    opt = config.Optimizer
    opt["multi_precision"] = bool(config.Engine.mix_precision.enable)
    lr = opt.get("lr")
    if lr is not None and "decay_steps" in lr:
        if lr.get("decay_steps") is None:
            lr["decay_steps"] = config.Engine.max_steps
        if not lr.get("_scaled_by_batch", False):
            lr["decay_steps"] *= config.Global.global_batch_size
            lr["_scaled_by_batch"] = True


def process_inference_configs(config) -> None:
    inf = config.get("Inference")
    if not inf:
        return
    if inf.get("model_dir") is None:
        inf["model_dir"] = config.Engine.save_load.output_dir
    if inf.get("mp_degree") is None:
        inf["mp_degree"] = config.Distributed.mp_degree


def process_configs(config):
    process_data_configs(config)
    process_model_configs(config)
    process_optim_configs(config)
    process_inference_configs(config)
    return config


def get_model_size(l: int, h: int, v: int, s: int, kv_hidden: Optional[int] = None, ffn: Optional[int] = None,
                   ffn_activation: str = "gelu") -> float:
    """Parameter count; ``kv_hidden`` = K/V heads x head_dim (grouped-query attention), default ``h``: QKV is h (h + 2 kv_hidden).  ``ffn``
    is the FFN width F (default 4h): 2hF + F + h parameters under GELU, 3hF + 2F + h under SwiGLU (``linear1`` is [2F, h])."""
    kv = h if kv_hidden is None else kv_hidden
    f = 4 * h if ffn is None else ffn
    ffn_params = (3 * h * f + 2 * f + h) if ffn_activation == "swiglu" else (2 * h * f + f + h)
    p = (v + s) * h + (2 * h * h + 2 * h * kv + 2 * h + 2 * kv) * l + (2 * (2 * h)) * l + ffn_params * l + 2 * h
    logger.info("Model Size: {:.2f} B".format(p / 1e9))
    return p


_MODEL_KEYS = ("vocab_size", "hidden_size", "num_layers", "num_attention_heads", "ffn_hidden_size", "hidden_dropout_prob",
               "attention_probs_dropout_prob", "max_position_embeddings", "type_vocab_size", "initializer_range", "use_recompute",
               "recompute_granularity", "no_recompute_layers", "fused_linear", "fuse_attn_qkv", "scale_qk_by_layer_num",
               "sequence_parallel", "use_flash_attn", "fused_softmax_with_triangular", "moe_configs", "use_rope", "normalization", "virtual_pp_degree",
               "num_key_value_heads", "ffn_activation", "reset_attention_mask")


def model_kwargs(config) -> dict:
    return {k: config.Model[k] for k in _MODEL_KEYS if k in config.Model and config.Model[k] is not None}


def _param_dtype(config):
    amp = config.Engine.mix_precision
    if amp.get("enable") and str(amp.get("level", "O2")).upper() == "O2" and str(config.Global.get("device", "gpu")) == "gpu" \
            and torch.cuda.is_available():
        return torch.bfloat16 if str(amp.get("dtype", "float16")) == "bfloat16" else torch.float16
    return torch.float32


def _device(config):
    return torch.device("cuda", torch.cuda.current_device()) if str(config.Global.get("device", "gpu")) == "gpu" and torch.cuda.is_available() \
        else torch.device("cpu")


# ------------------------------------------------------------------------------------ modules
class LanguageModule(BasicModule):
    def __init__(self, configs):
        from ...parallel import tp_layers as _tp

        _tp.configure(configs.get("Fused", {}))
        self.nranks = env.world_size()
        self.data_world_size = env.get_data_world_size()
        super().__init__(configs)
        self.loss_fn = self.get_loss_fn()

    def process_configs(self, configs):
        return process_configs(configs)

    def forward(self, tokens, ids):
        return self.model(tokens, ids)

    def _context_parallel_slice(self, batch):
        """``Distributed.cp_degree`` > 1: the ranks of a context-parallel group receive the same batch; each keeps its contiguous slice of the
        sequence (tokens, GLOBAL position ids, labels, loss mask).  Attention re-assembles the sequence per head group (Ulysses)."""
        from ...distributed.apis import env as _env

        hcg = getattr(_env, "_hcg", None)
        c = getattr(hcg, "cp", 1) if hcg is not None else 1
        if c == 1:
            return batch
        r = hcg.get_context_parallel_rank()
        if getattr(hcg, "cp_mode", "ulysses") == "ring":          # chunks r and 2c-1-r of 2c: equal causal work on every rank at every ring step
            from ...parallel.ring_attention import zigzag_slice

            return [zigzag_slice(t, c, r, dim=1).contiguous() for t in batch]
        assert batch[0].shape[1] % c == 0, f"sequence length {batch[0].shape[1]} % cp_degree {c}"
        return [t.chunk(c, dim=1)[r].contiguous() for t in batch]

    def _context_parallel_loss(self, loss, loss_mask):
        """The criterion divides by THIS rank's mask count; the gradient reduction then averages the cp ranks.  With an uneven mask (padding,
        masked-out EOS) the mean of the ranks' masked means is not the masked mean over the whole sequences, so rescale by
        ``local count x c / group count``: the average over the group becomes ``sum(CE x mask) / sum(mask)`` exactly."""
        from ...distributed.apis import env as _env

        hcg = getattr(_env, "_hcg", None)
        c = getattr(hcg, "cp", 1) if hcg is not None else 1
        if c == 1:
            return loss
        pg = hcg.get_context_parallel_group().process_group
        local = loss_mask.detach().float().sum()
        total = local.clone()
        torch.distributed.all_reduce(total, group=pg)
        scaled = loss * (local * c / total)
        # report the loss of the whole sequences on every rank of the group (what a run without cp logs); the gradient stays this shard's
        mean = scaled.detach().clone()
        torch.distributed.all_reduce(mean, group=pg)
        return scaled + (mean / c - scaled.detach())

    def training_step(self, batch):
        tokens, position_ids, labels, loss_mask = self._context_parallel_slice(batch)
        preds = self(tokens, position_ids)
        return self._context_parallel_loss(self.loss_fn(preds, labels, loss_mask), loss_mask)

    def training_step_end(self, log_dict):
        speed = 1.0 / log_dict["train_cost"]
        tokens = self.configs.Global.global_batch_size * self.configs.Data.Train.dataset.max_seq_len
        ls = "loss_scale: %.9f," % log_dict["loss_scale"] if log_dict.get("loss_scale") is not None else ""
        logger.train(
            "[train] epoch: [%d/%d], batch: [%d/%d], loss: %.9f, avg_batch_cost: %.5f sec, speed: %.2f step/s, "
            "ips_total: %.0f tokens/s, ips: %.0f tokens/s, %s learning rate: %.5e, found_inf: %.0f"
            % (log_dict["epoch"], log_dict["total_epoch"], log_dict["batch"], log_dict["total_step"], log_dict["loss"],
               log_dict["train_cost"], speed, speed * tokens, speed * tokens / self.data_world_size, ls, log_dict["lr"],
               log_dict["found_inf"]))

    def validation_step(self, batch):
        tokens, position_ids, labels, loss_mask = self._context_parallel_slice(batch)
        preds = self(tokens, position_ids)
        return self._context_parallel_loss(self.loss_fn(preds, labels, loss_mask), loss_mask)

    def validation_step_end(self, log_dict):
        speed = 1.0 / log_dict["eval_cost"]
        logger.eval("[eval] epoch: %d, batch: %d/%d, loss: %.9f, avg_eval_cost: %.5f sec, speed: %.2f step/s"
                    % (log_dict["epoch"], log_dict["batch"], log_dict["total_batch"], log_dict["loss"], log_dict["eval_cost"], speed))

    def test_step(self, batch):
        return self.validation_step(batch)

    def test_step_end(self, log_dict):
        speed = 1.0 / log_dict["test_cost"]
        logger.eval("[test] epoch: %d, batch: %d, loss: %.9f, avg_test_cost: %.5f sec, speed: %.2f step/s"
                    % (log_dict["epoch"], log_dict["batch"], log_dict["loss"], log_dict["test_cost"], speed))

    def training_epoch_end(self, log_dict):
        logger.info("[Training] epoch: %d, total time: %.5f sec" % (log_dict["epoch"], log_dict["train_cost"]))


class GPTModule(LanguageModule):
    """world == 1 -> plain GPT; pp == 1 -> TP/SP-aware GPT; pp > 1 -> ``GPTForPretrainingPipe``
    (reference language_module.py:148-225)."""

    def __init__(self, configs):
        super().__init__(configs)
        d = configs.Distributed
        if configs.Model.get("sequence_parallel", False) and d.mp_degree > 1:
            register_sequence_parallel_allreduce_hooks(self.model, configs.Engine.accumulate_steps,
                                                       d.get("fuse_sequence_parallel_allreduce", False),
                                                       env.get_hcg().get_model_parallel_group())

    def get_model(self):
        cfg = self.configs
        m = copy.deepcopy(dict(cfg.Model))
        d = cfg.Distributed
        hcg = env.get_hcg()
        mp_group = hcg.get_model_parallel_group() if d.mp_degree > 1 else None
        vocab = gpt.vocab_size_with_padding(m.get("vocab_size", 50304), m.get("vocab_size_divisible_unit", 128), d.mp_degree)
        cfg.Model["vocab_size"] = vocab
        kw = model_kwargs(cfg)
        kw["vocab_size"] = vocab
        kv_hidden = kw["hidden_size"] // kw["num_attention_heads"] * kw["num_key_value_heads"] if kw.get("num_key_value_heads") else None
        get_model_size(kw["num_layers"], kw["hidden_size"], vocab, kw.get("max_position_embeddings", 1024), kv_hidden, kw.get("ffn_hidden_size"),
                       kw.get("ffn_activation", "gelu"))
        dtype, device = _param_dtype(cfg), _device(cfg)
        fused_tp = bool(cfg.get("Fused", {}).get("tp_comm", False))
        if d.pp_degree > 1:
            from .gpt.pipe import GPTForPretrainingPipe

            return GPTForPretrainingPipe(hcg=hcg, mp_group=mp_group, dtype=dtype, device=device, fused_tp_comm=fused_tp,
                                         pp_recompute_interval=d.get("pp_recompute_interval", 1), **kw)
        core = gpt.GPTModel(mp_group=mp_group, dtype=dtype, device=device, fused_tp_comm=fused_tp, **kw)
        return gpt.GPTForPretraining(core)

    def get_loss_fn(self):
        d = self.configs.Distributed
        if d.pp_degree > 1:
            return None          # the pipeline model owns its criterion on the last stage
        hcg = env.get_hcg()
        return gpt.GPTPretrainingCriterion(hcg.get_model_parallel_group() if d.mp_degree > 1 else None)

    def pretreating_batch(self, batch):
        if self.configs.Distributed.pp_degree > 1:
            tokens, position_ids, labels, loss_mask = self._context_parallel_slice(batch)
            hcg = getattr(env, "_hcg", None)
            c = getattr(hcg, "cp", 1) if hcg is not None else 1
            if c > 1:
                # the pipeline computes the loss per micro-batch on the last stage: hand it each sample's share of the GROUP's live-token count,
                # so that the cp ranks' losses average to sum(CE x mask) / sum(mask) over whole sequences (same rule as _context_parallel_loss)
                rows = loss_mask.float().sum(dim=1)
                torch.distributed.all_reduce(rows, group=hcg.get_context_parallel_group().process_group)
                return [(tokens, position_ids), (labels, loss_mask, rows / c)]
            return [(tokens, position_ids), (labels, loss_mask)]
        return batch

    def input_spec(self):
        s = self.configs.Data.get("Test", self.configs.Data.get("Train")).dataset.max_seq_len
        return [dict(shape=[None, s], name="tokens", dtype="int64"), dict(shape=[None, s], name="ids", dtype="int64")]

    def inference_end(self, outputs):
        for k, v in (outputs.items() if isinstance(outputs, dict) else enumerate(outputs)):
            for i in range(len(v)):
                logger.info(f"{k}[{i}]: shape {tuple(v[i].shape)}")
        return outputs


# ---- names the reference keeps in this file (language_module.py:228-830) or in auto_utils.py; they live in sibling modules here
from ...utils.lazy import lazy_exports  # noqa: E402
from .gpt.model import vocab_size_with_padding  # noqa: E402,F401

__getattr__ = lazy_exports(__name__, {
    "GPTFinetuneModule": ".finetune_module", "GPTGenerationModule": ".generation_module", "GPTEvalModule": ".eval_module",
    "MoEModule": ".moe_module", "process_mesh_config": ".auto_module", "ProcessMesh": ".auto_module",
})
