"""``GPTFinetuneModule`` — full-parameter sequence-classification fine-tuning on GLUE (reference
language_module.py:228-487): ``GPTForSequenceClassification`` on a single card, ``pretrained.pdparams`` loading with
automatic fused<->split QKV conversion, loss and metric selected by name from the ``Model:`` block."""
from __future__ import annotations

import os
from typing import Optional

import torch
import torch.nn.functional as F

from ...utils.log import logger
from . import metrics as M
from .gpt import model as gpt
from .language_module import LanguageModule, _device, _param_dtype, model_kwargs

_LOSSES = {"CrossEntropyLoss": lambda logits, y: F.cross_entropy(logits.float(), y.long().reshape(-1)),
           "MSELoss": lambda logits, y: F.mse_loss(logits.float().reshape(-1), y.float().reshape(-1))}


def convert_qkv_layout(state: dict, fuse: bool, num_heads: int, num_kv_heads: Optional[int] = None) -> dict:
    """Fuse ``q_proj/k_proj/v_proj`` into ``qkv_proj`` ([heads, 3, head_dim] rows) or split it back
    (reference language_module.py:312-383, transposed to our [out, in] storage).  With ``num_kv_heads`` K/V heads (grouped-query
    attention, default ``num_heads``) the fused rows are ``[kv_heads, G + 2, head_dim]``: the G query heads of a group, its key, its value."""
    kvh = num_kv_heads or num_heads
    g = num_heads // kvh
    out = dict(state)
    if fuse:
        for k in [k for k in state if k.endswith("q_proj.weight") or k.endswith("q_proj.bias")]:
            base, kind = k.rsplit("q_proj.", 1)
            q, kk, v = state[base + "q_proj." + kind], state[base + "k_proj." + kind], state[base + "v_proj." + kind]
            hd = q.shape[0] // num_heads
            parts = [t.reshape(kvh, n, hd, *t.shape[1:]) for t, n in ((q, g), (kk, 1), (v, 1))]
            out[base + "qkv_proj." + kind] = torch.cat(parts, 1).reshape(q.shape[0] + 2 * kk.shape[0], *q.shape[1:])
            for n in ("q_proj.", "k_proj.", "v_proj."):
                out.pop(base + n + kind)
    else:
        for k in [k for k in state if "qkv_proj." in k]:
            base, kind = k.rsplit("qkv_proj.", 1)
            w = state[k]
            hd = w.shape[0] // (num_heads + 2 * kvh)
            w = w.reshape(kvh, g + 2, hd, *w.shape[1:])
            out[base + "q_proj." + kind] = w[:, :g].reshape(num_heads * hd, *w.shape[3:])
            for i, n in ((g, "k_proj."), (g + 1, "v_proj.")):
                out[base + n + kind] = w[:, i].reshape(kvh * hd, *w.shape[3:])
            out.pop(k)
    return out


class GPTFinetuneModule(LanguageModule):
    def __init__(self, configs):
        super().__init__(configs)
        assert self.nranks == 1 or configs.Distributed.mp_degree == 1, "GPT fine-tuning runs on a single card / pure data parallel"
        m = configs.Model
        self.metric = self._build_metric(m.get("metric", {"train": {"name": "Accuracy"}, "eval": {"name": "Accuracy"}}))
        self.best_metric = 0.0

    def process_configs(self, configs):
        from .language_module import process_model_configs, process_optim_configs

        process_model_configs(configs)
        process_optim_configs(configs)
        return configs

    def _build_metric(self, cfg):
        def one(c):
            c = dict(c or {"name": "Accuracy"})
            return getattr(M, c.pop("name"))(**c)
        return {"train": one(cfg.get("train")), "eval": one(cfg.get("eval"))}

    def get_model(self):
        cfg = self.configs
        kw = model_kwargs(cfg)
        num_classes = int(cfg.Model.get("num_classes", 2))
        core = gpt.GPTModel(dtype=_param_dtype(cfg), device=_device(cfg), **kw)
        model = gpt.GPTForSequenceClassification(core, num_classes, pad_token_id=int(cfg.Model.get("pad_token_id", 50256)))
        pretrained = cfg.Model.get("pretrained")
        if pretrained:
            path = pretrained if pretrained.endswith(".pdparams") else pretrained + ".pdparams"
            assert os.path.exists(path), f"{path} is not exists!"
            state = torch.load(path, map_location="cpu", weights_only=False)
            fused_ckpt = any("qkv_proj" in k for k in state)
            if fused_ckpt != bool(cfg.Model.get("fuse_attn_qkv", True)):
                state = convert_qkv_layout(state, bool(cfg.Model.get("fuse_attn_qkv", True)), cfg.Model.num_attention_heads,
                                           cfg.Model.get("num_key_value_heads"))
            own = model.state_dict()
            load = {k: v.to(own[k].dtype) for k, v in state.items() if k in own and own[k].shape == v.shape}
            missing = [k for k in own if k not in load]
            model.load_state_dict(load, strict=False)
            logger.info(f"loaded {len(load)} tensors from {path}; missing (newly initialised): {missing}")
        return model

    def get_loss_fn(self):
        name = self.configs.Model.get("loss", {}).get("train", {}).get("name", "CrossEntropyLoss") if isinstance(self.configs.Model.get("loss"), dict) else "CrossEntropyLoss"
        return _LOSSES[name]

    def forward(self, input_ids):
        return self.model(input_ids)

    @staticmethod
    def _unpack(batch):
        if isinstance(batch, dict):
            return batch["input_ids"], batch["labels"]
        return batch[0], batch[1]

    def training_step(self, batch):
        ids, labels = self._unpack(batch)
        logits = self(ids)
        return self.loss_fn(logits, labels)

    def training_step_end(self, log_dict):
        speed = 1.0 / log_dict["train_cost"]
        logger.train("[train] epoch: [%d/%d], step: [%d/%d], learning rate: %.7f, loss: %.9f, avg_batch_cost: %.5f sec, speed: %.2f step/s"
                     % (log_dict["epoch"], log_dict["total_epoch"], log_dict["batch"], log_dict["total_batch"], log_dict["lr"], log_dict["loss"],
                        log_dict["train_cost"], speed))

    def validation_step(self, batch):
        ids, labels = self._unpack(batch)
        logits = self(ids)
        loss = self.loss_fn(logits, labels)
        m = self.metric["eval"]
        m.update(m.compute(logits, labels))
        return loss

    def validation_epoch_end(self, log_dict):
        res = self.metric["eval"].accumulate()
        self.metric["eval"].reset()
        head = res[0] if isinstance(res, (tuple, list)) else res
        self.best_metric = max(self.best_metric, float(head))
        logger.eval(f"[Eval] epoch: {log_dict['epoch']}, total time: {log_dict['eval_cost']:.5f} sec, metric: {res}, best: {self.best_metric:.5f}")

    def test_step(self, batch):
        return self.validation_step(batch)

    def input_spec(self):
        return [dict(shape=[None, None], name="input_ids", dtype="int64")]
