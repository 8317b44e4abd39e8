"""Model compression: quantisation-aware training and structured pruning.

Reference: ppfleetx/utils/compression_helper.py:19-79 delegates to PaddleSlim (``QAT`` with PACT activation clipping,
``abs_max`` / ``channel_wise_abs_max`` weight and ``moving_average_abs_max`` activation quantisers, int8) and to
``L1NormFilterPruner`` / ``L2NormFilterPruner`` on the fused-QKV and FFN1 weights (axis 1, head-aware).  Both are
implemented natively here:

  * ``quant_model`` wraps every linear-like layer with fake-quant observers (straight-through estimator); ``convert_to_int8``
    turns the trained wrappers into ``Int8Linear`` layers that run the int8 tcgen05 GEMM,
  * ``prune_model`` physically removes the lowest-norm FFN channels and attention heads (ratio per layer), keeping QKV /
    out-proj / FFN2 shapes consistent.

YAML block (same as the reference)::

    Compress:
      pretrained:
      Quantization: {enable: True, weight_quantize_type: abs_max, activation_quantize_type: moving_average_abs_max,
                     weight_bits: 8, activation_bits: 8, onnx_format: True, activation_preprocess_type: PACT,
                     quantizable_layer_type: [Linear, ColumnParallelLinear, RowParallelLinear]}
      Prune: {enable: True, criterion: l1_norm, ratio: 0.125}
"""
from __future__ import annotations

import os
from typing import Tuple

import torch
import torch.nn as nn
import torch.nn.functional as F

from ..ops import functional as OF
from .log import logger


class _RoundSTE(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return torch.round(x)

    @staticmethod
    def backward(ctx, g):
        return g


def fake_quant(x: torch.Tensor, scale: torch.Tensor, bits: int = 8) -> torch.Tensor:
    qmax = 2 ** (bits - 1) - 1
    s = (scale / qmax).clamp(min=1e-12)
    return torch.clamp(_RoundSTE.apply(x / s), -qmax, qmax) * s


class PACT(nn.Module):
    """Learnable symmetric clipping of activations before quantisation (``activation_preprocess_type: PACT``)."""

    def __init__(self, init_alpha: float = 20.0):
        super().__init__()
        self.alpha = nn.Parameter(torch.tensor(float(init_alpha)))
        self.alpha.no_weight_decay = True

    def forward(self, x):
        a = self.alpha.to(x.dtype)
        return x - F.relu(x - a) + F.relu(-a - x)


class QuantLinearWrapper(nn.Module):
    """Fake-quant wrapper around any module that owns ``weight`` [out(/n), in(/n)] (+ optional ``bias``) and a forward that
    consumes them through ``OF.linear`` — the wrapped layer's parallel semantics are preserved by quantising its weight in
    place for the duration of the call."""

    def __init__(self, layer: nn.Module, weight_bits=8, act_bits=8, weight_type="abs_max", act_type="moving_average_abs_max",
                 moving_rate=0.9, pact: bool = False):
        super().__init__()
        self.layer = layer
        self.wbits, self.abits = weight_bits, act_bits
        self.channel_wise = "channel_wise" in weight_type
        self.moving_rate = moving_rate
        self.pact = PACT() if pact else None
        self.register_buffer("act_scale", torch.zeros(()))
        self.register_buffer("act_state", torch.zeros(()))
        self.register_buffer("act_accum", torch.zeros(()))

    @property
    def weight(self):
        return self.layer.weight

    @property
    def bias(self):
        return getattr(self.layer, "bias", None)

    def _observe(self, x):
        cur = x.detach().abs().max().float()
        if self.training:
            self.act_state.mul_(self.moving_rate).add_(1.0)
            self.act_accum.mul_(self.moving_rate).add_(cur)
            self.act_scale.copy_(self.act_accum / self.act_state)
        return self.act_scale if float(self.act_state) > 0 else cur

    def weight_scale(self) -> torch.Tensor:
        w = self.layer.weight.detach().float()
        return w.abs().amax(1, keepdim=True) if self.channel_wise else w.abs().max()

    def forward(self, x, *args, **kwargs):
        if self.pact is not None:
            x = self.pact(x)
        x = fake_quant(x, self._observe(x).to(x.dtype), self.abits)
        w = self.layer.weight
        orig = w.data
        wq = fake_quant(w, self.weight_scale().to(w.dtype), self.wbits)
        # run the wrapped layer with the fake-quantised weight; STE keeps the gradient on the real parameter
        self.layer.weight.data = wq.detach()
        try:
            y = self.layer(x, *args, **kwargs)
        finally:
            self.layer.weight.data = orig
        return y


_DEFAULT_TYPES = ("Linear", "ColumnParallelLinear", "RowParallelLinear", "ColumnSequenceParallelLinear", "RowSequenceParallelLinear")


def quant_model(model: nn.Module, cfg: dict) -> nn.Module:
    types = tuple(cfg.get("quantizable_layer_type") or _DEFAULT_TYPES)
    skip = tuple(cfg.get("skip_tensor_map", cfg.get("skip_layers", [])) or [])
    n = 0
    for name, mod in list(model.named_modules()):
        for child_name, child in list(mod.named_children()):
            full = f"{name}.{child_name}" if name else child_name
            if child.__class__.__name__ in types and not isinstance(child, QuantLinearWrapper) and not any(s in full for s in skip):
                setattr(mod, child_name, QuantLinearWrapper(child, cfg.get("weight_bits", 8), cfg.get("activation_bits", 8),
                                                            cfg.get("weight_quantize_type", "abs_max"),
                                                            cfg.get("activation_quantize_type", "moving_average_abs_max"),
                                                            cfg.get("moving_rate", 0.9), cfg.get("activation_preprocess_type") == "PACT"))
                n += 1
    logger.info(f"QAT: wrapped {n} layers with fake-quant observers")
    return model


def convert_to_int8(model: nn.Module) -> nn.Module:
    """Replace trained ``QuantLinearWrapper(nn.Linear)`` layers by ``Int8Linear`` (export time, single-card layers)."""
    from ..ops.quant import Int8Linear

    for name, mod in list(model.named_modules()):
        for child_name, child in list(mod.named_children()):
            if isinstance(child, QuantLinearWrapper) and isinstance(child.layer, nn.Linear):
                act = float(child.act_scale) if float(child.act_state) > 0 else None
                setattr(mod, child_name, Int8Linear.from_float(child.layer.weight.data, child.layer.bias, None, act))
    return model


# ------------------------------------------------------------------------------------------ pruning
def _norm(w: torch.Tensor, criterion: str, dims) -> torch.Tensor:
    return w.float().abs().sum(dims) if criterion.startswith("l1") else w.float().pow(2).sum(dims).sqrt()


def get_pruned_params(model: nn.Module) -> list:
    """Names of the weights structured pruning acts on: 2-D weights of (tensor-parallel) linear layers that are a fused QKV projection
    (``out = 3 * in``) or a first FFN projection (``out = 4 * in``); their consumers (attention output / second FFN projection) are pruned
    along with them (reference utils/compression_helper.py:19-42 — there in Paddle's ``[in, out]`` layout, here ``[out, in]``)."""
    from ..parallel.tp_layers import ColumnParallelLinear, RowParallelLinear

    names = []
    for mod_name, mod in model.named_modules():
        if not isinstance(mod, (nn.Linear, ColumnParallelLinear, RowParallelLinear)):
            continue
        w = getattr(mod, "weight", None)
        if w is None or w.dim() != 2:
            continue
        world = getattr(mod, "world", None) or 1
        out_f, in_f = w.shape[0] * (world if isinstance(mod, ColumnParallelLinear) else 1), w.shape[1]
        if out_f in (3 * in_f, 4 * in_f):
            names.append(f"{mod_name}.weight" if mod_name else "weight")
    return names


def prune_model(model: nn.Module, cfg: dict) -> nn.Module:
    """Structured pruning of every GPT-style decoder layer: FFN channels (linear1 out / linear2 in) and attention heads
    (qkv rows per head / out_proj columns)."""
    ratio = float(cfg.get("ratio", 0.125))
    crit = cfg.get("criterion", "l1_norm")
    n_layers = 0
    for mod in model.modules():
        if hasattr(mod, "linear1") and hasattr(mod, "linear2") and hasattr(mod.linear1, "weight"):
            if getattr(mod, "ffn_activation", "gelu") == "swiglu":
                raise ValueError("structured pruning does not support ffn_activation: swiglu (linear1 holds gate / up pairs)")
            w1, w2 = mod.linear1.weight, mod.linear2.weight
            keep = max(int(round(w1.shape[0] * (1 - ratio) / 8)) * 8, 8)
            idx = torch.topk(_norm(w1.data, crit, 1), keep).indices.sort().values
            mod.linear1.weight = nn.Parameter(w1.data[idx].clone())
            if getattr(mod.linear1, "bias", None) is not None:
                mod.linear1.bias = nn.Parameter(mod.linear1.bias.data[idx].clone())
            mod.linear2.weight = nn.Parameter(w2.data[:, idx].clone())
            n_layers += 1
        attn = getattr(mod, "self_attn", None)
        if attn is not None and hasattr(attn, "qkv_proj") and cfg.get("prune_heads", True):
            if getattr(attn, "group", 1) > 1:
                raise ValueError("head pruning does not support grouped-query attention (num_key_value_heads < num_attention_heads); "
                                 "set Compress.Prune.prune_heads=False to prune the FFN only")
            h, d = attn.local_heads, attn.head_dim
            keep_h = max(int(round(h * (1 - ratio))), 1)
            w = attn.qkv_proj.weight.data.view(h, 3 * d, -1)
            idx = torch.topk(_norm(w, crit, (1, 2)), keep_h).indices.sort().values
            attn.qkv_proj.weight = nn.Parameter(w[idx].reshape(keep_h * 3 * d, -1).clone())
            if attn.qkv_proj.bias is not None:
                attn.qkv_proj.bias = nn.Parameter(attn.qkv_proj.bias.data.view(h, 3 * d)[idx].reshape(-1).clone())
            wo = attn.out_proj.weight.data.view(attn.out_proj.weight.shape[0], h, d)
            attn.out_proj.weight = nn.Parameter(wo[:, idx].reshape(wo.shape[0], keep_h * d).clone())
            attn.local_heads, attn.num_heads = keep_h, keep_h * getattr(attn, "world", 1)
            attn.local_kv_heads, attn.num_kv_heads = attn.local_heads, attn.num_heads
    logger.info(f"pruned {n_layers} decoder layers with ratio {ratio} ({crit})")
    return model


def compress_model(model: nn.Module, compress_cfg: dict, device=None) -> Tuple[nn.Module, bool]:
    """Engine hook (reference eager_engine.py:757-774): load ``Compress.pretrained`` then prune and/or quantise."""
    pretrained = compress_cfg.get("pretrained")
    if pretrained:
        path = pretrained if os.path.isfile(pretrained) else os.path.join(pretrained, "model.pdparams")
        if os.path.isfile(path):
            state = torch.load(path, map_location="cpu", weights_only=False)
            own = model.state_dict()
            model.load_state_dict({k: v.to(own[k].dtype) for k, v in state.items() if k in own and own[k].shape == v.shape}, strict=False)
            logger.info(f"compress: loaded pretrained weights from {path}")
    quant_mode = False
    prune = compress_cfg.get("Prune") or {}
    if prune.get("enable", False):
        model = prune_model(model, prune)
    quant = compress_cfg.get("Quantization") or {}
    if quant.get("enable", False):
        model = quant_model(model, quant)
        quant_mode = True
    return model, quant_mode
