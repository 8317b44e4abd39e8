"""Parameter-efficient fine-tuning: LoRA and Prefix-Tuning.

The reference advertises both in its README (README.md:46,55) but ships no code (SURVEY F3); they are specified here from
the papers (Hu et al. 2021; Li & Liang 2021):

  * ``apply_lora(model, r, alpha, dropout, target_modules)`` freezes the base model and adds ``W + (alpha / r) B A`` adapters
    to the selected linear-like layers (works on the tensor-parallel layers too: A is replicated, B follows the layer's
    output sharding); ``merge_lora`` folds the adapters back for export,
  * ``apply_prefix_tuning(model, num_virtual_tokens)`` prepends trainable key/value prefixes to every attention layer of a
    GPT model (re-parameterised through a small MLP during training).
"""
from __future__ import annotations

import math
from typing import Iterable, List

import torch
import torch.nn as nn

from ..ops import functional as OF

_TARGET_TYPES = ("Linear", "ColumnParallelLinear", "RowParallelLinear", "ColumnSequenceParallelLinear", "RowSequenceParallelLinear")


class LoRALinear(nn.Module):
    def __init__(self, layer: nn.Module, r: int = 8, alpha: int = 16, dropout: float = 0.0):
        super().__init__()
        self.layer = layer
        w = layer.weight
        out_f, in_f = w.shape
        self.r, self.scaling, self.dropout = r, alpha / r, dropout
        self.lora_A = nn.Parameter(torch.empty(r, in_f, dtype=w.dtype, device=w.device))
        self.lora_B = nn.Parameter(torch.zeros(out_f, r, dtype=w.dtype, device=w.device))
        nn.init.kaiming_uniform_(self.lora_A, a=math.sqrt(5))
        self.lora_B.tp_sharded = bool(getattr(w, "tp_sharded", False)) and getattr(w, "split_axis", 0) == 0
        self.lora_A.tp_sharded = bool(getattr(w, "tp_sharded", False)) and getattr(w, "split_axis", 0) == 1
        self.merged = False
        self.needs_forward = True       # fused call sites that read ``.weight`` directly must not bypass the low-rank branch
        for p in layer.parameters():
            p.requires_grad = False

    @property
    def weight(self):
        return self.layer.weight

    @property
    def bias(self):
        return getattr(self.layer, "bias", None)

    def forward(self, x, *args, **kwargs):
        y = self.layer(x, *args, **kwargs)
        if self.merged:
            return y
        xin = OF.dropout(x, self.dropout, self.training)
        delta = OF.linear(OF.linear(xin, self.lora_A), self.lora_B) * self.scaling
        if isinstance(y, tuple):          # (out, bias) layers that skip the bias add
            return (y[0] + delta[..., : y[0].shape[-1]] if delta.shape == y[0].shape else y[0] + delta, *y[1:])
        return y + delta if delta.shape == y.shape else y

    @torch.no_grad()
    def merge(self):
        if not self.merged:
            self.layer.weight.data += (self.lora_B.float() @ self.lora_A.float()).to(self.layer.weight.dtype) * self.scaling
            self.merged = True


def apply_lora(model: nn.Module, r: int = 8, alpha: int = 16, dropout: float = 0.0,
               target_modules: Iterable[str] = ("qkv_proj", "q_proj", "k_proj", "v_proj", "out_proj")) -> List[LoRALinear]:
    for p in model.parameters():
        p.requires_grad = False
    adapters = []
    targets = tuple(target_modules)
    for name, mod in list(model.named_modules()):
        for child_name, child in list(mod.named_children()):
            if child_name in targets and child.__class__.__name__ in _TARGET_TYPES and getattr(child, "world", 1) == 1:
                wrap = LoRALinear(child, r, alpha, dropout)
                setattr(mod, child_name, wrap)
                adapters.append(wrap)
    return adapters


def merge_lora(model: nn.Module) -> nn.Module:
    for name, mod in list(model.named_modules()):
        for child_name, child in list(mod.named_children()):
            if isinstance(child, LoRALinear):
                child.merge()
                setattr(mod, child_name, child.layer)
    return model


def lora_state_dict(model: nn.Module) -> dict:
    return {k: v for k, v in model.state_dict().items() if "lora_" in k}


class PrefixEncoder(nn.Module):
    """Trainable prefixes: ``[num_layers, 2, heads, tokens, head_dim]`` produced by an MLP over a small embedding."""

    def __init__(self, num_layers, heads, head_dim, num_virtual_tokens=16, hidden=512, reparam=True, dtype=None, device=None):
        super().__init__()
        self.shape = (num_layers, 2, heads, num_virtual_tokens, head_dim)
        out = num_layers * 2 * heads * head_dim
        self.embed = nn.Embedding(num_virtual_tokens, hidden if reparam else out, dtype=dtype, device=device)
        self.mlp = nn.Sequential(nn.Linear(hidden, hidden, dtype=dtype, device=device), nn.Tanh(), nn.Linear(hidden, out, dtype=dtype, device=device)) if reparam else None
        self.n = num_virtual_tokens

    def forward(self):
        e = self.embed(torch.arange(self.n, device=self.embed.weight.device))
        if self.mlp is not None:
            e = self.mlp(e)
        L, two, h, t, d = self.shape
        return e.view(t, L, two, h, d).permute(1, 2, 3, 0, 4)


def apply_prefix_tuning(gpt_model: nn.Module, num_virtual_tokens: int = 16, hidden: int = 512, reparam: bool = True) -> PrefixEncoder:
    """Freeze ``gpt_model`` (a ``GPTModel``) and make every attention layer attend to trainable prefix keys/values."""
    for p in gpt_model.parameters():
        p.requires_grad = False
    layers = gpt_model.decoder.layers
    att0 = layers[0].self_attn
    w = gpt_model.decoder.norm.weight
    enc = PrefixEncoder(len(layers), getattr(att0, "local_kv_heads", att0.local_heads), att0.head_dim, num_virtual_tokens, hidden, reparam, w.dtype, w.device)
    gpt_model.prefix_encoder = enc
    for i, layer in enumerate(layers):
        _patch_attention(layer.self_attn, enc, i)
    return enc


def _patch_attention(attn, enc: PrefixEncoder, index: int) -> None:
    import torch.nn.functional as F

    def core(q, k, v, attn_mask):
        pk, pv = enc()[index]                                  # [kv heads, tokens, d]
        b = q.shape[0]
        pk = pk.transpose(0, 1).unsqueeze(0).expand(b, -1, -1, -1).to(q.dtype)     # [b, tokens, heads, d]
        pv = pv.transpose(0, 1).unsqueeze(0).expand(b, -1, -1, -1).to(q.dtype)
        k2, v2 = torch.cat([pk, k], 1), torch.cat([pv, v], 1)
        sq, sk, t = q.shape[1], k.shape[1], pk.shape[1]
        causal = torch.ones(sq, sk, dtype=torch.bool, device=q.device).tril(sk - sq)
        mask = torch.cat([torch.ones(sq, t, dtype=torch.bool, device=q.device), causal], 1)
        gqa = {"enable_gqa": True} if k2.shape[2] != q.shape[2] else {}
        o = F.scaled_dot_product_attention(q.transpose(1, 2), k2.transpose(1, 2), v2.transpose(1, 2), attn_mask=mask,
                                           dropout_p=attn.attn_dropout if attn.training else 0.0, **gqa)
        return o.transpose(1, 2)

    attn._core = core


# ---------------------------------------------------------------------------------------------------- config-driven entry
def _core_gpt(model: nn.Module) -> nn.Module:
    """The module that owns ``decoder.layers`` (GPTModel), wherever the task wrapper keeps it."""
    for m in model.modules():
        dec = getattr(m, "decoder", None)
        if dec is not None and hasattr(dec, "layers"):
            return m
    raise ValueError("prefix tuning needs a GPT-style model (a module with ``decoder.layers``)")


def apply_peft(model: nn.Module, cfg) -> dict:
    """``PEFT`` section of a recipe -> adapters on ``model``; base parameters are frozen, so an optimizer built afterwards sees only the
    adapter parameters.

        PEFT: {method: lora, r: 8, alpha: 16, dropout: 0.05, target_modules: [qkv_proj, out_proj, linear1, linear2], pretrained: ./ckpt/345M}
        PEFT: {method: prefix, num_virtual_tokens: 16, hidden: 512, reparam: True, pretrained: ./ckpt/345M}

    ``pretrained`` (a ``model.pdparams`` file or its directory) is loaded into the base model first; ``train_modules`` lists name fragments of
    base parameters that stay trainable next to the adapters (e.g. a freshly initialised classification head)."""
    import os

    method = str(cfg.get("method", "lora")).lower()
    pretrained = cfg.get("pretrained")
    if pretrained:
        path = pretrained if os.path.isfile(pretrained) else os.path.join(pretrained, "model.pdparams")
        state = torch.load(path, map_location="cpu", weights_only=False)
        own = model.state_dict()
        missing = [k for k in own if k not in state]
        model.load_state_dict({k: v.to(own[k].dtype) for k, v in state.items() if k in own and own[k].shape == v.shape}, strict=False)
        if missing:
            from .log import logger

            logger.warning(f"PEFT.pretrained: {len(missing)} parameters not in {path} keep their initial values (e.g. {missing[:3]})")
    def names(value, default=()):
        """a YAML list, or the ``-o key=[a,b]`` / ``a,b`` spellings of one on the command line"""
        if value is None:
            return tuple(default)
        if isinstance(value, str):
            return tuple(v.strip().strip("'\"") for v in value.strip("[]() ").split(",") if v.strip())
        return tuple(value)

    if method == "lora":
        adapters = apply_lora(model, r=int(cfg.get("r", 8)), alpha=float(cfg.get("alpha", 16)), dropout=float(cfg.get("dropout", 0.0)),
                              target_modules=names(cfg.get("target_modules"), ("qkv_proj", "q_proj", "k_proj", "v_proj", "out_proj")))
        if not adapters:
            raise ValueError("PEFT.method=lora matched no layer: check PEFT.target_modules (tensor-parallel layers with world > 1 are not wrapped)")
        info = {"method": "lora", "adapters": len(adapters)}
    elif method in ("prefix", "prefix_tuning"):
        for p in model.parameters():
            p.requires_grad = False
        # the encoder registers itself on the core model (``<core>.prefix_encoder``): saved with it, seen by the optimizer
        apply_prefix_tuning(_core_gpt(model), num_virtual_tokens=int(cfg.get("num_virtual_tokens", 16)), hidden=int(cfg.get("hidden", 512)),
                            reparam=bool(cfg.get("reparam", True)))
        info = {"method": "prefix", "virtual_tokens": int(cfg.get("num_virtual_tokens", 16))}
    else:
        raise ValueError(f"unknown PEFT.method {method!r}; expected lora | prefix")
    for frag in names(cfg.get("train_modules")):
        for n, p in model.named_parameters():
            if frag in n:
                p.requires_grad = True
    info["trainable"] = sum(p.numel() for p in model.parameters() if p.requires_grad)
    info["total"] = sum(p.numel() for p in model.parameters())
    return info


def adapter_state_dict(model: nn.Module) -> dict:
    """Only what fine-tuning changed: every parameter that is trainable (LoRA factors, prefix encoder, ``train_modules``)."""
    trainable = {n for n, p in model.named_parameters() if p.requires_grad}
    return {k: v for k, v in model.state_dict().items() if k in trainable}

