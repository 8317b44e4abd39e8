"""Shift-SmoothQuant post-training quantisation for export (new capability: README-only in the reference, SURVEY F3).

SmoothQuant (Xiao et al. 2022) migrates activation outliers into the weights with a per-input-channel factor
``s_j = max|X_j|^alpha / max|W_j|^(1-alpha)`` so that ``(X / s)(W * s)^T == X W^T`` while both factors quantise well to int8.
The *shift* variant first centres every activation channel, ``X' = X - z`` with ``z_j = (max_j + min_j) / 2``, folding
``z W^T`` into the layer bias — asymmetric channels (post-GELU, post-LayerNorm with bias) then use the full int8 range.

``calibrate`` collects per-channel min / max over calibration batches with forward hooks; ``smooth_and_quantize`` rewrites
every ``nn.Linear``-like layer into ``ShiftSmoothInt8Linear`` running the int8 tcgen05 GEMM.
"""
from __future__ import annotations

from typing import Dict, Iterable, Optional

import torch
import torch.nn as nn

from ..ops.quant import Int8Linear, quantize_weight_int8

_TYPES = ("Linear", "ColumnParallelLinear", "RowParallelLinear")


class ActStats:
    def __init__(self):
        self.min: Optional[torch.Tensor] = None
        self.max: Optional[torch.Tensor] = None

    def update(self, x: torch.Tensor) -> None:
        x2 = x.detach().reshape(-1, x.shape[-1]).float()
        mn, mx = x2.amin(0), x2.amax(0)
        self.min = mn if self.min is None else torch.minimum(self.min, mn)
        self.max = mx if self.max is None else torch.maximum(self.max, mx)


def calibrate(model: nn.Module, batches: Iterable, forward_fn=None) -> Dict[str, ActStats]:
    """Per-input-channel activation min / max of every linear-like layer over ``batches``.  While calibrating, the layers carry
    ``needs_forward`` so that fused call sites (which read ``.weight`` directly, e.g. the fused FFN) route through ``forward()`` and the
    observation hooks see every layer's input."""
    stats: Dict[str, ActStats] = {}
    hooks, marked = [], []
    for name, mod in model.named_modules():
        if mod.__class__.__name__ in _TYPES:
            stats[name] = ActStats()
            hooks.append(mod.register_forward_pre_hook(lambda m, a, n=name: stats[n].update(a[0])))
            if not getattr(mod, "needs_forward", False):
                mod.needs_forward = True
                marked.append(mod)
    model.eval()
    try:
        with torch.no_grad():
            for b in batches:
                forward_fn(model, b) if forward_fn is not None else model(*b) if isinstance(b, (tuple, list)) else model(b)
    finally:
        for h in hooks:
            h.remove()
        for mod in marked:
            del mod.needs_forward
    return stats


class ShiftSmoothInt8Linear(nn.Module):
    def __init__(self, weight: torch.Tensor, bias: Optional[torch.Tensor], stats: ActStats, alpha: float = 0.5, shift: bool = True):
        super().__init__()
        if stats is None:            # shape-only construction (``empty``): buffers are filled by load_state_dict
            out_f, in_f = weight.shape
            self.register_buffer("shift", torch.zeros(in_f, dtype=weight.dtype, device=weight.device))
            self.inner = Int8Linear(torch.zeros(out_f, in_f, dtype=torch.int8, device=weight.device), torch.ones(out_f, device=weight.device),
                                    torch.zeros(out_f, dtype=weight.dtype, device=weight.device), torch.ones(in_f, device=weight.device))
            return
        w = weight.detach().float()
        z = ((stats.max + stats.min) / 2).to(w.device) if shift else torch.zeros(w.shape[1], device=w.device)
        amax = torch.maximum((stats.max.to(w.device) - z).abs(), (stats.min.to(w.device) - z).abs()).clamp(min=1e-5)
        wmax = w.abs().amax(0).clamp(min=1e-5)
        s = (amax.pow(alpha) / wmax.pow(1 - alpha)).clamp(min=1e-5)
        b = (bias.detach().float() if bias is not None else torch.zeros(w.shape[0], device=w.device)) + w @ z     # fold the shift
        self.register_buffer("shift", z.to(weight.dtype))
        self.inner = Int8Linear.from_float(w, b.to(weight.dtype), smooth=s)

    @classmethod
    def empty(cls, out_features: int, in_features: int, dtype=torch.bfloat16, device=None) -> "ShiftSmoothInt8Linear":
        """Same buffers as a calibrated layer, to be filled from an exported state dict (InferenceEngine)."""
        return cls(torch.empty(out_features, in_features, dtype=dtype, device=device or "cpu"), None, None)

    def forward(self, x):
        return self.inner(x - self.shift.to(x.dtype))


def _tp_single(child) -> bool:
    return child.__class__.__name__ in ("ColumnParallelLinear", "RowParallelLinear") and getattr(child, "world", 1) == 1 and child.weight is not None


def smooth_and_quantize(model: nn.Module, stats: Dict[str, ActStats], alpha: float = 0.5, shift: bool = True, skip=("score", "head")) -> nn.Module:
    """Rewrite every calibrated linear: ``nn.Linear`` is replaced by a ``ShiftSmoothInt8Linear``; the tensor-parallel linears (single-rank
    serving layout) keep their module — and their bias add — and get the quantised GEMM as ``.int8`` (the hook ``_tp_linear`` looks for), with
    only the shift term folded into the int8 layer's bias.  The names of the rewritten layers are recorded in ``model.smooth_quant_layers``."""
    done, sharded = [], 0
    for name, mod in list(model.named_modules()):
        for child_name, child in list(mod.named_children()):
            full = f"{name}.{child_name}" if name else child_name
            if full not in stats or stats[full].max is None or any(s in child_name for s in skip):
                continue
            if getattr(child, "world", 1) > 1:
                sharded += 1          # a sharded weight would need its smoothing factors agreed across the group: export with mp_degree 1
                continue
            if isinstance(child, nn.Linear):
                setattr(mod, child_name, ShiftSmoothInt8Linear(child.weight.data, child.bias, stats[full], alpha, shift))
                done.append({"name": full, "kind": "linear", "out": child.out_features, "in": child.in_features})
            elif _tp_single(child):
                out_f, in_f = child.weight.shape
                child.int8 = ShiftSmoothInt8Linear(child.weight.data, None, stats[full], alpha, shift)
                child._parameters["weight"] = None          # free the high-precision copy
                done.append({"name": full, "kind": "tp", "out": out_f, "in": in_f})
    if sharded:
        from .log import logger

        logger.warning(f"SmoothQuant: {sharded} tensor-parallel layers (mp_degree > 1) left in high precision; export on the mp1 layout "
                       "(tools/reshard.py converts a checkpoint) to quantise them")
    model.smooth_quant_layers = done
    return model


def install_empty(model: nn.Module, layers, dtype=torch.bfloat16) -> nn.Module:
    """Re-create the module structure ``smooth_and_quantize`` produced (from the layer list stored in an export recipe) so that the exported
    state dict can be loaded into a freshly built model."""
    mods = dict(model.named_modules())
    for spec in layers:
        parent_name, _, child_name = spec["name"].rpartition(".")
        parent, child = mods[parent_name] if parent_name else model, mods[spec["name"]]
        dev = next((p.device for p in child.parameters()), torch.device("cpu"))
        empty = ShiftSmoothInt8Linear.empty(spec["out"], spec["in"], dtype, dev)
        if spec["kind"] == "linear":
            setattr(parent, child_name, empty)
        else:
            child.int8 = empty
            child._parameters["weight"] = None
    model.smooth_quant_layers = list(layers)
    return model


def calibration_batches(configs, n: int, batch_size: int = 4, seq_len: Optional[int] = None):
    """``n`` batches of ``(tokens, position_ids)``: the recipe's ``Data.Eval`` set when it can be built on this machine, uniform random tokens of
    the model's vocabulary otherwise (ranges from random tokens are cruder — pass real text for production exports)."""
    from .log import logger

    out = []
    try:
        from ..data import build_dataloader

        if "Data" in configs and "Eval" in configs.Data:
            for batch in build_dataloader(configs.Data, "Eval"):
                out.append((batch[0], batch[1]))
                if len(out) >= n:
                    return out
    except (OSError, KeyError, ValueError, AssertionError, TypeError, AttributeError) as exc:      # missing files or a recipe without a usable Eval block
        logger.warning(f"SmoothQuant calibration: Data.Eval is not usable here ({type(exc).__name__}: {exc}); using random tokens")
    vocab = int(configs.Model.get("vocab_size", 50304))
    seq = int(seq_len or min(int(configs.Model.get("max_position_embeddings", 1024)), 512))
    g = torch.Generator().manual_seed(0)
    while len(out) < n:
        out.append((torch.randint(0, vocab, (batch_size, seq), generator=g), torch.arange(seq).unsqueeze(0).expand(batch_size, seq).contiguous()))
    return out
