"""Offline checkpoint conversion between parallel layouts ("universal checkpoint").

The reference can only resume a checkpoint on the exact ``mp × sharding × pp`` layout it was written with (each rank loads
``mp_XX_sharding_XX_pp_XX/`` — ppfleetx/core/engine/eager_engine.py:757-830) and ships one ad-hoc converter for fused/unfused
QKV (language_module.py:312-383).  Hardware changes are the norm when moving a job onto 180 GB B200s (fewer, larger shards), so
this module turns any checkpoint written by ``distributed/apis/io.py`` into layout-independent form and back:

* ``merge_checkpoint(dir)``  → ``(model_state, named_optimizer_state, meta)`` with every tensor-parallel entry concatenated
  along its split axis (axes are recorded in ``meta_state.pdopt['tp_axes']``), all pipeline stages unioned (pipeline keys carry
  the *global* layer index) and every ZeRO optimizer shard stitched back into per-parameter moments / fp32 masters.
* ``split_checkpoint(...)``  → writes ``mp_XX_sharding_00_pp_00`` folders for a new tensor-parallel degree; the optimizer file
  is written in the ``format: named`` form which ``FusedAdamW.set_state_dict`` slices into whatever bucket/shard layout the new
  job uses, so the sharding degree/stage never needs converting.
* ``gpt_pipe_to_plain`` / ``gpt_plain_to_pipe`` rename keys between ``GPTForPretrainingPipe`` and ``GPTForPretraining``.

CLI: ``python tools/reshard.py --src output/epoch_0_step_1000 --dst output/resharded --mp 2 [--to-plain]``.
"""
from __future__ import annotations

import os
import re
from typing import Dict, List, Optional, Tuple

import torch

_SUB = re.compile(r"mp_(\d+)_sharding_(\d+)_pp_(\d+)$")
_CHUNK = re.compile(r"^_model_chunks\.\d+\.")


def _load(path):
    return torch.load(path, map_location="cpu", weights_only=False)


def discover(ckpt_dir: str) -> Dict[Tuple[int, int, int], str]:
    """Map ``(mp, sharding, pp)`` rank → folder.  A single-process checkpoint (files directly in ``ckpt_dir``) is ``(0,0,0)``."""
    if os.path.isfile(os.path.join(ckpt_dir, "model.pdparams")):
        return {(0, 0, 0): ckpt_dir}
    out = {}
    for name in sorted(os.listdir(ckpt_dir)):
        m = _SUB.match(name)
        if m and os.path.isfile(os.path.join(ckpt_dir, name, "model.pdparams")):
            out[tuple(int(x) for x in m.groups())] = os.path.join(ckpt_dir, name)
    if not out:
        raise FileNotFoundError(f"no checkpoint shards under {ckpt_dir}")
    return out


def _fallback_axis(name: str) -> Optional[int]:
    """Split axis by naming convention, for checkpoints that predate the ``tp_axes`` record."""
    if re.search(r"(qkv_proj|q_proj|k_proj|v_proj|linear1|word_embeddings|gate_up)\.(weight|bias)$", name):
        return 0
    if re.search(r"(out_proj|linear2)\.weight$", name):
        return 1
    return None


def _named_from_flat(opt_shards: List[dict]) -> Tuple[dict, dict]:
    """Stitch ZeRO shards (ordered by sharding rank) of one (mp, pp) position into ``{name: {moment1, moment2, master}}``."""
    named, extra = {}, {"step": opt_shards[0].get("step", 0)}
    if "LR_Scheduler" in opt_shards[0]:
        extra["LR_Scheduler"] = opt_shards[0]["LR_Scheduler"]
    if "groups" not in opt_shards[0]:          # per-parameter optimizers (Momentum) are already named
        return opt_shards[0], extra
    for gi, g0 in enumerate(opt_shards[0]["groups"]):
        parts = sorted((s["groups"][gi] for s in opt_shards), key=lambda g: g["lo"])
        if parts[0]["lo"] != 0 or parts[-1]["hi"] != g0["numel"]:
            # stage-1/2 shards written by sharding rank 0 only: the moments of other ranks are not in this folder set
            raise ValueError("optimizer shards do not cover the flat buffer; pass every sharding_XX folder")
        full = {k: torch.cat([p[k] for p in parts]) if parts[0][k] is not None else None for k in ("moment1", "moment2", "master")}
        for name, off, shape in zip(g0["names"], g0["offsets"], g0["shapes"]):
            n = 1
            for d in shape:
                n *= d
            named[name] = {k: (v[off:off + n].view(shape).clone() if v is not None else None) for k, v in full.items()}
    return named, extra


def _strip_chunk(state: dict) -> dict:
    return {_CHUNK.sub("layers.", k) if _CHUNK.match(k) else k: v for k, v in state.items()}


def merge_checkpoint(ckpt_dir: str, with_optimizer: bool = True):
    shards = discover(ckpt_dir)
    mps = sorted({k[0] for k in shards})
    pps = sorted({k[2] for k in shards})
    shs = sorted({k[1] for k in shards})
    meta = _load(os.path.join(next(iter(shards.values())), "meta_state.pdopt")) if os.path.isfile(
        os.path.join(next(iter(shards.values())), "meta_state.pdopt")) else {}
    model, optim, opt_extra = {}, {}, {}
    for pp in pps:
        per_mp_model, per_mp_opt, axes = [], [], {}
        for mp in mps:
            folder0 = shards[(mp, shs[0], pp)]
            per_mp_model.append(_strip_chunk(_load(os.path.join(folder0, "model.pdparams"))))
            mpath = os.path.join(folder0, "meta_state.pdopt")
            if os.path.isfile(mpath):
                axes.update({(_CHUNK.sub("layers.", k) if _CHUNK.match(k) else k): v for k, v in _load(mpath).get("tp_axes", {}).items()})
            if with_optimizer and os.path.isfile(os.path.join(folder0, "model_state.pdopt")):
                flat = [_load(os.path.join(shards[(mp, sh, pp)], "model_state.pdopt")) for sh in shs]
                named, opt_extra = _named_from_flat(flat)
                per_mp_opt.append({(_CHUNK.sub("layers.", k) if _CHUNK.match(k) else k): v for k, v in named.items()})
        for name in per_mp_model[0]:
            if name in model:
                # a layer shared between pipeline stages (tied embedding): the FIRST stage's copy is the authoritative one.  The word
                # embedding is kept identical on both stages by the shared-weight gradient all-reduce, but everything else in the shared
                # layer that only the first stage uses (position embeddings) is never trained on the last stage and would be stale.
                continue
            axis = axes.get(name, _fallback_axis(name) if len(mps) > 1 else None)
            if len(mps) > 1 and axis is not None:
                model[name] = torch.cat([m[name] for m in per_mp_model], dim=axis)
            else:
                model[name] = per_mp_model[0][name]
            if per_mp_opt and name in per_mp_opt[0]:
                if len(mps) > 1 and axis is not None:
                    optim[name] = {k: (torch.cat([o[name][k] for o in per_mp_opt], dim=axis) if per_mp_opt[0][name][k] is not None else None)
                                   for k in per_mp_opt[0][name]}
                else:
                    optim[name] = per_mp_opt[0][name]
        meta.setdefault("merged_tp_axes", {}).update(axes)
    return model, ({"format": "named", "state": optim, **opt_extra} if optim else None), meta


def split_checkpoint(model: dict, optim: Optional[dict], meta: dict, dst: str, mp: int = 1, tp_axes: Optional[dict] = None):
    """Write ``dst/mp_XX_sharding_00_pp_00`` (or ``dst`` itself for ``mp == 1``)."""
    axes = dict(meta.get("merged_tp_axes", {}))
    axes.update(tp_axes or {})
    for r in range(mp):
        folder = dst if mp == 1 else os.path.join(dst, "mp_{:0>2d}_sharding_00_pp_00".format(r))
        os.makedirs(folder, exist_ok=True)

        def cut(name, t):
            axis = axes.get(name, _fallback_axis(name))
            if mp == 1 or axis is None or t is None:
                return t
            assert t.shape[axis] % mp == 0, f"{name}: dim {axis} of {tuple(t.shape)} not divisible by mp={mp}"
            return t.chunk(mp, dim=axis)[r].clone()

        torch.save({k: cut(k, v) for k, v in model.items()}, os.path.join(folder, "model.pdparams"))
        if optim is not None:
            st = {k: {kk: cut(k, vv) for kk, vv in v.items()} for k, v in optim["state"].items()}
            torch.save({**{k: v for k, v in optim.items() if k != "state"}, "state": st}, os.path.join(folder, "model_state.pdopt"))
        m = {k: v for k, v in meta.items() if k not in ("merged_tp_axes",)}
        m["tp_axes"] = {k: v for k, v in axes.items() if k in model} if mp > 1 else {}
        m["layout"] = {"mp": mp, "pp": 1, "sharding": 1, "dp": 1}
        torch.save(m, os.path.join(folder, "meta_state.pdopt"))
    return dst


# ------------------------------------------------------------------------------------------------ GPT pipe <-> plain key names
def gpt_pipe_to_plain(state: dict, num_layers: int) -> dict:
    """``shared_layers.embed.*`` / ``layers.<global idx>.*`` (GPTForPretrainingPipe; desc 0 = embedding, 1..L = decoder layers,
    L+1 = final norm) → ``gpt.embeddings.* / gpt.decoder.layers.<i>.* / gpt.decoder.norm.*`` (GPTForPretraining)."""
    out = {}
    for k, v in state.items():
        if k.startswith("shared_layers.embed."):
            out["gpt.embeddings." + k[len("shared_layers.embed."):]] = v
            continue
        m = re.match(r"layers\.(\d+)\.(.*)$", k)
        if m:
            idx, rest = int(m.group(1)), m.group(2)
            if 1 <= idx <= num_layers:
                out[f"gpt.decoder.layers.{idx - 1}.{rest}"] = v
            elif idx == num_layers + 1:
                out["gpt.decoder." + rest] = v          # rest == "norm.weight" / "norm.bias"
            else:
                out[k] = v
        else:
            out[k] = v
    return out


def gpt_plain_to_pipe(state: dict, num_layers: int) -> dict:
    out = {}
    for k, v in state.items():
        if k.startswith("gpt.embeddings."):
            out["shared_layers.embed." + k[len("gpt.embeddings."):]] = v
            continue
        m = re.match(r"gpt\.decoder\.layers\.(\d+)\.(.*)$", k)
        if m:
            out[f"layers.{int(m.group(1)) + 1}.{m.group(2)}"] = v
        elif k.startswith("gpt.decoder.norm."):
            out[f"layers.{num_layers + 1}.norm." + k[len("gpt.decoder.norm."):]] = v
        else:
            out[k] = v
    return out


def convert(src: str, dst: str, mp: int = 1, to_plain_layers: Optional[int] = None, fuse_qkv: Optional[bool] = None, num_heads: Optional[int] = None,
            num_kv_heads: Optional[int] = None):
    """``num_kv_heads``: K/V heads of a grouped-query model (default ``num_heads``), used by the QKV re-layout."""
    model, optim, meta = merge_checkpoint(src)
    if to_plain_layers is not None:
        model = gpt_pipe_to_plain(model, to_plain_layers)
        if optim is not None:
            optim["state"] = gpt_pipe_to_plain(optim["state"], to_plain_layers)
        meta["merged_tp_axes"] = gpt_pipe_to_plain(meta.get("merged_tp_axes", {}), to_plain_layers)
    if fuse_qkv is not None:
        from ..models.language_model.finetune_module import convert_qkv_layout

        assert num_heads, "--num-heads is required with --fuse-qkv/--split-qkv"
        model = convert_qkv_layout(model, fuse_qkv, num_heads, num_kv_heads)
        optim = None        # moments do not survive a re-layout of fused rows; restart the optimizer
    return split_checkpoint(model, optim, meta, dst, mp)
