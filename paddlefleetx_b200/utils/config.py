"""YAML config system: ``_base_`` inheritance, ``-o a.b.0.c=v`` overrides and the derived
fields every other layer relies on.

Parity notes (behaviour, not code, follows ppfleetx/utils/config.py):
  * ``_base_: rel/path.yaml`` is resolved recursively, child dicts deep-merge onto the parent
    unless the child dict carries ``_inherited_: False`` (config.py:242-281).
  * ``AttrDict.setdefault`` treats an explicit ``None`` as "missing" (config.py:214-219).
  * overrides accept dotted paths with list indices, values are evaluated as Python literals
    and unknown keys are created with a notice (config.py:333-395).
  * ``dp_degree`` is derived as ``world / (mp*pp*sharding)`` and the product is asserted
    (config.py:33-101); ``global = local * dp * sharding`` and
    ``accumulate_steps = local // micro`` (config.py:104-189).

The world size comes from ``torch.distributed`` when initialised, else from ``WORLD_SIZE``
(torchrun) — there is no separate launcher protocol.
"""
from __future__ import annotations

import argparse
import ast
import copy
import os
import sys
from typing import Any, Iterable, Optional

import yaml

from .log import advertise, logger

__all__ = [
    "AttrDict", "get_config", "get_auto_config", "parse_args", "print_config",
    "override_config", "parse_config", "world_size_hint",
]


class AttrDict(dict):
    """dict with attribute access. ``setdefault`` fills keys whose value is ``None`` too."""

    def __getattr__(self, key: str) -> Any:
        try:
            return self[key]
        except KeyError as e:
            raise AttributeError(key) from e

    def __setattr__(self, key: str, value: Any) -> None:
        self[key] = value

    def __delattr__(self, key: str) -> None:
        del self[key]

    def setdefault(self, key, default=None):
        cur = self.get(key, None)
        if cur is None:
            self[key] = default
            return default
        return cur

    def __deepcopy__(self, memo):
        out = type(self)()
        memo[id(self)] = out
        for k, v in self.items():
            out[k] = copy.deepcopy(v, memo)
        return out


def _wrap(node: Any) -> Any:
    """Recursively convert dicts to AttrDict and literal-looking strings to values."""
    if isinstance(node, dict):
        return AttrDict({k: _wrap(v) for k, v in node.items()})
    if isinstance(node, list):
        return [_wrap(v) for v in node]
    if isinstance(node, str):
        try:
            return ast.literal_eval(node)
        except (ValueError, SyntaxError, MemoryError, RecursionError):
            return node
    return node


def _merge(child: dict, parent: dict) -> dict:
    if child.get("_inherited_", True) is False:
        out = dict(child)
        out.pop("_inherited_")
        return out
    out = dict(parent)
    for k, v in child.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict):
            out[k] = _merge(v, out[k])
        else:
            out[k] = v
    return out


def _load_yaml_tree(path: str, _seen: Optional[set] = None) -> dict:
    _seen = _seen or set()
    real = os.path.realpath(path)
    if real in _seen:
        raise ValueError(f"cyclic _base_ chain at {path}")
    _seen.add(real)
    with open(path, "r", encoding="utf-8") as fh:
        tree = yaml.safe_load(fh) or {}
    base = tree.pop("_base_", None)
    if base is not None:
        parent = _load_yaml_tree(os.path.join(os.path.dirname(path), base), _seen)
        tree = _merge(tree, parent)
    return tree


def create_attr_dict(yaml_config: dict) -> dict:
    """In-place: nested plain dicts become ``AttrDict`` and literal-looking strings (``"1e-4"``, ``"[1, 2]"``, ``"True"``) their values
    (reference utils/config.py:226-240).  ``parse_config`` does the same on a freshly loaded tree; this is the entry point for a config that
    was assembled by hand."""
    for key, value in list(yaml_config.items()):
        yaml_config[key] = _wrap(value)
    return yaml_config


def parse_config(cfg_file: str) -> AttrDict:
    return _wrap(_load_yaml_tree(cfg_file))


# ----------------------------------------------------------------------------- overrides
def _literal(text: str) -> Any:
    try:
        return ast.literal_eval(text)
    except (ValueError, SyntaxError):
        low = text.strip().lower()
        if low in ("true", "false"):
            return low == "true"
        if low in ("none", "null", ""):
            return None
        return text


def _assign(node: Any, keys: list, value: str) -> None:
    head, rest = keys[0], keys[1:]
    if isinstance(node, list):
        idx = int(head)
        if idx >= len(node):
            raise IndexError(f"override index {idx} out of range for list of {len(node)}")
        if rest:
            _assign(node[idx], rest, value)
        else:
            node[idx] = _wrap(_literal(value))
        return
    if not isinstance(node, dict):
        raise TypeError(f"cannot descend into {type(node).__name__} with key {head!r}")
    if rest:
        if head not in node or node[head] is None:
            print(f"A new Series field ({head}) detected!")
            node[head] = AttrDict()
        _assign(node[head], rest, value)
    else:
        if head not in node:
            print(f"A new field ({head}) detected!")
        node[head] = _wrap(_literal(value))


def override(dl, ks: list, v: str) -> None:
    """Set ``dl[ks[0]][ks[1]]... = v`` on a tree of dicts and lists; list levels take integer keys, unknown dict keys are created with a
    printed notice, the value string is read as a Python literal when it is one (reference utils/config.py:333-367)."""
    assert isinstance(dl, (list, dict)), f"{dl} should be a list or a dict"
    assert len(ks) > 0, "length of keys should be larger than 0"
    _assign(dl, list(ks), v)


def override_config(config: AttrDict, options: Optional[Iterable[str]] = None) -> AttrDict:
    for opt in options or ():
        if not isinstance(opt, str) or opt.count("=") < 1:
            raise ValueError(f"override {opt!r} must look like key.sub=value")
        key, value = opt.split("=", 1)
        _assign(config, key.split("."), value)
    return config


# --------------------------------------------------------------------- derived quantities
def world_size_hint() -> int:
    try:
        import torch.distributed as dist

        if dist.is_available() and dist.is_initialized():
            return dist.get_world_size()
    except ImportError:  # pragma: no cover - torch import problems surface elsewhere
        pass
    return int(os.environ.get("WORLD_SIZE", os.environ.get("PADDLE_TRAINERS_NUM", "1")))


def process_dist_config(cfg: AttrDict, nranks: Optional[int] = None) -> None:
    nranks = nranks or world_size_hint()
    dist_cfg = cfg.setdefault("Distributed", AttrDict())
    dist_cfg.setdefault("hcg", "HybridCommunicateGroup")
    mp = dist_cfg.setdefault("mp_degree", 1)
    pp = dist_cfg.setdefault("pp_degree", 1)
    dist_cfg.setdefault("pp_recompute_interval", 1)
    sh = dist_cfg.setdefault("sharding", AttrDict())
    sd = sh.setdefault("sharding_degree", 1)
    sh.setdefault("sharding_stage", 2)
    sh.setdefault("sharding_offload", False)
    sh.setdefault("reduce_overlap", False)
    sh.setdefault("broadcast_overlap", False)

    other = mp * pp * sd
    if nranks % other != 0:
        raise AssertionError(
            f"unreasonable config of dist_strategy: world {nranks} not divisible by mp*pp*sharding={other}")
    dp = dist_cfg.setdefault("dp_degree", nranks // other)
    if dp * other != nranks:
        raise AssertionError(
            f"Mismatched config using {nranks} cards with dp_degree[{dp}], mp_degree[{mp}], "
            f"pp_degree[{pp}] and sharding_degree[{sd}]")

    cp = dist_cfg.setdefault("cp_degree", 1) or 1
    dist_cfg["cp_degree"] = cp
    mode = str(dist_cfg.setdefault("cp_mode", "ulysses") or "ulysses").lower()
    if mode not in ("ulysses", "ring"):
        raise AssertionError(f"cp_mode[{mode}] must be 'ulysses' (all-to-all around attention, cp <= heads / mp) or 'ring' (K / V blocks passed round the group)")
    dist_cfg["cp_mode"] = mode
    if cp > 1:        # context parallelism: cp consecutive data ranks share a batch and split its sequence
        if (dp * sd) % cp != 0:
            raise AssertionError(f"cp_degree[{cp}] must divide dp_degree[{dp}] x sharding_degree[{sd}]")

    if sd > 1 and (sh.sharding_stage == 3 or sh.sharding_offload):
        for flag in ("reduce_overlap", "broadcast_overlap"):
            if sh[flag]:
                logger.warning(f"{flag} only valid for sharding stage 2 without offload")
                sh[flag] = False
    if sh.broadcast_overlap and cfg.get("Engine", {}).get("logging_freq", 1) == 1:
        logger.warning("logging_freq == 1 disables broadcast_overlap; raise logging_freq to keep it.")
        sh.broadcast_overlap = False
    if "fuse_sequence_parallel_allreduce" not in dist_cfg:
        dist_cfg["fuse_sequence_parallel_allreduce"] = False
    if dist_cfg.get("use_main_grad") is True or \
            cfg.get("Engine", {}).get("mix_precision", {}).get("use_main_grad") is True:
        dist_cfg["fuse_sequence_parallel_allreduce"] = False


def process_global_configs(cfg: AttrDict) -> None:
    dist_cfg = cfg.Distributed
    dp, pp, sd = dist_cfg.dp_degree, dist_cfg.pp_degree, dist_cfg.sharding.sharding_degree
    g = cfg.setdefault("Global", AttrDict())
    g["enable_partial_send_recv"] = not (cfg.get("Model", {}).get("sequence_parallel", False) and pp > 1)
    if not g["enable_partial_send_recv"]:
        logger.warning("sequence_parallel with pp_degree > 1: enable_partial_send_recv forced off")

    # Global.flags are process-level knobs; known torch backends ones are applied, rest kept as env.
    for k, v in (g.get("flags") or {}).items():
        os.environ[str(k)] = str(v)
        logger.info(f"Environment variable {k} is set {v}.")

    gbs, lbs = g.get("global_batch_size"), g.get("local_batch_size")
    replicas = dp * sd // int(dist_cfg.get("cp_degree", 1) or 1)          # a context-parallel group consumes one batch
    if gbs is None and lbs is None:
        raise ValueError("global_batch_size or local_batch_size should be set.")
    if gbs is not None and lbs is not None:
        assert gbs // lbs == replicas, (
            f"global_batch_size[{gbs}] should be local_batch_size[{lbs}] x dp[{dp}] x sharding[{sd}]")
    elif gbs is not None:
        assert gbs % replicas == 0, (
            f"global_batch_size[{gbs}] should be divisible by dp[{dp}] x sharding[{sd}]")
        g["local_batch_size"] = gbs // replicas
    else:
        g["global_batch_size"] = lbs * replicas
    g.setdefault("micro_batch_size", g["local_batch_size"])
    assert g["local_batch_size"] % g["micro_batch_size"] == 0, "local_batch_size % micro_batch_size != 0"


def process_engine_config(cfg: AttrDict) -> None:
    eng = cfg.setdefault("Engine", AttrDict())
    sl = eng.setdefault("save_load", AttrDict())
    if sl.get("save_steps") in (None, -1):
        sl["save_steps"] = sys.maxsize
    if sl.get("save_epoch") in (None, -1):
        sl["save_epoch"] = 1
    sl.setdefault("output_dir", "./output")
    if "ckpt_dir" not in sl:
        sl["ckpt_dir"] = None

    amp = eng.setdefault("mix_precision", AttrDict())
    amp.setdefault("enable", False)
    amp.setdefault("scale_loss", 32768)
    for k in ("custom_black_list", "custom_white_list"):
        if k not in amp:
            amp[k] = None

    eng.setdefault("max_steps", 500000)
    eng.setdefault("eval_freq", -1)
    eng.setdefault("eval_iters", 0)
    eng.setdefault("logging_freq", 1)
    eng.setdefault("num_train_epochs", 1)
    if eng.get("test_iters") is None:
        eng["test_iters"] = eng["eval_iters"] * 10
    eng["accumulate_steps"] = cfg.Global.local_batch_size // cfg.Global.micro_batch_size


_VALID_DEVICES = ("gpu", "cpu")


def check_config(cfg: AttrDict) -> None:
    """One backend (CUDA sm_90a) plus the CPU/gloo correctness path; XPU/NPU/MLU/ROCm dropped."""
    device = str(cfg.Global.get("device", "gpu")).lower()
    if device not in _VALID_DEVICES:
        raise ValueError(f"device({device}) is not in {list(_VALID_DEVICES)}; this framework targets H100 "
                         "(gpu) with a cpu/gloo path for tests")
    if device == "gpu":
        import torch

        if not torch.cuda.is_available():
            logger.warning("Global.device=gpu but no CUDA device is visible; falling back to cpu")
            cfg.Global["device"] = "cpu"


def print_dict(d: dict, delimiter: int = 0) -> None:
    """Log a nested dict one key per line, children indented by four columns, a rule after every top-level section
    (reference utils/config.py:284-301)."""
    pad = " " * delimiter
    for k in sorted(d, key=str):
        v = d[k]
        if isinstance(v, dict):
            logger.info(f"{pad}{k} : ")
            print_dict(v, delimiter + 4)
        elif isinstance(v, list) and v and isinstance(v[0], dict):
            logger.info(f"{pad}{k} : ")
            for item in v:
                if isinstance(item, dict):
                    print_dict(item, delimiter + 4)
                else:          # a bare op name among ``{op: {args}}`` entries (``- ToCHWImage``)
                    logger.info(f"{pad}    {item}")
        else:
            logger.info(f"{pad}{k} : {v}")
        if delimiter == 0:
            logger.info("-" * 60)


def print_config(cfg: AttrDict) -> None:
    advertise()
    print_dict(cfg)


def get_config(fname: str, overrides: Optional[Iterable[str]] = None, show: bool = False,
               nranks: Optional[int] = None) -> AttrDict:
    if not os.path.exists(fname):
        raise FileNotFoundError(f"config file({fname}) is not exist")
    cfg = parse_config(fname)
    override_config(cfg, overrides)
    process_dist_config(cfg, nranks)
    process_global_configs(cfg)
    process_engine_config(cfg)
    cfg = _wrap(cfg)
    if show:
        print_config(cfg)
    check_config(cfg)
    return cfg


def get_auto_config(fname: str, overrides: Optional[Iterable[str]] = None, show: bool = False,
                    nranks: Optional[int] = None) -> AttrDict:
    """Auto-parallel configs (reference: config.py:418-634) share the eager pipeline here: the
    ``ProcessMesh`` the reference hands to its static-graph planner is just our hybrid topology,
    so the mesh is recorded under ``Distributed.mesh`` and the eager engine executes it."""
    raw = parse_config(fname)
    override_config(raw, overrides)
    raw = _wrap(raw)
    if (raw.get("Distributed") or {}).get("auto_layout", False):
        # ``Distributed.auto_layout: True``: the planner (utils/layout_planner.py) picks degrees, ZeRO stage, micro-batch and recompute for this
        # world size and the config is derived with them; the global batch stays what the YAML's per-GPU batch implies
        from .layout_planner import ModelShape, plan_layouts

        world = nranks or world_size_hint()
        d0, g0 = raw.Distributed, raw.Global
        lb0 = int(g0.get("local_batch_size") or g0.get("micro_batch_size") or 1)
        per_gpu = max(lb0 // (int(d0.get("mp_degree", 1) or 1) * int(d0.get("pp_degree", 1) or 1)), 1)
        plans = plan_layouts(ModelShape.from_config(raw), world, per_gpu, top=1)
        if not plans:
            raise ValueError(f"auto_layout: no layout of this model fits {world} x 80 GB; add GPUs or reduce the batch / sequence length")
        best = plans[0]
        extra = best.overrides() + [f"Global.local_batch_size={per_gpu * best.mp * best.pp * best.cp}", "Global.global_batch_size=None",
                                    "Distributed.auto_layout=False"]
        cfg = get_config(fname, list(overrides or []) + extra, show=False, nranks=nranks)
        cfg.Distributed["plan"] = AttrDict(describe=best.describe(), est_step_ms=best.est_step_s * 1e3, est_mem_gb=best.est_mem_gb,
                                          breakdown_ms={k: v * 1e3 for k, v in best.breakdown.items()})
    else:
        cfg = get_config(fname, overrides, show=False, nranks=nranks)
    d = cfg.Distributed
    cfg.Distributed["mesh"] = AttrDict(
        dim_names=["pp", "dp", "mp"], shape=[d.pp_degree, d.dp_degree * d.sharding.sharding_degree, d.mp_degree])
    if show:
        print_config(cfg)
    return cfg


# ---- the reference's auto-parallel config steps (utils/config.py:418-613) as individually callable functions.  ``get_auto_config`` above
# derives the same quantities through the eager pipeline; these serve code that assembles an auto config step by step.
def process_auto_dist_configs(config: AttrDict, nranks: Optional[int] = None) -> None:
    """Degrees for the auto engine: ``dp = nranks / (mp * pp)`` — ZeRO sharding lives INSIDE the data dimension here (it is a strategy of the
    data-parallel ranks, ``Strategy.sharding``), unlike the eager path where it is a topology axis of its own."""
    d = config["Distributed"]
    nranks = nranks or world_size_hint()
    mp, pp = d.setdefault("mp_degree", 1) or 1, d.setdefault("pp_degree", 1) or 1
    sh = d.setdefault("sharding", AttrDict())
    sd = sh.setdefault("sharding_degree", 1) or 1
    other = mp * pp
    assert nranks % other == 0, "Requires nranks should be divided by mp_degree*pp_degree."
    dp = d.setdefault("dp_degree", nranks // other) or nranks // other
    d["dp_degree"] = dp
    assert nranks == dp * other, (f"Mismatched config using {nranks} cards with dp_degree[{dp}],mp_degree[{mp}], pp_degree[{pp}] and "
                                  f"sharding_degree[{sd}]")


def process_auto_global_configs(config: AttrDict) -> None:
    d, g = config["Distributed"], config["Global"]
    dp, pp = d["dp_degree"], d["pp_degree"]
    g["enable_partial_send_recv"] = True
    if (config.get("Model") or {}).get("sequence_parallel") and pp > 1:
        g["enable_partial_send_recv"] = False
        logger.warning("if config.Distributed.pp_degree > 1 and config.Model.sequence_parallel is True, "
                       "config.Global.enable_partial_send_recv will be set False.")
    gbs, lbs = g.get("global_batch_size"), g.get("local_batch_size")
    if gbs is None and lbs is None:
        raise ValueError("global_batch_size or local_batch_size should be set.")
    if gbs is not None and lbs is not None:
        assert gbs // lbs == dp, f"global_batch_size[{gbs}] should be divided by local_batch_size[{lbs}] when dp_degree is [{dp}]"
    elif gbs is not None:
        assert gbs % dp == 0, f"global_batch_size[{gbs}] should be divided by dp_degree[{dp}]"
        g["local_batch_size"] = gbs // dp
    else:
        g["global_batch_size"] = lbs * dp
    assert g["local_batch_size"] % g["micro_batch_size"] == 0


def process_auto_engine_configs(config: AttrDict) -> None:
    e = config.Engine
    if e.get("verbose") is None:
        e["verbose"] = 2
    if e.get("logging_freq") is None:
        e["logging_freq"] = 10
    sl = e.setdefault("save_load", AttrDict())
    if sl.get("save_steps") in (None, -1):
        sl["save_steps"] = sys.maxsize
    if sl.get("save_epoch") in (None, -1):
        sl["save_epoch"] = 1
    sl.setdefault("output_dir", "./output")
    sl.setdefault("ckpt_dir", None)
    for key, default in (("max_steps", 500000), ("eval_freq", -1), ("eval_iters", 0), ("num_train_epochs", 1)):
        e.setdefault(key, default)
    if e.get("test_iters") is None:
        e["test_iters"] = e["eval_iters"] * 10
    e["accumulate_steps"] = config.Global.local_batch_size // config.Global.micro_batch_size


def process_auto_strategy(config: AttrDict) -> None:
    """``Engine.strategy``: the knobs the reference hands to ``auto.Strategy`` (amp, recompute, sharding, gradient merge, QAT, tuning) as one
    plain ``AttrDict`` with the same section / field names — ``AutoEngine`` reads them from here."""
    e = config.Engine
    amp_cfg = e.get("mix_precision") or {}
    st = AttrDict(auto_mode="semi", seed=config.Global.get("seed"))
    st["amp"] = AttrDict(enable=amp_cfg.get("enable", False), dtype=amp_cfg.get("dtype", "float16"), level=amp_cfg.get("level", "o2"),
                         init_loss_scaling=amp_cfg.get("scale_loss", 32768), custom_black_list=amp_cfg.get("custom_black_list") or [],
                         custom_white_list=amp_cfg.get("custom_white_list") or [], use_fp16_guard=amp_cfg.get("use_fp16_guard", False),
                         use_bf16_guard=amp_cfg.get("use_bf16_guard", False))
    st["recompute"] = AttrDict(enable=False, no_recompute_segments=[], enable_tuning=False)
    model = config.get("Model")
    if model is not None:
        skip = model.get("no_recompute_layers") or []
        assert isinstance(skip, list), "no_recompute_layers should be a list"
        assert all(isinstance(i, int) for i in skip), "all values in no_recompute_layers should be an integer"
        if skip:
            assert min(skip) >= 0, "the min value in no_recompute_layers should >= 0"
            assert max(skip) < model["num_layers"], "the max value in no_recompute_layers should < num_layers"
        skip = sorted(set(skip))
        model["no_recompute_layers"] = skip
        tuning = config.get("Tuning") or {}
        st["recompute"] = AttrDict(enable=model.get("use_recompute", False), no_recompute_segments=skip,
                                   enable_tuning=bool(tuning) and bool(tuning.get("tuning_recompute", False)))
    sh = config.Distributed.get("sharding") or {}
    st["sharding"] = AttrDict(enable=sh.get("sharding_degree", 1) > 1, degree=sh.get("sharding_degree", 1), stage=sh.get("sharding_stage", 1))
    k = e.get("accumulate_steps", 1) or 1
    st["gradient_merge"] = AttrDict(enable=k > 1, k_steps=k)
    q = config.get("Quantization") or {}
    st["qat"] = AttrDict(enable=q.get("enable", False), channel_wise_abs_max=q.get("channel_wise_abs_max", True), weight_bits=q.get("weight_bits", 8),
                         activation_bits=q.get("activation_bits", 8), onnx_format=q.get("onnx_format", True))
    t = config.get("Tuning") or {}
    st["tuning"] = AttrDict(enable=t.get("enable", False), profile_start_step=t.get("profile_start_step", 1),
                            profile_end_step=t.get("profile_end_step", 1), run_after_tuning=t.get("run_after_tuning", True), debug=t.get("debug", True))
    e["strategy"] = st


def process_auto_ckpt_dir(config: AttrDict) -> None:
    """``Engine.save_load.ckpt_dir`` of an auto run is a ``dirname/prefix`` (files ``<prefix>_dist<rank>.*``), not a directory; a prefix
    whose parent directory does not exist is dropped with a warning so that training starts from scratch."""
    sl = config["Engine"]["save_load"]
    ckpt = sl.get("ckpt_dir")
    if ckpt is None:
        return
    assert not os.path.isdir(ckpt), (f"Wrong setting of ckpt_dir! ckpt_dir can't be a folder, but {ckpt} is a folder. Your `ckpt_dir` should be "
                                     "`dirname/prefix` like `output/auto` if your model path is `output/auto_dist0.pdparams`")
    assert not os.path.exists(ckpt), "Wrong setting of ckpt_dir: give the checkpoint prefix (e.g. gpt_auto_model_save/auto), not a file"
    parent = os.path.split(ckpt)[0]
    if parent and not os.path.exists(parent):
        logger.warning(f"{parent} path is not existed! we will set ckpt_dir None.")
        sl["ckpt_dir"] = None


def parse_args(argv: Optional[list] = None) -> argparse.Namespace:
    parser = argparse.ArgumentParser("paddlefleetx_b200 train/eval/export script")
    parser.add_argument("-c", "--config", type=str, default="configs/config.yaml", help="config file path")
    parser.add_argument("-o", "--override", action="append", default=[], help="config options to be overridden")
    return parser.parse_args(argv)
