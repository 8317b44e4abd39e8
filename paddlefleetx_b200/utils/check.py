"""Config / environment sanity checks (reference ppfleetx/utils/check.py: check_version, check_device, check_config)."""
import torch

from .log import logger


def check_version():
    from .version import version_check

    return version_check()


def check_device(device: str):
    if device in ("gpu", "cuda") and not torch.cuda.is_available():
        raise RuntimeError("Global.device is gpu but no CUDA device is visible; set Global.device=cpu for functional runs")
    if device not in ("gpu", "cuda", "cpu"):
        raise ValueError(f"unsupported device '{device}': this framework targets NVIDIA H100 (gpu) with a cpu functional path")


def check_config(cfg):
    g, d = cfg.Global, cfg.get("Distributed", {})
    for key in ("local_batch_size", "micro_batch_size"):
        if g.get(key) is not None and g[key] <= 0:
            raise ValueError(f"Global.{key} must be positive")
    if g.get("local_batch_size") and g.get("micro_batch_size") and g.local_batch_size % g.micro_batch_size:
        raise ValueError("local_batch_size must be a multiple of micro_batch_size")
    sh = d.get("sharding", {}) or {}
    if sh.get("sharding_stage", 1) not in (1, 2, 3):
        raise ValueError("sharding_stage must be 1, 2 or 3")
    if d.get("pp_degree", 1) > 1 and sh.get("sharding_stage", 1) == 3:
        raise ValueError("sharding stage 3 cannot be combined with pipeline parallelism")
    m = cfg.get("Model", {})
    if m.get("hidden_size") and m.get("num_attention_heads") and m.hidden_size % m.num_attention_heads:
        raise ValueError("hidden_size must be divisible by num_attention_heads")
    if m.get("num_attention_heads") and d.get("mp_degree", 1) > 1 and m.num_attention_heads % d.mp_degree:
        raise ValueError("num_attention_heads must be divisible by mp_degree")
    logger.debug("config checks passed")
    return True
