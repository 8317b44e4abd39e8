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


def check_kv_heads(m, d, compress) -> None:
    """``Model.num_key_value_heads`` (grouped-query attention; unset = ``num_attention_heads``)."""
    heads, kv = m.get("num_attention_heads"), m.get("num_key_value_heads")
    if kv is None or not heads:
        return
    if kv < 1 or heads % kv:
        raise ValueError(f"num_attention_heads ({heads}) must be a multiple of num_key_value_heads ({kv})")
    if d.get("mp_degree", 1) > 1 and kv % d.mp_degree:
        raise ValueError(f"num_key_value_heads ({kv}) must be divisible by mp_degree ({d.mp_degree}): tensor parallelism shards whole K/V groups")
    if kv == heads:
        return
    if d.get("cp_degree", 1) > 1:
        raise ValueError("num_key_value_heads < num_attention_heads is not supported with context parallelism (Distributed.cp_degree > 1)")
    prune = compress.get("Prune") or {}
    if prune.get("enable", False) and prune.get("prune_heads", True):
        raise ValueError("Compress.Prune head pruning does not support num_key_value_heads < num_attention_heads; "
                         "set Compress.Prune.prune_heads=False to prune the FFN only")


def check_ffn_activation(m, d, compress) -> None:
    """``Model.ffn_activation``: ``gelu`` (default) or ``swiglu`` (gated FFN of width ``ffn_hidden_size``, ``linear1`` holding gate / up pairs)."""
    act = m.get("ffn_activation")
    if act is None or act == "gelu":
        return
    if act != "swiglu":
        raise ValueError(f"Model.ffn_activation must be gelu or swiglu, got {act!r}")
    if (m.get("moe_configs") or {}).get("expert_mode", False):
        raise ValueError("ffn_activation: swiglu is not supported with moe_configs (the MoE experts keep the GELU FFN)")
    prune = compress.get("Prune") or {}
    if prune.get("enable", False):
        raise ValueError("Compress.Prune does not support ffn_activation: swiglu (FFN channel pruning would have to remove gate / up pairs)")
    f, mp = m.get("ffn_hidden_size"), d.get("mp_degree", 1)
    if f and mp > 1 and f % mp:
        raise ValueError(f"ffn_hidden_size ({f}) must be divisible by mp_degree ({mp}) under ffn_activation: swiglu: "
                         "tensor parallelism shards whole gate / up pairs")


def check_document_mask(m, d, data) -> None:
    """``Model.reset_attention_mask`` (attention stays inside each packed document) needs ``Data.*.dataset.reset_position_ids``, which
    produces the position ids the mask is derived from, and a layout whose attention sees whole sequences with their positions."""
    if not m.get("reset_attention_mask", False):
        return
    sets = [data[k].get("dataset", {}) or {} for k in ("Train", "Eval") if data.get(k)]
    if not sets or not all(ds.get("reset_position_ids", False) for ds in sets):
        raise ValueError("Model.reset_attention_mask needs Data.*.dataset.reset_position_ids: true (without restarting positions the "
                         "document mask would silently be plain causal)")
    if d.get("pp_degree", 1) > 1:
        raise ValueError("Model.reset_attention_mask is not supported with pipeline parallelism (Distributed.pp_degree > 1): "
                         "later stages receive no position ids")
    if d.get("cp_degree", 1) > 1:
        raise ValueError("Model.reset_attention_mask is not supported with context parallelism (Distributed.cp_degree > 1): "
                         "the ring and Ulysses layouts shard the sequence")


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
    check_kv_heads(m, d, cfg.get("Compress", {}) or {})
    check_ffn_activation(m, d, cfg.get("Compress", {}) or {})
    check_document_mask(m, d, cfg.get("Data", {}) or {})
    logger.debug("config checks passed")
    return True
