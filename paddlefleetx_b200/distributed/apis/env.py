"""Process bootstrap, topology singleton and the seed policy.

Reference behaviour (ppfleetx/distributed/apis/env.py:34-178):
  * python/numpy seed  = ``seed + 100 * pp_rank``
  * ``global_seed``    = same inside an mp group, differs across pp/dp/sharding
  * ``local_seed``     = unique per rank
  * data-parallel rank for sampling = ``dp_rank * sharding_size + sharding_rank``

Bootstrap is torchrun-compatible (RANK / LOCAL_RANK / WORLD_SIZE / MASTER_ADDR / MASTER_PORT): one
process per GPU, NCCL on CUDA and gloo on CPU.
"""
from __future__ import annotations

import datetime
import os
import random
from dataclasses import dataclass, field
from typing import Optional

import numpy as np
import torch
import torch.distributed as dist

from ...parallel.rng import get_rng_state_tracker
from ...parallel.topology import HybridCommGroupForMoE, HybridCommunicateGroup
from ...utils.log import logger

_seed: Optional[int] = None
_dp_seed: Optional[int] = None
_hcg: Optional[HybridCommunicateGroup] = None
_strategy = None


@dataclass
class DistributedStrategy:
    """The handful of knobs the reference passes through ``fleet.DistributedStrategy``
    (env.py:124-148)."""

    hybrid_configs: dict = field(default_factory=lambda: dict(dp_degree=1, mp_degree=1, pp_degree=1, sharding_degree=1))
    pipeline_configs: dict = field(default_factory=lambda: dict(accumulate_steps=1, micro_batch_size=1,
                                                                enable_partial_send_recv=True))
    tensor_parallel_configs: dict = field(default_factory=lambda: dict(tensor_init_seed=1024))
    sharding_configs: dict = field(default_factory=dict)


def world_size() -> int:
    return dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1


def global_rank() -> int:
    return dist.get_rank() if dist.is_available() and dist.is_initialized() else 0


def get_local_rank() -> int:
    return int(os.environ.get("LOCAL_RANK", os.environ.get("PADDLE_RANK_IN_NODE", 0)))


def init_process_group(device: str = "gpu", timeout_s: int = 1800) -> None:
    """Idempotent torchrun-style init.  No-op for a single process without RANK in env."""
    if dist.is_initialized():
        return
    if "RANK" not in os.environ or int(os.environ.get("WORLD_SIZE", "1")) <= 1:
        return
    use_cuda = device == "gpu" and torch.cuda.is_available()
    if use_cuda:
        torch.cuda.set_device(get_local_rank() % max(torch.cuda.device_count(), 1))
    os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
    os.environ.setdefault("MASTER_PORT", "29500")
    kwargs = {}
    if use_cuda:
        kwargs["device_id"] = torch.device("cuda", torch.cuda.current_device())
    dist.init_process_group(backend="nccl" if use_cuda else "gloo",
                            timeout=datetime.timedelta(seconds=timeout_s), **kwargs)


def destroy_process_group() -> None:
    """End of a launcher-started job: every rank meets at a barrier, then the default group and all subgroups are destroyed, so the
    communicator's threads are joined before the interpreter shuts down (left alive, they can abort the process at exit).  No-op without
    a process group."""
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()


def set_hcg(hcg) -> None:
    global _hcg
    _hcg = hcg


def get_hcg() -> HybridCommunicateGroup:
    global _hcg
    if _hcg is None:
        _hcg = HybridCommunicateGroup(world_size=1, rank=0, build_groups=False) if world_size() == 1 \
            else HybridCommunicateGroup(dp=world_size())
    return _hcg


def get_strategy() -> DistributedStrategy:
    global _strategy
    if _strategy is None:
        _strategy = DistributedStrategy()
    return _strategy


def get_seed():
    return _seed


def get_dp_seed():
    return _dp_seed


def init_dist_env(config) -> HybridCommunicateGroup:
    global _strategy
    device = str(config.Global.get("device", "gpu")).lower()
    init_process_group(device)
    d = config.Distributed
    if d.pp_degree > 1 and config.Model.get("sequence_parallel", False):
        assert config.Global.enable_partial_send_recv is False, \
            "pp_degree > 1 with sequence_parallel requires enable_partial_send_recv=False"
    st = DistributedStrategy()
    st.hybrid_configs = dict(dp_degree=d.dp_degree, mp_degree=d.mp_degree, pp_degree=d.pp_degree,
                             sharding_degree=d.sharding.sharding_degree, cp_degree=int(d.get("cp_degree", 1) or 1), cp_mode=str(d.get("cp_mode", "ulysses") or "ulysses"))
    st.pipeline_configs = dict(
        accumulate_steps=config.Global.local_batch_size // config.Global.micro_batch_size,
        micro_batch_size=config.Global.micro_batch_size,
        enable_partial_send_recv=config.Global.enable_partial_send_recv)
    st.tensor_parallel_configs = dict(tensor_init_seed=config.Global.seed)
    st.sharding_configs = dict(d.sharding)
    _strategy = st
    from . import comm_groups

    hcg = comm_groups.create_hcg(st, hcg_name=d.get("hcg", "HybridCommunicateGroup"))
    set_hcg(hcg)
    return hcg


def set_seed(seed: int) -> None:
    global _seed, _dp_seed
    if world_size() > 1:
        h = get_hcg()
        mp_rank, mp_size = h.get_model_parallel_rank(), h.get_model_parallel_world_size()
        pp_rank, pp_size = h.get_stage_id(), h.get_pipe_parallel_world_size()
        dp_rank, dp_size = h.get_data_parallel_rank(), h.get_data_parallel_world_size()
        sh_rank = h.get_sharding_parallel_rank()
    else:
        mp_rank, mp_size, pp_rank, pp_size, dp_rank, dp_size, sh_rank = 0, 1, 0, 1, 0, 1, 0

    random.seed(seed + 100 * pp_rank)
    np.random.seed(seed + 100 * pp_rank)

    ws = world_size()
    non_mp = pp_rank * mp_size + dp_rank * (mp_size * pp_size) + sh_rank * (mp_size * pp_size * dp_size)
    global_seed = seed + 1024 + ws + non_mp
    local_seed = seed + 1024 + 2 * ws + mp_rank + non_mp

    tracker = get_rng_state_tracker()
    tracker.reset()
    tracker.add("global_seed", global_seed)
    tracker.add("local_seed", local_seed)
    torch.manual_seed(global_seed)
    logger.info(f"The global seed is set to {global_seed} and local seed is set to {local_seed}.")
    _seed, _dp_seed = seed, global_seed


def get_data_world_size() -> int:
    if world_size() == 1:
        return 1
    h = get_hcg()
    return h.get_data_parallel_world_size() * h.get_sharding_parallel_world_size() // getattr(h, "cp", 1)      # a context-parallel group is ONE data replica


def get_data_world_rank() -> int:
    if world_size() == 1:
        return 0
    h = get_hcg()
    return (h.get_data_parallel_rank() * h.get_sharding_parallel_world_size() + h.get_sharding_parallel_rank()) // getattr(h, "cp", 1)


def work_at_local_rank0(func):
    def wrapper(*args, **kwargs):
        if get_local_rank() == 0:
            out = func(*args, **kwargs)
        else:
            out = None
        if world_size() > 1:
            dist.barrier()
        return out

    return wrapper
