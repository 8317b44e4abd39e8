"""Optimizers.  ``FusedAdamW`` is the workhorse: flat-buffer multi-precision AdamW that is *also* the ZeRO-1/2
sharding optimizer and the data-parallel gradient reducer.

Reference pieces folded into this one class:
  * ``FusedAdamW`` + ``tensor_fusion`` (ppfleetx/optims/optimizer.py:31-56, utils/tensor_fusion_helper.py),
    weight decay skipped for biases and norm parameters,
  * Paddle's ``DygraphShardingOptimizer`` / ``GroupShardedOptimizerStage2`` (stage 1/2: optimizer state and
    gradient shards per sharding rank, param broadcast after the step; ``reduce_overlap`` /
    ``broadcast_overlap`` flags — eager_engine.py:274-307),
  * ``HybridParallelOptimizer``'s cross-group global-norm clip and the scaler's found-inf exchange,
  * ``MixPrecisionOptimizer`` main-grad handling (distributed/apis/amp.py:120-190).

Layout: parameters are packed by ``parallel/flat_buffer.py`` into buckets; every bucket is split evenly over
the sharding group, rank r owning slice r of every bucket (so a bucket can be reduce-scattered as soon as its
gradients are complete, while backward is still running).  On CUDA one step is, per bucket: [reduce-scatter]
-> sumsq kernel -> (one tiny all-reduce) -> clip-coefficient kernel -> fused AdamW kernel -> [all-gather];
the clip coefficient and found-inf flag never visit the host.  With ``use_p2p`` (the CUDA multi-GPU default) the buckets live in
symmetric memory (parallel/symmetric_memory.py) and the ZeRO traffic runs through our own kernels (csrc/comm_nvls.cu): the
reduce-scatter is an in-switch reduction (``multimem.ld_reduce``) that also emits the gradient-norm partial, and AdamW stores the
new low-precision weights once to the multicast address (update + all-gather in one kernel), bucket by bucket underneath the next
forward pass.  Those kernels fit on an SM next to a persistent GEMM CTA, which NCCL's do not.
"""
from __future__ import annotations

import math
import os as _os
from typing import Callable, Dict, List, Optional

import torch
import torch.distributed as dist

from ..ops import _native
from ..ops import functional as OF
from ..parallel import comm_ops as C
from ..parallel import debug_poison as _debug
from ..parallel.flat_buffer import FlatGroup, attach_grad_views, build_flat_groups
from ..utils.log import logger
from .grad_clip import ClipGradByGlobalNorm, ClipGradForMOEByGlobalNorm
from .lr_scheduler import LRScheduler


_DTYPE_CODE = {torch.float16: 0, torch.bfloat16: 1, torch.float32: 3}


def default_decay_fn(name: str, p: torch.nn.Parameter) -> bool:
    """No decay for every bias and every normalisation weight, decay for Linear/Embedding weights — the effect
    of the reference's substring test on Paddle auto-names (optims/optimizer.py:44-49; SURVEY §5.4)."""
    if getattr(p, "no_weight_decay", False):
        return False
    lname = name.lower()
    return not (p.ndim <= 1 or lname.endswith("bias") or "norm" in lname)


_STACKED_EXPERT = {"w1": ("htoh4", "weight"), "b1": ("htoh4", "bias"), "w2": ("h4toh", "weight"), "b2": ("h4toh", "bias")}


def _named_entry(named: dict, name: str) -> dict:
    """Per-parameter optimizer state by name, across the two spellings of MoE expert parameters: a layer on the grouped-GEMM path owns
    stacked tensors (``...grouped.w1`` = [E, 4h, h]) while the expert-loop path (and every checkpoint's model file) names them per expert
    (``...experts.3.htoh4.weight``).  State saved under one spelling loads into the other."""
    if name in named:
        return named[name]
    parts = name.split(".")
    if len(parts) >= 2 and parts[-2] == "grouped" and parts[-1] in _STACKED_EXPERT:       # want stacked, have per expert
        lin, attr = _STACKED_EXPERT[parts[-1]]
        prefix = ".".join(parts[:-2])
        prefix = prefix + "." if prefix else ""
        per, e = [], 0
        while f"{prefix}experts.{e}.{lin}.{attr}" in named:
            per.append(named[f"{prefix}experts.{e}.{lin}.{attr}"])
            e += 1
        if per:
            return {k: (torch.stack([st[k] for st in per]) if all(st.get(k) is not None for st in per) else None) for k in ("moment1", "moment2", "master")}
    if len(parts) >= 4 and parts[-4] == "experts" and parts[-3].isdigit():                  # want per expert, have stacked
        lin, attr = parts[-2], parts[-1]
        stacked = next((k for k, v in _STACKED_EXPERT.items() if v == (lin, attr)), None)
        key = ".".join(parts[:-4] + ["grouped", stacked]) if stacked else None
        if key in named:
            e = int(parts[-3])
            return {k: (v[e] if v is not None else None) for k, v in named[key].items() if k in ("moment1", "moment2", "master")}
    raise KeyError(f"optimizer state has no entry for parameter {name!r}")


class FusedAdamW:
    def __init__(self, learning_rate, parameters=None, beta1: float = 0.9, beta2: float = 0.999, epsilon: float = 1e-8,
                 weight_decay: float = 0.01, grad_clip=None, multi_precision: bool = False, tensor_fusion: bool = True,
                 named_parameters=None, apply_decay_param_fun: Optional[Callable] = None, hcg=None, sharding_stage: int = 1,
                 use_main_grad: bool = False, bucket_mb: int = 512, reduce_overlap: bool = False, broadcast_overlap: bool = False,
                 use_p2p: bool = False, lazy_init: bool = False, params_are_shards: bool = False, direct_grad: Optional[bool] = None,
                 offload: bool = False, step_overlap: bool = False, **unused):
        self._learning_rate = learning_rate
        self.beta1, self.beta2, self.eps, self.weight_decay = float(beta1), float(beta2), float(epsilon), float(weight_decay)
        self.grad_clip = grad_clip
        self.multi_precision = multi_precision
        self.hcg = hcg
        self.use_main_grad = use_main_grad
        self.reduce_overlap = reduce_overlap
        self.broadcast_overlap = broadcast_overlap
        self.sharding_stage = sharding_stage
        self.loss_scale = 1.0            # set by the GradScaler for fp16
        self._step_count = 0
        self._accumulating = False       # inside no_sync(): hooks must not launch reductions
        if named_parameters is None:
            named_parameters = [(f"param_{i}", p) for i, p in enumerate(parameters)]
        named = [(n, p) for n, p in named_parameters if p.requires_grad]
        self._names = {id(p): n for n, p in named}
        decay_fn = apply_decay_param_fun or default_decay_fn
        self._decay = {id(p): bool(decay_fn(n, p)) for n, p in named}

        self.sh_group = hcg.get_sharding_parallel_group() if hcg is not None else None
        self.dp_group = hcg.get_data_parallel_group() if hcg is not None else None
        self.sh_world = C.group_size(self.sh_group)
        self.sh_rank = C.group_rank(self.sh_group)
        self.dp_world = C.group_size(self.dp_group)
        self.replicas = self.sh_world * self.dp_world          # data replicas the gradient is averaged over
        if self.replicas > 1:
            # gradient collectives run beside the backward GEMMs: those keep the 128 x 128 tile, which leaves room on the SM for them
            OF.set_wide_backward(False)
        if params_are_shards:
            # ZeRO-3: the "parameters" handed in are already per-rank shards (parallel/sharding.py): no further
            # partitioning or reduce-scatter here, only the dp all-reduce, the cross-group norm and the update
            self.sh_world, self.sh_rank = 1, 0
        self.offload = bool(offload)
        self.use_p2p = bool(use_p2p) and self.sh_world > 1 and named[0][1].is_cuda and not self.offload
        # ``step_overlap``: the AdamW update of step t is issued bucket by bucket on the side stream in FORWARD order and each module's
        # forward pre-hook waits only for its own buckets, so all but the first bucket's update (bandwidth-bound, ~16 B/parameter streamed)
        # runs underneath the compute-bound GEMMs of the next forward pass instead of in front of it.  Needs direct gradient writes (no
        # memset of the gradient buffer between step and backward) and the device-resident native update.
        self.step_overlap = (bool(step_overlap) or self.use_p2p) and named[0][1].is_cuda and not self.offload
        # the side-stream kernels co-reside with the GEMMs, and the shorter they run the less GEMM time they perturb: 2 CTAs per SM each
        # (at full width the AdamW update takes the whole memory system and the forward GEMMs beside it slow down)
        two_per_sm = str(2 * torch.cuda.get_device_properties(named[0][1].device).multi_processor_count) if named[0][1].is_cuda else "264"
        self._rs_ctas = int(_os.environ.get("PFX_RS_CTAS", two_per_sm))
        self._adamw_ctas = int(_os.environ.get("PFX_ADAMW_CTAS", two_per_sm))      # 0 = 8 CTAs per SM
        self._bcast_ctas = int(_os.environ.get("PFX_BCAST_CTAS", two_per_sm))

        # ---- bucket assignment (reverse registration order: last layers finish backward first)
        bucket_bytes = bucket_mb * 1024 * 1024 if (self.replicas > 1 or self.step_overlap) else (1 << 62)
        bucket_of: Dict[int, int] = {}
        cur, cur_bytes = 0, 0
        for n, p in reversed(named):
            if not self._decay[id(p)]:
                bucket_of[id(p)] = -1          # small no-decay params: one trailing bucket
                continue
            bucket_of[id(p)] = cur
            cur_bytes += p.numel() * p.element_size()
            if cur_bytes >= bucket_bytes:
                cur, cur_bytes = cur + 1, 0

        def key_fn(p):
            return (bucket_of[id(p)], self._decay[id(p)], bool(getattr(p, "tp_sharded", False)), bool(getattr(p, "is_expert", False)),
                    bool(getattr(p, "pp_shared_duplicate", False)))   # [4]: tied copy on another stage, skipped in the norm

        params = [p for _, p in named]
        grad_dtype = torch.float32 if use_main_grad else None
        alloc = None
        self._symm = None
        if self.use_p2p:
            from ..parallel.symmetric_memory import get_allocator

            self._symm = get_allocator(self.sh_group)
            alloc = self._symm.alloc_tensor
        # Direct gradient writes: autograd never owns a view of the flat grad buffer.  ``p.main_grad`` (bf16 or fp32 view) is
        # the only persistent gradient; the wgrad GEMM stores straight into it (first touch after clear_grad = plain store, no
        # zero-fill pass and no read-modify-write), every other parameter's grad is moved in by the post-accumulate hook.
        # That removes the per-parameter ``grad += new`` passes and the whole-buffer memset of the classic layout.
        self.direct_grad = bool(use_main_grad or ((params[0].is_cuda if direct_grad is None else direct_grad) and not params_are_shards))
        # ZeRO stage 2: the full-size gradient of a bucket exists only while its layers are in backward.  Bucketed groups write into a
        # small RING of bucket-sized buffers (bucket i uses slot i % K); when the last gradient of a bucket has arrived it is
        # reduce-scattered into the rank's persistent 1/N gradient shard and the slot is reused K buckets later.  Needs direct gradient
        # writes (a reused slot holds another bucket's data: the first write must be a store, not an accumulation).
        self.grad_ring = bool(self.sharding_stage == 2 and self.sh_world > 1 and self.direct_grad and not params_are_shards and not self.offload
                              and _os.environ.get("PFX_ZERO2_RING", "1") != "0")
        self.groups: List[FlatGroup] = build_flat_groups(params, key_fn, pad_multiple=self.sh_world, grad_dtype=grad_dtype, alloc_fn=alloc,
                                                         allocate_grads=not self.grad_ring)
        self.groups.sort(key=lambda g: (g.key[0] if g.key[0] >= 0 else 1 << 30))
        if self.grad_ring:
            self._build_grad_ring(grad_dtype, alloc)
        if self.direct_grad:
            for g in self.groups:
                attach_grad_views(g, main_grad=True)
                for p in g.params:
                    p._grad_fresh = True
        dev = params[0].device
        self._dev = dev
        for g in self.groups:
            lo, hi = g.shard_range(self.sh_rank, self.sh_world)
            g.meta["lo"], g.meta["hi"] = lo, hi
            lowp = g.param_buf.dtype != torch.float32
            g.meta["has_master"] = lowp and multi_precision
            if lowp and not multi_precision:
                logger.warning("low-precision parameters without multi_precision: optimizer math runs on fp32 copies anyway")
                g.meta["has_master"] = True
            g.meta["master"] = g.param_buf[lo:hi].float().clone() if g.meta["has_master"] else g.param_buf[lo:hi]
            g.meta["m"] = torch.zeros(hi - lo, dtype=torch.float32, device=dev)
            g.meta["v"] = torch.zeros(hi - lo, dtype=torch.float32, device=dev)
            if self.offload:
                # reference ``sharding_offload`` (group_sharded stage 2 + CPU offload, eager_engine.py:295-307): fp32 master weights and both
                # moments live in (pinned) host memory, the update runs on the host and only the low-precision weights return to the device.
                # With 80 GB per GPU this is a capacity escape hatch, not a performance path.
                pin = dev.type == "cuda"
                g.meta["has_master"] = True
                for k2 in ("master", "m", "v"):
                    src = g.meta[k2].detach().float().cpu()
                    g.meta[k2] = src.pin_memory() if pin else src.clone()
            g.meta["pending"] = 0
            g.meta["synced"] = False
            if self.use_p2p:
                g.meta["peer_grads"] = self._symm.peer_ptrs(g.grad_buf)
                g.meta["peer_params"] = self._symm.peer_ptrs(g.param_buf)
                # Multicast includes the sender: an NVLS reduce-scatter / broadcast moves world/(world-1) x the unicast bytes over the
                # busier link direction but needs 1/(world-1) of the load / store instructions (measured at world 2: 0.215 vs 0.126 ms on a
                # 64 MiB shard).  From world 4 the instruction saving wins; below that — or without NVLS — the unicast kernels run (mc = 0).
                use_mc = self.sh_world >= int(_os.environ.get("PFX_NVLS_MIN_WORLD", "4"))
                g.meta["mc_grads"] = self._symm.mc_ptr(g.grad_buf) if use_mc else 0
                g.meta["mc_params"] = self._symm.mc_ptr(g.param_buf) if use_mc else 0
        self._sq = torch.zeros(1, dtype=torch.float32, device=dev)
        self._gscale = torch.ones(1, dtype=torch.float32, device=dev)
        self._found_inf = torch.zeros(1, dtype=torch.float32, device=dev)
        self._gnorm = torch.zeros(1, dtype=torch.float32, device=dev)
        self._comm_stream = torch.cuda.Stream() if dev.type == "cuda" else None
        C.register_side_stream(self._comm_stream)
        C.register_pre_backward(self.finish_param_sync)
        self._hooks = []
        if self.replicas > 1 or self.direct_grad:
            self._register_hooks()
        self._ag_events: Dict[int, "torch.cuda.Event"] = {}
        self._fwd_hooks_installed = False

    # ------------------------------------------------------------------ ZeRO-2 gradient ring
    def _build_grad_ring(self, grad_dtype, alloc) -> None:
        slots = int(_os.environ.get("PFX_ZERO2_SLOTS", "3"))
        dev = self.groups[0].param_buf.device
        mk = (lambda n, dt, d: alloc(n, dt, d).zero_()) if alloc else (lambda n, dt, d: torch.zeros(n, dtype=dt, device=d))
        ring_groups = [g for g in self.groups if g.key[0] >= 0 and not g.key[3]]          # bucketed, not expert-private
        by_dtype: Dict[torch.dtype, List[FlatGroup]] = {}
        for g in ring_groups:
            by_dtype.setdefault(grad_dtype or g.param_buf.dtype, []).append(g)
        self._ring: Dict[torch.dtype, List[torch.Tensor]] = {}
        for g in self.groups:
            gd = grad_dtype or g.param_buf.dtype
            peers = by_dtype.get(gd, [])
            if g in peers and len(peers) > slots:
                if gd not in self._ring:
                    size = max(x.numel for x in peers)
                    self._ring[gd] = [mk(size, gd, dev) for _ in range(slots)]
                idx = peers.index(g)                                  # backward completes buckets in this order
                g.grad_buf = self._ring[gd][idx % slots][:g.numel]
                lo, hi = g.shard_range(self.sh_rank, self.sh_world)
                g.meta["grad_shard"] = torch.zeros(hi - lo, dtype=gd, device=dev)
                g.meta["ring_idx"], g.meta["ring_dtype"], g.meta["shard_fresh"] = idx, gd, True
            else:
                g.grad_buf = mk(g.numel, gd, dev)                     # small / private groups keep a full buffer of their own
        self._ring_order = {gd: [x for x in gs if "ring_idx" in x.meta] for gd, gs in by_dtype.items()}
        self._ring_slots = slots
        n_ring = sum(len(v) for v in self._ring_order.values())
        if n_ring:
            full = sum(x.numel * x.grad_buf.element_size() for v in self._ring_order.values() for x in v)
            held = sum(t.numel() * t.element_size() for v in self._ring.values() for t in v) + sum(
                x.meta["grad_shard"].numel() * x.meta["grad_shard"].element_size() for v in self._ring_order.values() for x in v)
            logger.info(f"ZeRO-2: {n_ring} gradient buckets share {slots} ring slots: {held / 2 ** 20:.0f} MiB of gradient memory instead of {full / 2 ** 20:.0f} MiB")

    def _grad_for_update(self, g: FlatGroup) -> torch.Tensor:
        """This rank's reduced gradient shard of the group."""
        sh = g.meta.get("grad_shard")
        return sh if sh is not None else g.grad_buf[g.meta["lo"]:g.meta["hi"]]

    # ------------------------------------------------------------------ exposed-communication accounting
    def comm_meter_start(self) -> None:
        """Start measuring how long the COMPUTE stream is blocked on the communication stream (gradient reduce-scatter not finished
        when the step needs it, parameter update / all-gather of a bucket not landed when its layer runs).  Every such wait is
        bracketed by two CUDA events on the compute stream: the first completes when the preceding compute work is done, the second when
        the wait is satisfied, so their distance is pure exposed time — 0 when the side stream was ahead."""
        self._meter = []

    def comm_meter_read(self) -> float:
        """Milliseconds of exposed waits since ``comm_meter_start`` (synchronises the device) and stops the meter."""
        pairs, self._meter = (self._meter or []), None
        if pairs:
            torch.cuda.synchronize()
        return float(sum(a.elapsed_time(b) for a, b in pairs))

    def _wait(self, what) -> None:
        """Make the current (compute) stream wait for a stream or event; metered when the meter is on."""
        cur = torch.cuda.current_stream()
        meter = getattr(self, "_meter", None)
        if meter is not None:
            a = torch.cuda.Event(enable_timing=True)
            a.record(cur)
        if isinstance(what, torch.cuda.Stream):
            cur.wait_stream(what)
        else:
            cur.wait_event(what)
        if meter is not None:
            b = torch.cuda.Event(enable_timing=True)
            b.record(cur)
            meter.append((a, b))

    # ------------------------------------------------------------------ basic API
    @property
    def all_fused_tensors(self):
        return [g.param_buf for g in self.groups]

    def parameters(self) -> List[torch.nn.Parameter]:
        return [p for g in self.groups for p in g.params]

    def get_lr(self) -> float:
        lr = self._learning_rate
        return float(lr()) if isinstance(lr, LRScheduler) else float(lr)

    def set_lr(self, lr: float) -> None:
        self._learning_rate = float(lr)

    def clear_grad(self, set_to_zero: bool = True) -> None:
        for g in self.groups:
            g.meta["synced"] = False
            g.meta["pending"] = len(g.params)
            if "grad_shard" in g.meta:
                g.meta["shard_fresh"] = True
            if self.direct_grad:
                for p in g.params:          # lazy zero: the first writer of the step overwrites (see _finalize_fresh)
                    p.grad = None
                    p._grad_fresh = True
            else:
                g.grad_buf.zero_()

    def _finalize_fresh(self, g: FlatGroup) -> None:
        """Parameters that received no gradient since ``clear_grad`` still hold last step's values: zero them now."""
        if not self.direct_grad:
            return
        for p in g.params:
            if p._grad_fresh:
                p.main_grad.zero_()
                p._grad_fresh = False

    zero_grad = clear_grad

    # ------------------------------------------------------------------ gradient readiness hooks
    def _register_hooks(self) -> None:
        for g in self.groups:
            g.meta["pending"] = len(g.params)
            for p in g.params:
                self._hooks.append(p.register_post_accumulate_grad_hook(self._make_hook(g, p)))

    def _make_hook(self, g: FlatGroup, p: torch.nn.Parameter):
        def hook(param):
            if self.direct_grad and param.grad is not None:
                if not getattr(param, "grad_added_to_main_grad", False):
                    mg = param.main_grad
                    if param._grad_fresh:
                        mg.copy_(param.grad)
                    elif mg.dtype == torch.float32 and param.grad.is_cuda and param.grad.dtype != torch.float32 and _native.available():
                        _native.require().accumulate_f32_(mg.view(-1), param.grad.contiguous().view(-1), 1.0)
                        OF._count()
                    else:
                        mg.add_(param.grad)
                param._grad_fresh = False
                param.grad_added_to_main_grad = False
                param.grad = None
            ring = "ring_idx" in g.meta
            if self.replicas == 1:
                # single replica: nothing to reduce, but the bucket's share of the global gradient norm can be taken now, on the side
                # stream underneath the rest of the backward pass, instead of 26 serial passes in front of the update
                if self.step_overlap and not self._accumulating and self._comm_stream is not None and param.is_cuda:
                    g.meta["pending"] -= 1
                    if g.meta["pending"] == 0 and self._norm_counted(g) and _native.available():
                        self._finalize_fresh(g)
                        self._comm_stream.wait_stream(torch.cuda.current_stream())
                        with torch.cuda.stream(self._comm_stream):
                            _native.require().sumsq_(self._grad_for_update(g), self._sq, True)
                        g.meta["sq_fused"] = True
                        OF._count(2)
                return
            if not ring and (self._accumulating or not self.reduce_overlap):
                return
            g.meta["pending"] -= 1
            if g.meta["pending"] == 0 and self.replicas > 1:
                # a ring bucket must leave its slot now — also in the middle of gradient accumulation (its shard accumulates instead)
                self._sync_group_grads(g, async_op=self.reduce_overlap)
                if ring:
                    g.meta["pending"] = len(g.params)
                    g.meta["synced"] = not self._accumulating
        return hook

    class _NoSync:
        def __init__(self, opt):
            self.opt = opt

        def __enter__(self):
            self.prev = self.opt._accumulating
            self.opt._accumulating = True

        def __exit__(self, *exc):
            self.opt._accumulating = self.prev

    def no_sync(self):
        """Gradient-accumulation micro-batches: hooks accumulate locally and launch no collective."""
        return FusedAdamW._NoSync(self)

    # ------------------------------------------------------------------ gradient sync (DP all-reduce / ZeRO reduce-scatter)
    def _sync_group_grads(self, g: FlatGroup, async_op: bool = False) -> None:
        self._finalize_fresh(g)
        if g.meta["synced"] or self.replicas == 1 or g.key[3]:
            g.meta["synced"] = True      # expert parameters are private to their rank: no replica reduction
            return
        lo, hi = g.meta["lo"], g.meta["hi"]
        ring = "ring_idx" in g.meta
        shard = g.meta.get("grad_shard")
        acc = bool(ring and not g.meta["shard_fresh"])       # later micro-batches of an accumulation step add to the shard
        stream_ctx = None
        if async_op and self._comm_stream is not None:
            self._comm_stream.wait_stream(torch.cuda.current_stream())
            stream_ctx = torch.cuda.stream(self._comm_stream)
            stream_ctx.__enter__()
        try:
            out = shard if ring else g.grad_buf[lo:hi]
            if self.sh_world > 1:
                if self.use_p2p:
                    # rank r reduces slice r of every rank's bucket — in the switch (multimem.ld_reduce) or by pulling over the
                    # unicast mappings — and writes the sum back into slice r of its own bucket (nobody else reads that slice).
                    # One barrier in front (every rank's gradients of this bucket are complete); the barrier behind every AdamW
                    # broadcast of the same step is what protects the buckets against the next backward pass.
                    self._symm.barrier()
                    fuse_sq = self._norm_counted(g) and self.dp_world == 1 and not ring
                    _native.require().symm_reduce_scatter(self._symm.mc_ptr(g.grad_buf) if g.meta["mc_grads"] else 0, self._symm.peer_ptrs(g.grad_buf) if ring
                                                          else g.meta["peer_grads"], lo, out, self.sh_rank, _DTYPE_CODE[g.grad_buf.dtype], 1.0, acc,
                                                          self._sq if fuse_sq else None, self._rs_ctas)
                    g.meta["sq_fused"] = fuse_sq
                    if ring:
                        self._symm.barrier()        # the slot is rewritten by another bucket soon: every peer must have finished reading it
                    OF._count(2)
                elif ring:
                    self._nccl_rs_into(g, out, acc)
                else:
                    self._nccl_rs(g)
            if self.dp_world > 1 and self.dp_group.process_group is not None:
                if acc:
                    raise RuntimeError("ZeRO-2 gradient ring with gradient accumulation needs dp_degree == 1 (the dp all-reduce would re-reduce the accumulated shard)")
                dist.all_reduce(out, group=self.dp_group.process_group)
            if ring:
                ev = None
                if g.grad_buf.is_cuda:
                    ev = torch.cuda.Event()
                    ev.record(torch.cuda.current_stream())
                g.meta["rs_done"] = ev
                g.meta["shard_fresh"] = False
                for p in g.params:                   # the slot now belongs to the next bucket: this bucket's next write is a store again
                    p._grad_fresh = True
        finally:
            if stream_ctx is not None:
                stream_ctx.__exit__(None, None, None)
        if ring and g.grad_buf.is_cuda:
            # slot reuse: bucket i+2 writes where bucket i+2-K lived; make the compute stream wait for that reduction now (one bucket of
            # slack against gradients that arrive slightly out of bucket order)
            order = self._ring_order[g.meta["ring_dtype"]]
            j = g.meta["ring_idx"] + 2 - self._ring_slots
            if 0 <= j < len(order) and order[j].meta.get("rs_done") is not None:
                self._wait(order[j].meta["rs_done"])
        g.meta["synced"] = True

    def _nccl_rs_into(self, g: FlatGroup, out: torch.Tensor, accumulate: bool) -> None:
        lo, hi = g.meta["lo"], g.meta["hi"]
        pg = self.sh_group.process_group
        if g.grad_buf.is_cuda:
            dst = torch.empty_like(out) if accumulate else out
            dist.reduce_scatter_tensor(dst, g.grad_buf, group=pg)
        else:   # gloo: no reduce-scatter
            dist.all_reduce(g.grad_buf, group=pg)
            dst = g.grad_buf[lo:hi]
        if accumulate:
            out.add_(dst)
        elif dst is not out:
            out.copy_(dst)

    def _norm_counted(self, g: FlatGroup) -> bool:
        """Does this group enter the (dense) global gradient norm on this rank?  TP-sharded tensors count on every mp rank,
        replicated ones on mp rank 0 only, tied pipeline duplicates never; expert groups have their own norm."""
        mp_rank = self.hcg.get_model_parallel_rank() if self.hcg is not None else 0
        return bool((g.key[2] or mp_rank == 0) and not g.key[4] and not g.key[3])

    def _nccl_rs(self, g: FlatGroup) -> None:
        lo, hi = g.meta["lo"], g.meta["hi"]
        pg = self.sh_group.process_group
        if g.grad_buf.is_cuda:
            dist.reduce_scatter_tensor(g.grad_buf[lo:hi], g.grad_buf, group=pg)
        else:   # gloo: no reduce-scatter
            dist.all_reduce(g.grad_buf, group=pg)

    def _all_gather_params(self, g: FlatGroup) -> None:
        if self.sh_world == 1:
            return
        lo, hi = g.meta["lo"], g.meta["hi"]
        pg = self.sh_group.process_group
        if g.param_buf.is_cuda:
            dist.all_gather_into_tensor(g.param_buf, g.param_buf[lo:hi], group=pg)
        else:
            parts = [torch.empty(hi - lo, dtype=g.param_buf.dtype) for _ in range(self.sh_world)]
            dist.all_gather(parts, g.param_buf[lo:hi].contiguous(), group=pg)
            g.param_buf.copy_(torch.cat(parts))

    # ------------------------------------------------------------------ step
    @torch.no_grad()
    def step(self) -> None:
        """One optimizer step over every flat group: finish the outstanding gradient reductions, global gradient norm (local shards + the mp / pp /
        sharding / expert groups) and clip coefficient on the device, found-inf check for fp16, then the fused multi-precision AdamW on this rank's
        shard — under ZeRO the same kernel delivers the new low-precision weights to every rank (NVLS / peer stores, or an NCCL all-gather) — on the
        side stream when ``step_overlap`` is on, so that the update of the later layers runs beneath the next forward pass."""
        lr = self.get_lr()
        self._step_count += 1
        if _debug.enabled():
            # PFX_DEBUG_POISON=1: the previous step's broadcast must have delivered every parameter (fresh symmetric memory is NaN-poisoned,
            # a consumer that ran ahead of its producer leaves NaN behind) and every rank must have issued the same barriers
            torch.cuda.synchronize() if self._dev.type == "cuda" else None
            for g in self.groups:
                _debug.check_finite(g.param_buf, f"parameter bucket {g.key} before optimizer step {self._step_count}", self.sh_rank)
            if getattr(self, "_symm", None) is not None and hasattr(self._symm, "_bar_counts"):
                _debug.barrier_skew_check(self._symm._bar_counts, self._symm.group)
        if self._comm_stream is not None:
            self._wait(self._comm_stream)
        for g in self.groups:
            self._sync_group_grads(g)
        native = self._dev.type == "cuda" and _native.use_native(self.groups[0].param_buf)
        native_update = native and not self.offload
        inv_scale = 1.0 / (self.loss_scale * self.replicas)
        clip_norm = self.grad_clip.clip_norm if self.grad_clip is not None else 0.0

        # ---- global grad norm over the local shards (+ groups).  ``self._sq`` is zeroed right after it was consumed (end of the
        # previous step), so the symmetric-memory reduce-scatter kernels of THIS step have already added their shards' partials.
        moe_sq = None
        if native:
            lib = _native.require()
            for g in self.groups:
                if self._norm_counted(g) and not g.meta.pop("sq_fused", False):
                    lib.sumsq_(self._grad_for_update(g), self._sq, True)
                    OF._count(2)
            sq = self._sq
            if any(g.key[3] for g in self.groups):
                moe_sq = torch.zeros_like(self._sq)
                for g in self.groups:
                    if g.key[3]:
                        lib.sumsq_(self._grad_for_update(g), moe_sq, True)
        else:
            mp_rank = self.hcg.get_model_parallel_rank() if self.hcg is not None else 0
            sq = torch.zeros(1, dtype=torch.float32, device=self._dev)
            for g in self.groups:
                if g.key[4]:
                    continue
                s = self._grad_for_update(g).float().pow(2).sum()
                if g.key[3]:
                    moe_sq = s.reshape(1) if moe_sq is None else moe_sq + s
                elif g.key[2] or mp_rank == 0:
                    sq += s
        sq = self._reduce_norm(sq, moe_sq)

        # ---- clip coefficient / found-inf on device, fused update
        overlapped = native_update and self.step_overlap and self.direct_grad and self._comm_stream is not None
        if overlapped:
            lib.clip_coef_(sq, inv_scale, clip_norm, self._gscale, self._found_inf, self._gnorm)
            self._sq.zero_()
            OF._count()
            # The side stream starts once the clip coefficient exists; buckets go out in forward order (small no-decay bucket, first
            # layers, ..., last layers).  Under ZeRO the update kernel also delivers the new low-precision weights to every rank
            # (multimem.st / peer stores) and is followed by a group barrier ("every rank's part of this bucket has landed") and an
            # event.  The compute stream is ordered after bucket k only when a module that owns parameters of bucket k runs
            # (install_forward_hooks), so the update of the later layers runs underneath the forward pass of the earlier ones.
            self._comm_stream.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(self._comm_stream):
                for g in sorted(self.groups, key=lambda g: (0 if g.key[0] < 0 else 1, -g.key[0])):
                    lo, hi = g.meta["lo"], g.meta["hi"]
                    wd = self.weight_decay if g.key[1] else 0.0
                    lp = g.param_buf[lo:hi] if g.meta["has_master"] else None
                    shared = self.sh_world > 1 and not g.key[3]
                    if self.use_p2p and shared and g.meta["has_master"]:
                        lib.adamw_symm_broadcast_(g.meta["mc_params"], g.meta["peer_params"], lo, g.meta["master"], self._grad_for_update(g), g.meta["m"],
                                                  g.meta["v"], lr, self.beta1, self.beta2, self.eps, wd, self._step_count, self._gscale,
                                                  self._found_inf, _DTYPE_CODE[g.param_buf.dtype], self.sh_rank, self._bcast_ctas)
                        self._symm.barrier()
                        OF._count(2)
                    else:
                        lib.adamw_flat_(lp, g.meta["master"], self._grad_for_update(g), g.meta["m"], g.meta["v"], lr, self.beta1, self.beta2, self.eps,
                                        wd, self._step_count, self._gscale, self._found_inf, self._adamw_ctas)
                        OF._count()
                        if shared:
                            if self.use_p2p:
                                lib.symm_all_gather(g.meta["mc_params"], g.meta["peer_params"], lo * g.param_buf.element_size(),
                                                    g.param_buf[lo:hi], self.sh_rank, self._rs_ctas)
                                self._symm.barrier()
                                OF._count(2)
                            else:
                                self._all_gather_params(g)
                    ev = torch.cuda.Event()
                    ev.record(self._comm_stream)
                    self._ag_events[id(g)] = ev
            if not self._fwd_hooks_installed:
                self.finish_param_sync()
            return
        if native_update:
            lib.clip_coef_(sq, inv_scale, clip_norm, self._gscale, self._found_inf, self._gnorm)
            self._sq.zero_()
            OF._count()
            for g in self.groups:
                lo, hi = g.meta["lo"], g.meta["hi"]
                wd = self.weight_decay if g.key[1] else 0.0
                lp = g.param_buf[lo:hi] if g.meta["has_master"] else None
                lib.adamw_flat_(lp, g.meta["master"], self._grad_for_update(g), g.meta["m"], g.meta["v"], lr, self.beta1, self.beta2, self.eps,
                                wd, self._step_count, self._gscale, self._found_inf)
                OF._count()
        else:
            norm = sq.sqrt() * inv_scale
            if native:
                self._sq.zero_()          # consumed (``norm`` is a new tensor); the next step's kernels accumulate from zero
            bad = not bool(torch.isfinite(norm))
            coef = 1.0
            if clip_norm > 0 and not bad:
                coef = min(1.0, clip_norm / (float(norm) + 1e-6))
            self._gnorm.copy_(norm.reshape(1))
            self._found_inf.fill_(1.0 if bad else 0.0)
            if not bad:
                bc1 = 1.0 - self.beta1 ** self._step_count
                bc2 = 1.0 - self.beta2 ** self._step_count
                for g in self.groups:
                    lo, hi = g.meta["lo"], g.meta["hi"]
                    grad = self._grad_for_update(g).float() * (inv_scale * coef)
                    m, v, w = g.meta["m"], g.meta["v"], g.meta["master"]
                    if self.offload:
                        grad = grad.to(m.device)              # D2H: the update runs where the state lives
                    m.mul_(self.beta1).add_(grad, alpha=1 - self.beta1)
                    v.mul_(self.beta2).addcmul_(grad, grad, value=1 - self.beta2)
                    wd = self.weight_decay if g.key[1] else 0.0
                    wf = w.float() if w.dtype != torch.float32 else w
                    wf.mul_(1.0 - lr * wd)
                    wf.addcdiv_(m, (v.sqrt() / math.sqrt(bc2)).add_(self.eps), value=-lr / bc1)
                    if wf is not w:
                        w.copy_(wf)
                    if g.meta["has_master"]:
                        g.param_buf[lo:hi].copy_(w)

        # ---- parameter all-gather (ZeRO) — optionally overlapped with the next forward
        if self.sh_world > 1:
            if self.broadcast_overlap and self._comm_stream is not None and self._fwd_hooks_installed:
                # all-gathers run on the communication stream in FORWARD order (small no-decay bucket, then the buckets of
                # the first layers ...); each module's forward pre-hook waits only for the buckets it reads, so layer 0 starts
                # while the gathers of the later layers are still in flight
                self._comm_stream.wait_stream(torch.cuda.current_stream())
                with torch.cuda.stream(self._comm_stream):
                    for g in sorted(self.groups, key=lambda g: (0 if g.key[0] < 0 else 1, -g.key[0])):
                        self._all_gather_params(g)
                        ev = torch.cuda.Event()
                        ev.record(self._comm_stream)
                        self._ag_events[id(g)] = ev
            else:
                for g in self.groups:
                    self._all_gather_params(g)

    # ------------------------------------------------------------------ overlapped parameter all-gather: consumer side
    def install_forward_hooks(self, model: torch.nn.Module) -> None:
        """Make every module wait (on the compute stream) for the side-stream work — parameter all-gather and, with ``step_overlap``, the
        AdamW update — of the buckets holding its own parameters."""
        wanted = (self.broadcast_overlap and self.sh_world > 1) or self.step_overlap or self.use_p2p
        if not (wanted and self._comm_stream is not None) or self._fwd_hooks_installed:
            return
        group_of = {id(p): g for g in self.groups for p in g.params}

        def make(gids):
            def pre_hook(module, inputs):
                if self._ag_events:
                    for gid in gids:
                        ev = self._ag_events.pop(gid, None)
                        if ev is not None:
                            self._wait(ev)
            return pre_hook

        # A module waits for the buckets of the parameters it owns AND of those its direct children own: fused call sites read a child's
        # tensors without calling the child (``OF.fused_ffn(x, self.linear1.weight, ...)``, ``OF.layer_norm(x, self.norm1.weight, ...)``), so the
        # child's own pre-hook would never fire.  Contract: a forward() may touch parameters at most one level below itself directly.
        for mod in model.modules():
            gids = []
            owned = list(mod.parameters(recurse=False))
            for child in mod.children():
                owned.extend(child.parameters(recurse=False))
            for p in owned:
                g = group_of.get(id(p))
                if g is not None and id(g) not in gids:
                    gids.append(id(g))
            if gids:
                mod.register_forward_pre_hook(make(tuple(gids)))
        self._fwd_hooks_installed = True

    def finish_param_sync(self) -> None:
        """Block the compute stream until every in-flight side-stream update / parameter all-gather has landed (checkpointing,
        evaluation of tied / externally-read weights, reading ``found_inf`` / parameters from the host)."""
        if self._ag_events:
            for ev in self._ag_events.values():
                self._wait(ev)
            self._ag_events.clear()

    def _reduce_norm(self, sq: torch.Tensor, moe_sq: Optional[torch.Tensor]) -> torch.Tensor:
        h = self.hcg
        if h is None or not (dist.is_available() and dist.is_initialized()):
            return sq if moe_sq is None else sq + moe_sq
        if moe_sq is not None:
            grp = h.get_moe_group()
            if grp.nranks > 1 and grp.process_group is not None:
                dist.all_reduce(moe_sq, group=grp.process_group)
            # dense part: shards over sharding group, TP/PP parts over check group
        for grp in (h.get_check_parallel_group(), h.get_sharding_parallel_group()):
            if grp.nranks > 1 and grp.process_group is not None:
                dist.all_reduce(sq, group=grp.process_group)
        return sq if moe_sq is None else sq + moe_sq

    # ------------------------------------------------------------------ introspection used by the engine / scaler
    def found_inf(self) -> bool:
        return bool(self._found_inf.item() != 0)

    def grad_norm(self) -> float:
        return float(self._gnorm.item())

    # ------------------------------------------------------------------ checkpointing
    def state_dict(self) -> dict:
        self.finish_param_sync()
        sd = {"step": self._step_count, "groups": []}
        for g in self.groups:
            sd["groups"].append({"key": g.key, "numel": g.numel, "lo": g.meta["lo"], "hi": g.meta["hi"],
                                 "names": [self._names[id(p)] for p in g.params], "offsets": list(g.offsets),
                                 "shapes": [tuple(p.shape) for p in g.params],
                                 "master": g.meta["master"].detach().float().cpu() if g.meta["has_master"] else None,
                                 "moment1": g.meta["m"].cpu(), "moment2": g.meta["v"].cpu()})
        if isinstance(self._learning_rate, LRScheduler):
            sd["LR_Scheduler"] = self._learning_rate.state_dict()
        return sd

    def load_named_state(self, named: dict, step: int = 0) -> None:
        """Fill this rank's shard from a layout-independent ``{param_name: {moment1, moment2, master}}`` dict of full
        (TP-local) tensors — the "universal" optimizer checkpoint written by ``utils/ckpt_convert.py``."""
        self._step_count = step
        for g in self.groups:
            lo, hi = g.meta["lo"], g.meta["hi"]
            for p, off in zip(g.params, g.offsets):
                n = p.numel()
                a, b = max(off, lo), min(off + n, hi)
                if a >= b:
                    continue
                st = _named_entry(named, self._names[id(p)])
                for key, dst in (("moment1", g.meta["m"]), ("moment2", g.meta["v"]), ("master", g.meta["master"] if g.meta["has_master"] else None)):
                    if dst is None or st.get(key) is None:
                        continue
                    dst[a - lo:b - lo].copy_(st[key].reshape(-1)[a - off:b - off])

    def set_state_dict(self, sd: dict) -> None:
        if sd.get("format") == "named":
            self.load_named_state(sd["state"], sd.get("step", 0))
            if "LR_Scheduler" in sd and isinstance(self._learning_rate, LRScheduler):
                self._learning_rate.set_state_dict(sd["LR_Scheduler"])
            return
        self._step_count = sd.get("step", 0)
        assert len(sd["groups"]) == len(self.groups), "optimizer layout mismatch (different bucket/sharding layout?)"
        for g, s in zip(self.groups, sd["groups"]):
            assert s["numel"] == g.numel and s["lo"] == g.meta["lo"], "optimizer shard layout mismatch"
            if s["master"] is not None and g.meta["has_master"]:
                g.meta["master"].copy_(s["master"])
            g.meta["m"].copy_(s["moment1"])
            g.meta["v"].copy_(s["moment2"])
        if "LR_Scheduler" in sd and isinstance(self._learning_rate, LRScheduler):
            self._learning_rate.set_state_dict(sd["LR_Scheduler"])

    load_state_dict = set_state_dict


class AdamW(FusedAdamW):
    """Same engine; kept as a distinct name for configs that say ``name: AdamW``."""


class Adam(FusedAdamW):
    def __init__(self, learning_rate, parameters=None, weight_decay: float = 0.0, **kw):
        # Adam with L2 in the reference configs is always used with weight_decay 0; coupled L2 is not offered
        super().__init__(learning_rate, parameters, weight_decay=0.0 if weight_decay is None else weight_decay, **kw)


class Momentum:
    """SGD with momentum (ViT fine-tune configs).  Per-tensor torch ops: this optimizer is not on any headline
    path (reference re-exports paddle.optimizer.Momentum, optims/optimizer.py:20-28)."""

    def __init__(self, learning_rate, parameters=None, momentum: float = 0.9, weight_decay: float = 0.0, grad_clip=None,
                 named_parameters=None, use_nesterov: bool = False, multi_precision: bool = False, hcg=None, **unused):
        if named_parameters is None:
            named_parameters = [(f"param_{i}", p) for i, p in enumerate(parameters)]
        self._named = [(n, p) for n, p in named_parameters if p.requires_grad]
        self._learning_rate = learning_rate
        self.momentum, self.weight_decay, self.nesterov = momentum, float(weight_decay or 0.0), use_nesterov
        self.grad_clip = grad_clip
        self.hcg = hcg
        self._vel = {id(p): torch.zeros_like(p, dtype=torch.float32) for _, p in self._named}
        self._master = {id(p): p.detach().float().clone() for _, p in self._named if p.dtype != torch.float32}
        self._dp_group = hcg.get_dp_sharding_group() if hcg is not None else None
        self._found_inf = False
        self.loss_scale = 1.0

    def parameters(self):
        return [p for _, p in self._named]

    def get_lr(self) -> float:
        lr = self._learning_rate
        return float(lr()) if isinstance(lr, LRScheduler) else float(lr)

    def no_sync(self):
        import contextlib
        return contextlib.nullcontext()

    def clear_grad(self, set_to_zero: bool = True) -> None:
        for _, p in self._named:
            p.grad = None

    zero_grad = clear_grad

    def found_inf(self) -> bool:
        return self._found_inf

    @torch.no_grad()
    def step(self) -> None:
        params = [p for _, p in self._named if p.grad is not None]
        C.fused_allreduce_gradients(params, self._dp_group)
        if self.loss_scale != 1.0:
            for p in params:
                p.grad.div_(self.loss_scale)
        self._found_inf = not all(bool(torch.isfinite(p.grad).all()) for p in params)
        if self._found_inf:
            return
        if self.grad_clip is not None:
            self.grad_clip(params)
        lr = self.get_lr()
        for p in params:
            w = self._master.get(id(p), p)
            g = p.grad.float()
            if self.weight_decay:
                g = g.add(w.float(), alpha=self.weight_decay)
            v = self._vel[id(p)]
            v.mul_(self.momentum).add_(g)
            upd = g.add(v, alpha=self.momentum) if self.nesterov else v
            w.add_(upd, alpha=-lr)
            if w is not p:
                p.copy_(w)

    def state_dict(self) -> dict:
        sd = {"velocity": {n: self._vel[id(p)].cpu() for n, p in self._named},
              "master_weights": {n: self._master[id(p)].cpu() for n, p in self._named if id(p) in self._master}}
        if isinstance(self._learning_rate, LRScheduler):
            sd["LR_Scheduler"] = self._learning_rate.state_dict()
        return sd

    def set_state_dict(self, sd: dict) -> None:
        for n, p in self._named:
            if n in sd.get("velocity", {}):
                self._vel[id(p)].copy_(sd["velocity"][n])
            if n in sd.get("master_weights", {}) and id(p) in self._master:
                self._master[id(p)].copy_(sd["master_weights"][n])
        if "LR_Scheduler" in sd and isinstance(self._learning_rate, LRScheduler):
            self._learning_rate.set_state_dict(sd["LR_Scheduler"])

    load_state_dict = set_state_dict
