"""ZeRO stage 3: parameter sharding with per-layer gather / release and gradient reduce-scatter.

Role of Paddle's ``group_sharded_parallel(level='p_g_os')`` / ``GroupShardedStage3`` in the reference
(eager_engine.py:281-307,564-572,736-737).  Stage 1/2 (optimizer-state / gradient sharding) live in the flat
optimizer (``optims/optimizer.py``); this module adds the parameter dimension:

  * the model is cut into *units* (each transformer layer = one unit, everything else = a resident unit),
  * every unit owns flat buffers (one per parameter class: decay x tensor-parallel) whose 1/world shard is the only
    persistent copy; the optimizer updates those shards,
  * forward: ``pre-forward`` hook all-gathers the unit (and prefetches the next one on the communication stream),
    ``post-forward`` releases it; backward: ``pre-backward`` hook re-gathers, and once every parameter of the unit
    has its gradient the flat gradient is reduce-scattered into the shard gradient and the unit is released,
  * activation recompute composes: the re-forward inside backward gathers through the same hook and the unit stays
    resident until its gradients are reduced,
  * unlike the reference, stage 3 composes with tensor parallelism (BASELINE config #3: mp x stage-3),
  * on CUDA the gathers and the gradient reduce-scatter are OUR kernels over symmetric memory (csrc/comm_nvls.cu): every rank stores its
    shard once through the NVLink-SHARP multicast address (``multimem.st``: the switch replicates it into all ranks' copy of the unit
    buffer) and reduces its gradient slice in the switch (``multimem.ld_reduce``); the full-size unit buffers come from a pool of
    symmetric buffers that is reused layer after layer.  ``PFX_ZERO3_NCCL=1`` (or CPU / gloo) selects the plain collectives.
"""
from __future__ import annotations

import contextlib
from typing import Dict, List, Optional, Tuple

import torch
import torch.distributed as dist
import torch.nn as nn

from . import comm_ops as C
from .flat_buffer import FlatGroup, _align


class _Unit:
    def __init__(self, name: str, module: Optional[nn.Module], params: List[Tuple[str, nn.Parameter]], resident: bool):
        self.name, self.module, self.named, self.resident = name, module, params, resident
        self.groups: List[dict] = []
        self.gathered = False
        self.pending_grads = 0
        self.grads_attached = False
        self.gather_event = None       # set while a prefetched all-gather is in flight on the communication stream
        self.index = 0


class GroupShardedStage3(nn.Module):
    def __init__(self, model: nn.Module, hcg, unit_classes: Tuple[str, ...] = ("TransformerDecoderLayer", "TransformerEncoderLayer", "Block"),
                 decay_fn=None, offload: bool = False):
        super().__init__()
        from ..optims.optimizer import default_decay_fn

        self._layers = model
        self.hcg = hcg
        self.group = hcg.get_sharding_parallel_group()
        self.world, self.rank = C.group_size(self.group), C.group_rank(self.group)
        self.dp_group = hcg.get_data_parallel_group()
        self._decay_fn = decay_fn or default_decay_fn
        self._in_backward = False
        self._accumulating = False
        self._comm_stream = torch.cuda.Stream() if next(model.parameters()).is_cuda else None
        import os

        self._symm = None
        self._pool: Dict[Tuple, List[torch.Tensor]] = {}
        if self._comm_stream is not None and self.world > 1 and self.group.process_group is not None and os.environ.get("PFX_ZERO3_NCCL", "0") != "1":
            from ..ops import _native

            if _native.available():
                from .symmetric_memory import get_allocator

                self._symm = get_allocator(self.group)
                self._lib = _native.require()
        self.units: List[_Unit] = []
        self._build_units(unit_classes)
        self.prefetch = True
        for i, u in enumerate(self.units):
            u.index = i
            self._shard_unit(u)
            self._install_hooks(u)
        self._release_all(force=False)

    # ------------------------------------------------------------------ partitioning
    def _build_units(self, unit_classes) -> None:
        claimed = set()
        for mod_name, mod in self._layers.named_modules():
            if mod.__class__.__name__ in unit_classes:
                ps = [(f"{mod_name}.{n}", p) for n, p in mod.named_parameters() if p.requires_grad and id(p) not in claimed]
                if ps:
                    claimed.update(id(p) for _, p in ps)
                    self.units.append(_Unit(mod_name, mod, ps, resident=False))
        rest = [(n, p) for n, p in self._layers.named_parameters() if p.requires_grad and id(p) not in claimed]
        if rest:
            self.units.insert(0, _Unit("__resident__", None, rest, resident=True))

    def _shard_unit(self, u: _Unit) -> None:
        buckets: Dict[Tuple, List[Tuple[str, nn.Parameter]]] = {}
        for n, p in u.named:
            key = (bool(self._decay_fn(n, p)), bool(getattr(p, "tp_sharded", False)), bool(getattr(p, "is_expert", False)), p.dtype)
            buckets.setdefault(key, []).append((n, p))
        for key, plist in buckets.items():
            dtype, dev = key[3], plist[0][1].device
            esize = torch.empty(0, dtype=dtype).element_size()
            offsets, cur = [], 0
            for _, p in plist:
                offsets.append(cur)
                cur += _align(p.numel(), esize)
            unit_elems = max(256 // esize, 1) * self.world
            total = (cur + unit_elems - 1) // unit_elems * unit_elems
            full = torch.zeros(total, dtype=dtype, device=dev)
            for (_, p), o in zip(plist, offsets):
                full[o:o + p.numel()].copy_(p.data.reshape(-1))
                p.data = full[o:o + p.numel()].view(p.shape)      # from now on the parameter IS a view of the unit's flat buffer (what
                # load_state_dict / get_all_parameters rely on, also for the resident unit that is never re-gathered before the first step)
            s = total // self.world
            shard = nn.Parameter(full[self.rank * s:(self.rank + 1) * s].clone())
            shard.tp_sharded = key[1]
            if key[2]:
                shard.is_expert = True
            shard.grad = None
            u.groups.append(dict(key=key, params=[p for _, p in plist], names=[n for n, _ in plist], offsets=offsets, shapes=[p.shape for _, p in plist],
                                 total=total, shard=shard, full=full, grad_full=None))
        u.gathered = True

    # ------------------------------------------------------------------ hooks
    def _install_hooks(self, u: _Unit) -> None:
        if u.module is not None:
            u.module.register_forward_pre_hook(lambda m, a, u=u: self._use(u))
            u.module.register_forward_hook(lambda m, a, o, u=u: self._after_forward(u))
            u.module.register_full_backward_pre_hook(lambda m, g, u=u: self._before_backward(u))
        else:
            self._layers.register_forward_pre_hook(lambda m, a, u=u: self._gather(u))
        for g in u.groups:
            for p in g["params"]:
                p.register_post_accumulate_grad_hook(lambda param, u=u: self._grad_ready(u))

    def _alloc_full(self, g: dict) -> torch.Tensor:
        if self._symm is None:
            return torch.empty(g["total"], dtype=g["shard"].dtype, device=g["shard"].device)
        return self._pool_take(g["total"], g["shard"].dtype)

    # symmetric unit buffers: taken / returned in the same order on every rank (the program is SPMD), so the collective allocation of a
    # new buffer — when the free list of that size is empty — happens on all ranks together
    def _pool_take(self, numel: int, dtype) -> torch.Tensor:
        free = self._pool.setdefault((numel, dtype), [])
        return free.pop() if free else self._symm.alloc_tensor(numel, dtype)

    def _pool_give(self, t: Optional[torch.Tensor]) -> None:
        if t is None or self._symm is None or t.numel() == 0:
            return
        try:
            self._symm.peer_ptrs(t)        # the construction-time full buffers are ordinary tensors: they must not enter the pool
        except ValueError:
            return
        self._pool.setdefault((t.numel(), t.dtype), []).append(t)

    def _chan(self) -> int:
        """Barrier channel by issuing stream (prefetches run on the communication stream, everything else on the compute stream): two
        streams must never share a channel's arrival counter."""
        return 2 if (self._comm_stream is not None and torch.cuda.current_stream() == self._comm_stream) else 3

    def _symm_all_gather(self, full: torch.Tensor, shard: torch.Tensor) -> None:
        """full[r * s : (r + 1) * s] = rank r's shard, on every rank: barrier (every rank is done with this buffer's previous contents and
        its shard is final) -> one multimem / peer store pass -> barrier (everything has landed)."""
        sm, ch = self._symm, self._chan()
        sm.barrier(channel=ch)
        self._lib.symm_all_gather(sm.mc_ptr(full) if self.world >= 4 else 0, sm.peer_ptrs(full), self.rank * shard.numel() * shard.element_size(),
                                  shard, self.rank, 64)
        sm.barrier(channel=ch)

    def _gather(self, u: _Unit, prefetch: bool = False) -> None:
        """All-gather the unit's parameters.  ``prefetch`` issues the collective on the communication stream and returns at once;
        the consumer side (`_use`) makes the compute stream wait for it."""
        if u.gathered:
            return
        side = prefetch and self._comm_stream is not None and self.world > 1
        if side:
            self._comm_stream.wait_stream(torch.cuda.current_stream())      # shards are final (optimizer step) before we read them
        with (torch.cuda.stream(self._comm_stream) if side else contextlib.nullcontext()):
            for g in u.groups:
                full = self._alloc_full(g)
                if self.world > 1 and self.group.process_group is not None:
                    if self._symm is not None:
                        self._symm_all_gather(full, g["shard"].data)
                    elif full.is_cuda:
                        dist.all_gather_into_tensor(full, g["shard"].data, group=self.group.process_group)
                    else:
                        parts = [torch.empty_like(g["shard"].data) for _ in range(self.world)]
                        dist.all_gather(parts, g["shard"].data.contiguous(), group=self.group.process_group)
                        full.copy_(torch.cat(parts))
                else:
                    full.copy_(g["shard"].data)
                g["full"] = full
                for p, o, shp in zip(g["params"], g["offsets"], g["shapes"]):
                    p.data = full[o:o + shp.numel()].view(shp)
            if side:
                u.gather_event = torch.cuda.Event()
                u.gather_event.record(self._comm_stream)
        u.gathered = True

    def _use(self, u: _Unit) -> None:
        """Gather now if nobody prefetched; otherwise wait for the prefetch.  Then prefetch the neighbour that runs next
        (the following unit in forward, the preceding one in backward) so its all-gather overlaps this unit's compute."""
        self._gather(u)
        if u.gather_event is not None:
            cur = torch.cuda.current_stream()
            cur.wait_event(u.gather_event)
            for g in u.groups:
                if g["full"] is not None:
                    g["full"].record_stream(cur)         # allocated on the communication stream, consumed here
            u.gather_event = None
        if self._comm_stream is not None and self.world > 1 and self.prefetch:
            j = u.index + (-1 if self._in_backward else 1)
            if 0 <= j < len(self.units) and not self.units[j].resident and not self.units[j].gathered:
                self._gather(self.units[j], prefetch=True)

    def _release(self, u: _Unit, force: bool = False) -> None:
        if not u.gathered or (u.resident and not force):
            return
        if u.gather_event is not None:          # prefetched but never consumed: order the free after the collective
            torch.cuda.current_stream().wait_event(u.gather_event)
            u.gather_event = None
        for g in u.groups:
            for p in g["params"]:
                p.data = torch.empty(0, dtype=p.dtype, device=p.device)
            self._pool_give(g["full"])
            g["full"] = None
        u.gathered = False

    def _release_all(self, force: bool) -> None:
        for u in self.units:
            self._release(u, force)

    def _after_forward(self, u: _Unit) -> None:
        # training forward with autograd keeps nothing resident (re-gathered in backward); the recompute re-forward
        # that runs *inside* backward must keep the unit until its gradients have been reduced
        if not self._in_backward:
            self._release(u)

    def _attach_grad_buffers(self, u: _Unit) -> None:
        if u.grads_attached:
            return
        for g in u.groups:
            if self._symm is not None and not g["key"][2]:
                g["grad_full"] = self._pool_take(g["total"], g["shard"].dtype)
                g["grad_full"].zero_()
            else:
                g["grad_full"] = torch.zeros(g["total"], dtype=g["shard"].dtype, device=g["shard"].device)
            for p, o, shp in zip(g["params"], g["offsets"], g["shapes"]):
                p.grad = g["grad_full"][o:o + shp.numel()].view(shp)
        u.pending_grads = sum(len(g["params"]) for g in u.groups)
        u.grads_attached = True

    def _before_backward(self, u: _Unit) -> None:
        self._use(u)
        self._attach_grad_buffers(u)

    def _grad_ready(self, u: _Unit) -> None:
        if not u.grads_attached:          # resident unit / params reached without the module pre-hook
            return
        u.pending_grads -= 1
        if u.pending_grads == 0:
            self._reduce_unit(u)
            self._release(u)

    def _reduce_unit(self, u: _Unit) -> None:
        mp = self.hcg.get_model_parallel_group() if self.hcg is not None else None
        if C.group_size(mp) > 1:
            # sequence-parallel replicated parameters (LayerNorm, row-linear bias) hold sequence-partial gradients: sum them over the
            # mp group while they are still attached (after the reduce-scatter ``p.grad`` is None and the engine-level pass skips them)
            sp = [p for g in u.groups for p in g["params"] if getattr(p, "sequence_parallel", False) and p.grad is not None]
            if sp:
                C.fused_allreduce_gradients(sp, mp, scale=1.0)
        for g in u.groups:
            gf = g["grad_full"]
            if gf is None:
                continue
            s = g["total"] // self.world
            if g["key"][2]:                          # expert params: rank-private, no reduction
                piece = gf[self.rank * s:(self.rank + 1) * s]
            elif self.world > 1 and self.group.process_group is not None:
                if self._symm is not None:
                    # in-switch (or peer-pull) reduction of this rank's slice of every rank's unit gradient; the buffer returns to the pool
                    # only after every rank has finished reading it
                    piece = torch.empty(s, dtype=gf.dtype, device=gf.device)
                    sm, ch = self._symm, self._chan()
                    sm.barrier(channel=ch)
                    self._lib.symm_reduce_scatter(sm.mc_ptr(gf) if self.world >= 4 else 0, sm.peer_ptrs(gf), self.rank * s, piece, self.rank,
                                                  {torch.float16: 0, torch.bfloat16: 1, torch.float32: 3}[gf.dtype], 1.0, False, None, torch.cuda.get_device_properties(gf.device).multi_processor_count)
                    sm.barrier(channel=ch)
                    self._pool_give(gf)
                elif gf.is_cuda:
                    piece = torch.empty(s, dtype=gf.dtype, device=gf.device)
                    dist.reduce_scatter_tensor(piece, gf, group=self.group.process_group)
                else:
                    dist.all_reduce(gf, group=self.group.process_group)
                    piece = gf[self.rank * s:(self.rank + 1) * s]
            else:
                piece = gf
            shard = g["shard"]
            if shard.grad is None:
                shard.grad = piece if piece._base is None and piece is not gf else piece.clone()
            else:
                shard.grad.add_(piece)         # flat-optimizer grad view or gradient accumulation
            for p in g["params"]:
                p.grad = None
            g["grad_full"] = None
        u.grads_attached = False

    # ------------------------------------------------------------------ engine-facing API
    @contextlib.contextmanager
    def backward_phase(self):
        """The engine wraps ``loss.backward()`` with this so that recompute re-forwards keep their unit resident and the
        resident unit gets gradient buffers."""
        self._in_backward = True
        for u in self.units:
            if u.resident:
                self._gather(u)
                self._attach_grad_buffers(u)
        try:
            yield
        finally:
            self._in_backward = False
            for u in self.units:
                if u.grads_attached:      # resident unit (or anything the hooks did not finish)
                    self._reduce_unit(u)
                    self._release(u)

    def optimizer_named_parameters(self) -> List[Tuple[str, nn.Parameter]]:
        out = []
        for u in self.units:
            for i, g in enumerate(u.groups):
                kind = "decay" if g["key"][0] else "bias_norm"     # default_decay_fn keys on these substrings
                out.append((f"{u.name}.shard{i}.{'weight' if g['key'][0] else kind}", g["shard"]))
        return out

    def shard_decay_fn(self):
        decay = {id(g["shard"]): g["key"][0] for u in self.units for g in u.groups}
        return lambda name, p: decay.get(id(p), True)

    def after_optimizer_step(self) -> None:
        """The optimizer rewrote the shards: every full copy (the resident unit's included) is stale."""
        self._release_all(force=True)

    def get_all_parameters(self, convert2cpu: bool = False) -> None:
        for u in self.units:
            self._gather(u)

    def release_all_parameters(self) -> None:
        self._release_all(force=False)

    def forward(self, *args, **kwargs):
        out = self._layers(*args, **kwargs)
        if not torch.is_grad_enabled():
            self._release_all(force=False)
        return out

    def state_dict(self, *a, **k):
        self.get_all_parameters()
        sd = {key: v.detach().clone() for key, v in self._layers.state_dict(*a, **k).items()}
        self.release_all_parameters()
        return sd

    def load_state_dict(self, state, strict: bool = True):
        self._release_all(force=True)       # every parameter becomes a view of a freshly gathered flat buffer ...
        self.get_all_parameters()
        res = self._layers.load_state_dict(state, strict)      # ... so the in-place load lands in those buffers
        with torch.no_grad():           # refresh the persistent shards from the loaded full tensors
            for u in self.units:
                for g in u.groups:
                    s = g["total"] // self.world
                    g["shard"].data.copy_(g["full"][self.rank * s:(self.rank + 1) * s])
        self.release_all_parameters()
        return res

    def train(self, mode: bool = True):
        self._layers.train(mode)
        return super().train(mode)

    def __getattr__(self, name):
        try:
            return super().__getattr__(name)
        except AttributeError:
            return getattr(super().__getattr__("_layers"), name)


def group_sharded_parallel(model, optimizer, level: str, scaler=None, group=None, offload: bool = False, dp_group=None, hcg=None, **unused):
    """API-compatible entry (reference eager_engine.py:295-307): level ``os`` / ``os_g`` = stage 1 / 2 (handled by the
    flat optimizer), ``p_g_os`` = stage 3 (this wrapper)."""
    if level == "p_g_os":
        from ..distributed.apis import env

        model = GroupShardedStage3(model, hcg or env.get_hcg(), offload=offload)
    return model, optimizer, scaler
