"""``MoELayer`` — FastMoE-style expert-parallel FFN (reference moe/moe_layer.py:33-235).

    reshape -> [mp slice] -> gate -> count_by_gate -> MoEScatter (all-to-all to expert owners) -> local experts ->
    MoEGather (all-to-all back) -> gate-weighted combine -> [mp all-gather]

``num_experts`` is the number of experts PER RANK; the expert-parallel world is the ``moe`` = dp x mp group.  The
reference's latent attribute bug (``self.num_experts`` vs ``self.num_expert``, SURVEY F8) is not reproduced.
With ``fused_p2p`` the dispatch/combine run as peer-memory kernels (``fused_dispatch.py``) and the local experts as GROUPED tcgen05
GEMMs driven by the device-side segment table (``grouped_experts.py``): the layer never synchronises with the host.  The NCCL path
keeps the reference's structure (all-to-all + a loop of GEMMs over contiguous row ranges).
"""
from __future__ import annotations

import math
from typing import List, Optional

import torch
import torch.nn as nn

from ....ops import functional as OF
from ....parallel import comm_ops as C
from ....parallel.recompute import recompute
from .comm_ops import AllGather, MoEGather, MoEScatter, Slice
from .gate import BaseGate, GShardGate, NaiveGate, SwitchGate
from .utils import count_by_gate


class ExpertLayer(nn.Module):
    """h -> 4h -> GELU(tanh) -> h, or with ``activation="swiglu"`` the gated FFN of width ``d_hidden`` = F: ``htoh4`` is [2F, h] with
    pair-interleaved rows (2i the gate channel i, 2i + 1 its up channel, as the dense GPT's ``linear1``) and ``h4toh`` is [h, F], so the
    checkpoint keys stay those of a GELU expert.  Parameters are tagged ``is_expert`` (excluded from dp/mp broadcast, clipped with the
    expert-group norm) — the reference tags by renaming params with an ``expert_`` prefix (single_model.py:71-74)."""

    def __init__(self, d_model: int, d_hidden: int, init_std: float = 0.02, out_std: Optional[float] = None, dtype=None, device=None,
                 activation: str = "gelu"):
        super().__init__()
        if activation not in ("gelu", "swiglu"):
            raise ValueError(f"ExpertLayer activation must be gelu or swiglu, got {activation!r}")
        self.activation = activation
        self.htoh4 = nn.Linear(d_model, 2 * d_hidden if activation == "swiglu" else d_hidden, dtype=dtype, device=device)
        self.h4toh = nn.Linear(d_hidden, d_model, dtype=dtype, device=device)
        with torch.no_grad():
            self.htoh4.weight.normal_(0.0, init_std); self.htoh4.bias.zero_()
            self.h4toh.weight.normal_(0.0, out_std or init_std); self.h4toh.bias.zero_()
        for p in self.parameters():
            p.is_expert = True
            p.no_sync = True

    def forward(self, x):
        if self.activation == "swiglu":
            return OF.linear(OF.bias_swiglu(OF.linear(x, self.htoh4.weight), self.htoh4.bias), self.h4toh.weight, self.h4toh.bias)
        return OF.fused_ffn(x, self.htoh4.weight, self.htoh4.bias, self.h4toh.weight, self.h4toh.bias)


class MoELayer(nn.Module):
    _instances = 0

    def __init__(self, d_model: int, experts: List[nn.Module], gate=None, moe_group=None, mp_group=None, recompute_interval: int = 0,
                 recompute_ctx=None, top_k: int = 2, dtype=None, device=None, fused_p2p: bool = False, capacity_factor: float = 2.0,
                 grouped_gemm: bool = True):
        super().__init__()
        self.fused_p2p = fused_p2p              # peer-memory dispatch/combine kernels (fused_dispatch.py) instead of NCCL all-to-all
        self.capacity_factor = capacity_factor
        MoELayer._instances += 1
        self._layer_key = MoELayer._instances
        self.d_model = d_model
        self.experts = nn.ModuleList(experts)
        self.num_expert = len(experts)
        # With the peer-memory dispatch the experts run as grouped tcgen05 GEMMs over the device-side segment table (grouped_experts.py):
        # their parameters move into four stacked tensors; checkpoints keep the per-expert names through the two hooks below.
        self.grouped = None
        if fused_p2p and grouped_gemm:
            from .grouped_experts import GroupedExperts

            if GroupedExperts.supported(experts):
                self.grouped = GroupedExperts(experts)
                self._register_state_dict_hook(MoELayer._split_expert_state)
                self._register_load_state_dict_pre_hook(self._merge_expert_state)
        self.group = moe_group
        self.world_size = C.group_size(moe_group)
        self.mp_group = mp_group
        self.recompute_interval = recompute_interval
        gate = gate or {"type": "gshard", "top_k": 2}
        if isinstance(gate, dict):
            self.top_k = gate.get("top_k", top_k)
            kind = gate.get("type", "gshard")
            kw = dict(group=moe_group, dtype=dtype, device=device)
            if kind in ("naive", None):
                gate = NaiveGate(d_model, self.num_expert, topk=self.top_k, **kw)
            elif kind == "gshard":
                gate = GShardGate(d_model, self.num_expert, topk=self.top_k, **kw)
            elif kind == "switch":
                gate = SwitchGate(d_model, self.num_expert, topk=self.top_k, **kw)
            else:
                raise ValueError(f"unknown gate type {kind}; expected naive | gshard | switch")
        elif isinstance(gate, NaiveGate):
            self.top_k = gate.top_k
        else:
            raise TypeError("gate must be a dict or a NaiveGate instance")
        self.gate = gate

    @staticmethod
    def _split_expert_state(module, state_dict, prefix, local_metadata):
        module.grouped.split_state(state_dict, prefix + "grouped.", prefix + "experts.")

    def _merge_expert_state(self, state_dict, prefix, *args):
        self.grouped.merge_state(state_dict, prefix + "grouped.", prefix + "experts.")

    def _experts_forward(self, x: torch.Tensor, counts: List[int]) -> torch.Tensor:
        outs, start = [], 0
        for e, n in enumerate(counts):
            if n:
                outs.append(self.experts[e](x[start:start + n]))
            start += n
        if not outs:
            return x.new_zeros(0, self.d_model) + sum(p.sum() * 0 for p in self.experts.parameters())
        return torch.cat(outs, 0)

    def _experts_forward_segments(self, xs: torch.Tensor, starts: List[int], counts: List[int], total: int) -> torch.Tensor:
        """Expert-major rows with every expert's block padded to the dispatch alignment (pad rows are zero)."""
        outs = []
        for e in range(self.num_expert):
            end = starts[e + 1] if e + 1 < self.num_expert else total
            if end > starts[e]:
                outs.append(self.experts[e](xs[starts[e]:end]))
        if not outs:
            return xs.new_zeros(0, self.d_model) + sum(p.sum() * 0 for p in self.experts.parameters())
        return torch.cat(outs, 0)

    def _forward_p2p(self, x: torch.Tensor, value: torch.Tensor, gate_idx: torch.Tensor) -> torch.Tensor:
        from .fused_dispatch import FusedCombine, FusedDispatch, get_dispatcher, make_plan

        disp = get_dispatcher(self.group, self.d_model, self.num_expert, x.dtype, self.capacity_factor)
        if gate_idx.dim() == 1:
            gate_idx = gate_idx.unsqueeze(1)
        plan = make_plan(disp, gate_idx, x.shape[0])
        layer_key = self._layer_key if (self.training and torch.is_grad_enabled()) else None
        ge = self.grouped
        if ge is not None and OF.tensor_core_dtype(x, ge.w1, ge.b1, ge.w2, ge.b2):
            # sync-free: dispatch -> tile table -> 2 grouped GEMMs -> combine, all sized by the fixed capacity; the host never reads a count
            from .fused_dispatch import ALIGN
            from .grouped_experts import grouped_ffn

            xs, _ = FusedDispatch.apply(x, plan, layer_key, True)
            ys = grouped_ffn(xs, plan.tile_group, plan.seg2, self.grouped, disp, ALIGN, recompute_h=self.recompute_interval > 0 and self.training)
            disp.poll_overflow()
            return FusedCombine.apply(ys, value.reshape(x.shape[0], -1), plan)
        if self.grouped is not None:
            self.grouped.bind_views()
        xs, seg = FusedDispatch.apply(x, plan, layer_key, False)
        starts, counts, total = seg[:self.num_expert], seg[self.num_expert:2 * self.num_expert], seg[2 * self.num_expert]
        if self.recompute_interval > 0 and self.training and xs.requires_grad:
            ys = recompute(self._experts_forward_segments, xs, starts, counts, total)
        else:
            ys = self._experts_forward_segments(xs, starts, counts, total)
        return FusedCombine.apply(ys, value.reshape(x.shape[0], -1), plan)

    def forward(self, inp: torch.Tensor) -> torch.Tensor:
        origin_shape = inp.shape
        x = inp.reshape(-1, origin_shape[-1])
        mp_world = C.group_size(self.mp_group)
        if mp_world > 1:
            x = Slice.apply(x, self.mp_group.rank, mp_world, self.mp_group)
        value, gate_idx = self.gate(x)
        if self.fused_p2p and x.is_cuda and (self.world_size > 1 or self.grouped is not None):
            out = self._forward_p2p(x, value, gate_idx)
            if mp_world > 1:
                out = AllGather.apply(out, self.mp_group.rank, mp_world, self.mp_group)
            return out.reshape(origin_shape)
        if self.grouped is not None:
            self.grouped.bind_views()
        pos, lec, gec = count_by_gate(gate_idx, self.num_expert, self.world_size, group=self.group)
        fwd_counts = gec.view(self.world_size, self.num_expert).sum(0)
        counts = fwd_counts.tolist()                       # host sync #1 (sizes the expert loop); the P2P path avoids it
        fwd_batch = int(sum(counts))
        topk = gate_idx.shape[1] if gate_idx.dim() > 1 else 1
        xs = MoEScatter.apply(x, pos, lec, gec, fwd_batch, self.world_size, self.group, topk)
        if self.recompute_interval > 0 and self.training and xs.requires_grad:
            ys = recompute(self._experts_forward, xs, counts)
        else:
            ys = self._experts_forward(xs, counts)
        out_batch = x.shape[0] * topk
        ys = MoEGather.apply(ys, pos, lec, gec, out_batch, self.world_size, self.group)
        ys = ys.view(-1, topk, self.d_model)
        w = value.reshape(x.shape[0], 1, topk).to(ys.dtype)
        out = torch.bmm(w, ys).reshape(-1, self.d_model)
        if mp_world > 1:
            out = AllGather.apply(out, self.mp_group.rank, mp_world, self.mp_group)
        return out.reshape(origin_shape)


def build_moe_layer(hidden: int, ffn_hidden: int, moe_configs: dict, num_layers: int, init_std: float, mp_group, dtype, device,
                    layer_idx: int = 0, ffn_activation: str = "gelu") -> MoELayer:
    from ....distributed.apis import env

    hcg = env.get_hcg()
    moe_group = hcg.get_moe_group() if env.world_size() > 1 else None
    n = int(moe_configs.get("num_experts", 1))
    out_std = init_std / math.sqrt(2.0 * num_layers)
    experts = [ExpertLayer(hidden, ffn_hidden, init_std, out_std, dtype, device, ffn_activation) for _ in range(n)]
    gate_cfg = {"type": moe_configs.get("gate", "gshard"), "top_k": int(moe_configs.get("top_k", 2))}
    return MoELayer(hidden, experts, gate=gate_cfg, moe_group=moe_group, mp_group=mp_group if C.group_size(mp_group) > 1 else None,
                    recompute_interval=int(moe_configs.get("recompute_interval", 0)), dtype=dtype, device=device,
                    fused_p2p=bool(moe_configs.get("fused_p2p", False)), capacity_factor=float(moe_configs.get("p2p_capacity_factor", 2.0)),
                    grouped_gemm=bool(moe_configs.get("grouped_gemm", True)))
