"""Auto-parallel planner: choose (dp, sharding + ZeRO stage, mp, pp, micro-batch, recompute) for a transformer on N GPUs.

The reference delegates this to Paddle's static-graph auto-parallel engine: the user writes a process mesh, ``auto.shard_tensor``
annotations are propagated through the program and an ``OptimizationTuner`` profiles candidates (core/engine/auto_engine.py:39-209,
models/language_model/gpt/auto/auto_model.py).  In this framework parallelism lives in the layers (``parallel/tp_layers.py``,
``pipeline_parallel.py``, the flat ZeRO optimizer), so "auto" means: *search the layout space with a cost model of those concrete
implementations, keep what fits in 80 GB, rank by predicted step time, and (optionally) measure the top few* — ``AutoEngine`` applies
the winner to the config before anything is built.

Cost model (per optimizer step, one GPU's view).  The hardware constants are NVIDIA's data-sheet figures for the H100 SXM — nominal, not
measured; ``MEASURED_PEAKS.json`` at the repository root, when present, replaces the GEMM peak and the HBM bandwidth by measured ones:

* GEMMs — per-GEMM roofline ``max(flops / peak, bytes / hbm) + launch``: tensor parallelism shrinks N or K, sequence parallelism
  keeps M, so small shards fall off the tensor-core roof by themselves.  ``peak`` = dense bf16 tensor rate.
* attention — causal flash kernels at the tensor rate (an upper bound until they are timed).
* elementwise / norm / optimizer traffic — bytes over HBM bandwidth.
* tensor parallel — 8 collectives per layer per micro-batch of ``tokens x h`` bf16 over NVLink (450 GB/s per direction);
  1.6 wire times are charged as exposed with the fused GEMM+collective kernels and 2.1 with NCCL (assumptions, not H100 measurements).
* pipeline — 1F1B bubble ``(pp - 1) / (m + pp - 1)`` plus the boundary activations.
* data parallel / ZeRO — reduce-scatter + all-gather of the local parameters, overlapped with backward / the next forward; the hidden fraction is taken as 0.9.  Stage 3 adds a
  parameter all-gather per layer per pass.

Memory model: bf16 parameters, gradient buffer, fp32 master + two moments (sharded by ZeRO), activations ``~24 h`` bytes per token
per layer, logits, pipeline in-flight micro-batches, allocator slack.
"""
from __future__ import annotations

import json
import os
from dataclasses import asdict, dataclass, field
from typing import Dict, Iterable, List, Optional

HBM_GB = 80.0
_REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


@dataclass
class Hardware:
    peak_flops: float = 9.89e14          # dense bf16 tensor rate (H100 SXM data sheet, 700 W; nominal)
    hbm_bw: float = 3.35e12              # HBM3 bandwidth (data sheet)
    link_bw: float = 4.5e11              # NVLink 4 per direction (data sheet)
    attn_fwd_flops: float = 9.89e14      # causal flash attention: the tensor rate as an upper bound, not timed on H100
    attn_bwd_flops: float = 9.89e14
    launch_s: float = 4e-6
    mem_gb: float = HBM_GB
    step_efficiency: float = 1.0         # whole-step derating of the kernel times; 1.0 until a step has been profiled on H100

    @staticmethod
    def measured() -> "Hardware":
        hw = Hardware()
        try:
            with open(os.path.join(_REPO, "MEASURED_PEAKS.json")) as f:
                m = json.load(f)
            hw.peak_flops = float(m.get("bf16_tflops_sustained", hw.peak_flops / 1e12)) * 1e12
            hw.hbm_bw = float(m.get("hbm_gbs", hw.hbm_bw / 1e9)) * 1e9
        except (OSError, ValueError):
            pass
        return hw


@dataclass
class ModelShape:
    layers: int
    hidden: int
    heads: int
    vocab: int
    ffn: int
    seq: int
    moe_experts: int = 0                 # experts per MoE layer on one rank (0 = dense)
    kv_heads: int = 0                    # K/V heads (grouped-query attention); 0 = heads
    ffn_activation: str = "gelu"         # gelu | swiglu (FFN1 then has 2 ffn output rows: gate / up pairs)

    @property
    def n_kv_heads(self) -> int:
        return self.kv_heads or self.heads

    @property
    def qkv_width(self) -> float:
        """Output width of the fused QKV projection: (H + 2 Hkv) d."""
        return (self.heads + 2 * self.n_kv_heads) * (self.hidden / self.heads)

    @property
    def ffn1_width(self) -> int:
        """Output width of FFN1: f, or 2 f under SwiGLU."""
        return 2 * self.ffn if self.ffn_activation == "swiglu" else self.ffn

    @property
    def params_per_layer(self) -> float:
        # QKV h (H + 2 Hkv) d, out-proj h^2, FFN h (f1 + f) with f1 = ffn1_width; biases (H + 2 Hkv) d + h + h + f1, two norms 4 h
        return (self.hidden * self.qkv_width + self.hidden * self.hidden + self.hidden * (self.ffn1_width + self.ffn) + self.qkv_width + 6 * self.hidden
                + self.ffn1_width)

    @property
    def params(self) -> float:
        return self.layers * self.params_per_layer + (self.vocab + self.seq) * self.hidden

    @staticmethod
    def from_config(cfg) -> "ModelShape":
        m = cfg.Model
        h = int(m.get("hidden_size", 768))
        seq = 1024
        try:
            seq = int(cfg.Data.Train.dataset.get("max_seq_len", seq))
        except (AttributeError, KeyError):
            pass
        return ModelShape(layers=int(m.get("num_layers", m.get("num_hidden_layers", 12))), hidden=h, heads=int(m.get("num_attention_heads", 12)),
                          vocab=int(m.get("vocab_size", 50304)), ffn=int(m.get("ffn_hidden_size", 4 * h) or 4 * h), seq=seq,
                          kv_heads=int(m.get("num_key_value_heads") or 0), ffn_activation=str(m.get("ffn_activation") or "gelu"))


@dataclass
class Plan:
    dp: int
    sharding: int
    stage: int
    mp: int
    pp: int
    micro_batch: int
    accumulate: int
    recompute: str                       # none | core_attn | full_attn | full
    sequence_parallel: bool
    fused_tp: bool
    cp: int = 1                          # context parallelism: cp of the (dp x sharding) data ranks share a batch and split its sequence
    cp_mode: str = "ulysses"             # ulysses: all-to-all around attention (cp divides the local heads); ring: K / V blocks on a ring, any cp
    est_step_s: float = 0.0
    est_mem_gb: float = 0.0
    tokens_per_s: float = 0.0
    breakdown: Dict[str, float] = field(default_factory=dict)
    measured_step_s: Optional[float] = None

    def overrides(self) -> List[str]:
        ov = [f"Distributed.dp_degree={self.dp}", f"Distributed.mp_degree={self.mp}", f"Distributed.pp_degree={self.pp}",
              f"Distributed.sharding.sharding_degree={self.sharding}", f"Distributed.sharding.sharding_stage={self.stage}",
              f"Global.micro_batch_size={self.micro_batch}", f"Model.use_recompute={self.recompute != 'none'}",
              f"Model.sequence_parallel={self.sequence_parallel}", f"Distributed.cp_degree={self.cp}"]
        if self.cp > 1:
            ov.append(f"Distributed.cp_mode={self.cp_mode}")
        if self.recompute != "none":
            ov.append(f"Model.recompute_granularity={self.recompute}")
        return ov

    def describe(self) -> str:
        return (f"dp{self.dp} x sharding{self.sharding}(stage {self.stage}){f' [cp{self.cp} {self.cp_mode}]' if self.cp > 1 else ''} x mp{self.mp}{'+sp' if self.sequence_parallel else ''} x pp{self.pp}, "
                f"micro {self.micro_batch} x {self.accumulate}, recompute {self.recompute}: {self.est_step_s * 1e3:.1f} ms/step, "
                f"{self.est_mem_gb:.0f} GB, {self.tokens_per_s:,.0f} tok/s")


def _gemm_time(hw: Hardware, m: float, n: float, k: float) -> float:
    flops = 2.0 * m * n * k
    bytes_ = 2.0 * (m * k + n * k + m * n)
    return max(flops / hw.peak_flops, bytes_ / hw.hbm_bw) + hw.launch_s


def _layer_time(hw: Hardware, s: ModelShape, tokens: float, mp: int, sp: bool, recompute: str) -> Dict[str, float]:
    """Forward + backward of one transformer layer for ``tokens`` tokens on one GPU of an ``mp``-way tensor-parallel group."""
    h, f = s.hidden, s.ffn
    fwd_gemm = (_gemm_time(hw, tokens, s.qkv_width / mp, h) + _gemm_time(hw, tokens, h, h / mp)
                + _gemm_time(hw, tokens, s.ffn1_width / mp, h) + _gemm_time(hw, tokens, h, f / mp))
    gemm = 3.0 * fwd_gemm                                        # dgrad + wgrad have the forward's shapes
    attn_flops = 2.0 * 2.0 * tokens * s.seq * h / mp / 2.0       # causal: half of QK^T and PV
    attn_fwd, attn_bwd = attn_flops / hw.attn_fwd_flops, 2.5 * attn_flops / hw.attn_bwd_flops
    # elementwise / norm / bias-grad traffic: the per-kernel table of the 6.7B trace (norm fwd + bwd, bias-dropout-residual fwd + bwd, bias
    # column sums, residual adds: ~0.6 ms per layer at 8192 tokens) is ~120 h bytes per token
    tok_local = tokens / (mp if sp else 1)
    elem = 120.0 * h * tok_local / hw.hbm_bw
    extra = {"none": 0.0, "core_attn": attn_fwd, "full_attn": attn_fwd + _gemm_time(hw, tokens, s.qkv_width / mp, h) + _gemm_time(hw, tokens, h, h / mp),
             "full": fwd_gemm + attn_fwd + elem / 3.0}[recompute]
    return {"gemm": gemm, "attn": attn_fwd + attn_bwd, "elementwise": elem, "recompute": extra}


def estimate(s: ModelShape, hw: Hardware, world: int, local_batch: int, plan: Plan) -> Plan:
    """Fill in the predicted step time, memory and throughput of ``plan`` (``local_batch`` = sequences per data-parallel rank per step)."""
    mp, pp, sd, dp, stage = plan.mp, plan.pp, plan.sharding, plan.dp, plan.stage
    data_ranks = dp * sd
    cp = max(int(plan.cp), 1)
    mb = plan.micro_batch
    n_micro = max(local_batch // mb, 1)
    tokens = float(mb * s.seq) / cp                      # a context-parallel rank holds 1 / cp of every sequence
    layers_local = s.layers / pp
    lt = _layer_time(hw, s, tokens, mp, plan.sequence_parallel, plan.recompute)
    per_micro = layers_local * sum(lt.values()) / hw.step_efficiency
    head = 3.0 * _gemm_time(hw, tokens, s.vocab / mp, s.hidden) + 10.0 * tokens * s.vocab / mp / hw.hbm_bw     # LM head + fused CE (last stage)
    per_micro += head / pp
    # tensor-parallel collectives: 4 forward + 4 backward per layer, (mp - 1) / mp of tokens x h bf16 each
    tp = 0.0
    if mp > 1:
        vol = 8.0 * layers_local * tokens * s.hidden * 2.0 * (mp - 1) / mp
        # exposed wire times per collective are assumptions (the full backward re-gathers and runs two smaller GEMMs per collective); not timed on H100
        tp = vol / hw.link_bw * (1.6 if plan.fused_tp else 2.1) + (0 if plan.fused_tp else 8.0 * layers_local * 12e-6)
    if cp > 1 and plan.cp_mode == "ring":
        # ring: (cp - 1) hops per layer of K and V forward (bf16), K / V again plus the fp32 dK / dV accumulators backward = 16 bytes per
        # token x h / mp per hop; each hop is posted before the block it overlaps, so only what the attention math cannot cover is exposed
        wire = 16.0 * (cp - 1) * tokens * s.hidden / mp / hw.link_bw
        tp += layers_local * (max(0.0, wire - lt["attn"]) + 3.0 * (cp - 1) * 12e-6)
    elif cp > 1:      # Ulysses: 4 all-to-alls per layer forward (q, k, v, out) and 4 backward, each moving (cp - 1) / cp of tokens x h / mp bf16
        tp += 8.0 * layers_local * tokens * s.hidden / mp * 2.0 * (cp - 1) / cp / hw.link_bw + 8.0 * layers_local * 12e-6
    pipe_p2p = 0.0 if pp == 1 else 2.0 * tokens * s.hidden * 2.0 / (mp if plan.sequence_parallel else 1) / hw.link_bw + 4 * 15e-6
    if pp > 1:
        per_micro *= 1.15            # blocking stage-to-stage transfers and ~7 k launches per step at micro-batch granularity (c15_bench_n8.json, named_layout)
    compute = n_micro * (per_micro + tp + pipe_p2p)
    bubble = compute * (pp - 1) / max(n_micro, 1) if pp > 1 else 0.0
    # gradient reduce-scatter + parameter all-gather of this rank's parameters over the data ranks (bf16 both ways)
    p_local = s.params / (mp * pp)
    dp_comm = 0.0
    if data_ranks > 1:
        dp_comm = 2.0 * p_local * 2.0 * (data_ranks - 1) / data_ranks / hw.link_bw
        if stage == 3:
            dp_comm += 2.0 * n_micro * p_local * 2.0 * (sd - 1) / sd / hw.link_bw     # per-layer gathers in forward and backward
    # 10 % of the exchange is exposed outright (first / last bucket); the hidden 90 % still costs about half its duration because the
    # collective kernels take SMs and HBM bandwidth from the GEMMs they run beside (an assumption, not timed on H100)
    exposed_dp = (0.1 + 0.5) * dp_comm + (0.0 if data_ranks == 1 else 1.5e-3)
    # AdamW over the local shard: 2 (bf16 w) + 4 (grad) + 12 (master, m, v read) + 12 (write) bytes per parameter; overlapped with the next forward
    opt = p_local / (sd if stage >= 1 else 1) * 30.0 / hw.hbm_bw
    exposed_opt = 0.6 * opt            # "overlapped" still costs: the forward GEMMs it runs beside slow down
    step = compute + bubble + exposed_dp + exposed_opt
    # ---- memory
    shard = sd if stage >= 1 else 1
    mem = p_local * 2.0 / (sd if stage == 3 else 1)                      # bf16 parameters
    mem += p_local * 4.0 / (sd if stage >= 2 else 1)                      # fp32 gradient buffer (main_grad)
    mem += p_local * 12.0 / shard                                          # master + m + v
    act_tok = {"none": 24.0, "core_attn": 20.0, "full_attn": 14.0, "full": 2.0}[plan.recompute] * s.hidden / (mp if plan.sequence_parallel else 1)
    if not plan.sequence_parallel and mp > 1:
        act_tok = act_tok * 0.55 + act_tok * 0.45 / mp                    # without SP only the GEMM-side activations shrink
    in_flight = min(pp, n_micro) if pp > 1 else 1
    mem += act_tok * tokens * layers_local * in_flight
    if plan.recompute == "full":
        mem += 24.0 * s.hidden * tokens / mp                               # one layer being recomputed
    mem += tokens * s.vocab / mp * 6.0 / (pp if pp > 1 else 1)             # bf16 logits + fp32 softmax workspace (last stage; amortised over stages)
    mem = mem * 1.06 + 2.5e9                                               # allocator slack, CUDA context, NCCL / symmetric buffers
    plan.est_step_s, plan.est_mem_gb = step, mem / 2 ** 30
    plan.tokens_per_s = local_batch * (data_ranks // cp) * s.seq / step
    plan.breakdown = {"compute": n_micro * per_micro, "tp_comm": n_micro * tp, "pipeline_bubble": bubble + n_micro * pipe_p2p,
                      "exposed_dp_comm": exposed_dp, "exposed_optimizer": exposed_opt}
    return plan


def _divisors(n: int) -> List[int]:
    return [d for d in range(1, n + 1) if n % d == 0]


def enumerate_plans(s: ModelShape, world: int, local_batch: int, stages: Iterable[int] = (1, 2, 3), allow_pp: bool = True) -> List[Plan]:
    """Every (mp, pp, sharding, dp, stage, micro-batch, recompute) combination the parallel layers support for this model and world size.
    ``local_batch`` is the per-GPU batch: a data rank of an (mp, pp) layout carries ``local_batch * mp * pp`` sequences."""
    out = []
    for mp in _divisors(world):
        if s.heads % mp or s.n_kv_heads % mp or s.hidden % mp or s.vocab % mp or mp > 8:
            continue
        for pp in _divisors(world // mp):
            if s.layers % pp or (pp > 1 and not allow_pp):
                continue
            rest = world // (mp * pp)
            rank_batch = local_batch * mp * pp
            for sd in _divisors(rest):
                dp = rest // sd
                for stage in (stages if sd > 1 else (1,)):
                    if stage == 3 and pp > 1:
                        continue                                           # the stage-3 wrapper and the pipeline schedule are not combined
                    cps = [(1, "ulysses")]                                 # context parallelism only where long sequences make activations the problem
                    for c in _divisors(rest):
                        if c > 1 and pp == 1 and s.seq >= 4096 and s.n_kv_heads == s.heads:   # (cp also runs under the pipeline schedule; not searched: RoPE models cannot use it; nor can grouped K/V heads)
                            if (s.heads // mp) % c == 0 and s.seq % c == 0:
                                cps.append((c, "ulysses"))
                            if s.seq % (2 * c) == 0:                       # zigzag shards: two chunks per rank
                                cps.append((c, "ring"))
                    for c, cmode in cps:
                        group_batch = rank_batch * c                       # the c ranks of a group pool their share of the global batch
                        for mb in _divisors(group_batch):
                            n_micro = group_batch // mb
                            if pp > 1 and n_micro < pp:
                                continue
                            for rc in ("none", "core_attn", "full"):
                                out.append(Plan(dp=dp, sharding=sd, stage=stage, mp=mp, pp=pp, micro_batch=mb, accumulate=n_micro, recompute=rc,
                                                sequence_parallel=mp > 1, fused_tp=mp > 1, cp=c, cp_mode=cmode))
    return out


def plan_layouts(s: ModelShape, world: int, local_batch: int, hw: Optional[Hardware] = None, mem_limit_gb: Optional[float] = None,
                 top: int = 0, **kw) -> List[Plan]:
    """Every feasible plan, fastest first.  ``local_batch`` is the per-GPU batch at pure data parallelism: a data rank of an
    (mp, pp) layout carries ``local_batch * mp * pp`` sequences, so every candidate processes the same global batch."""
    hw = hw or Hardware.measured()
    limit = mem_limit_gb if mem_limit_gb is not None else 0.92 * hw.mem_gb
    plans = []
    for p in enumerate_plans(s, world, local_batch, **kw):
        estimate(s, hw, world, local_batch * p.mp * p.pp * p.cp, p)
        if p.est_mem_gb <= limit:
            plans.append(p)
    plans.sort(key=lambda p: (p.est_step_s, p.est_mem_gb))
    seen, uniq = set(), []
    for p in plans:                                                       # one entry per layout: its best micro-batch / recompute
        key = (p.dp, p.sharding, p.stage, p.mp, p.pp, p.cp, p.cp_mode if p.cp > 1 else "")
        if key not in seen:
            seen.add(key)
            uniq.append(p)
    return uniq[:top] if top else uniq


def rank_layouts(cfg, world: Optional[int] = None, top: int = 0) -> List[Dict]:
    """Config-level entry (``AutoEngine.tune`` / ``tools/auto.py --plan``): dict rows, fastest first."""
    from .config import world_size_hint

    s = ModelShape.from_config(cfg)
    world = world or world_size_hint()
    lb = int(cfg.Global.get("local_batch_size") or cfg.Global.get("micro_batch_size") or 1)
    d = cfg.get("Distributed", {}) or {}
    cur = int(d.get("mp_degree", 1) or 1) * int(d.get("pp_degree", 1) or 1)
    lb = max(lb // max(cur, 1), 1)                                        # back to the per-GPU batch the config implies
    rows = []
    for p in plan_layouts(s, world, lb, top=top):
        r = asdict(p)
        r["describe"] = p.describe()
        rows.append(r)
    return rows


def best_plan(cfg, world: Optional[int] = None) -> Optional[Plan]:
    from .config import world_size_hint

    s = ModelShape.from_config(cfg)
    world = world or world_size_hint()
    lb = int(cfg.Global.get("local_batch_size") or cfg.Global.get("micro_batch_size") or 1)
    plans = plan_layouts(s, world, lb, top=1)
    return plans[0] if plans else None


def explain(plans: List[Plan], k: int = 8) -> str:
    lines = [f"{'#':>2}  layout"]
    for i, p in enumerate(plans[:k]):
        b = ", ".join(f"{n} {v * 1e3:.1f}" for n, v in p.breakdown.items())
        lines.append(f"{i:>2}  {p.describe()}   [{b} ms]")
    return "\n".join(lines)


if __name__ == "__main__":      # python -m paddlefleetx_b200.utils.layout_planner 6.7b 8
    import sys

    presets = {"345m": (24, 1024, 16), "1.3b": (24, 2048, 16), "6.7b": (32, 4096, 32), "13b": (40, 5120, 40), "175b": (96, 12288, 96)}
    name, world = (sys.argv[1] if len(sys.argv) > 1 else "6.7b"), int(sys.argv[2]) if len(sys.argv) > 2 else 8
    L, h, a = presets[name]
    shape = ModelShape(layers=L, hidden=h, heads=a, vocab=50304, ffn=4 * h, seq=int(sys.argv[3]) if len(sys.argv) > 3 else 1024)
    print(f"GPT {name}: {shape.params / 1e9:.2f} B parameters, {world} GPUs, 8 sequences / GPU")
    print(explain(plan_layouts(shape, world, 8), 12))
