"""Megatron-style tensor-parallel layers + their sequence-parallel variants.

What the reference gets from ``paddle.distributed.fleet.meta_parallel`` (contracts in SURVEY §2.5, call sites
gpt/dygraph/hybrid_model.py:139-196,589-605,699-704,951-952) and from its in-tree
``sequence_parallel_utils.py:215-398``:

    ColumnParallelLinear       W[out/n, in]   identity fwd / all-reduce bwd on the input
    RowParallelLinear          W[out, in/n]   GEMM -> all-reduce -> + bias
    ColumnSequenceParallelLinear  all-gather(seq) -> GEMM      (bwd: reduce-scatter)
    RowSequenceParallelLinear     GEMM -> reduce-scatter(seq)  (bwd: all-gather), then + bias
    VocabParallelEmbedding     vocab-sharded lookup + all-reduce
    ParallelCrossEntropy       vocab-parallel softmax-CE

Weights are stored ``[out, in]`` (torch convention, K-major for the wgmma GEMM).  ``mp_group=None`` or a
size-1 group degenerates every layer to its plain single-GPU form, so the same model code serves 1..N GPUs.
With ``Fused.tp_comm`` enabled on NVSwitch boxes the SP linears run the fused GEMM+collective kernels of
``parallel/fused_tp.py`` instead of NCCL + GEMM.
"""
from __future__ import annotations


import torch
import torch.nn as nn

from ..ops import functional as OF
from . import comm_ops as C


# process-wide defaults taken from the YAML ``Fused`` section (``configure`` is called by the task modules before the model is
# built): ``tp_comm`` = fused all-gather->GEMM / GEMM->reduce-scatter kernels in the SP linears, ``fp8_tp_gemm`` = forward GEMMs of
# the tensor-parallel linears in fp8-e4m3, backward in bf16; ``fp8_recipe`` = "mx" (default: OCP MX block scaling, one E8M0 scale per 32
# K-elements folded in by the GEMM's consumer threads) or "rowwise" (per-token x per-channel fp32 scales in the epilogue)
_OPTIONS = {"tp_comm": False, "fp8_tp_gemm": False, "fp8_recipe": "mx"}


def configure(fused_cfg=None) -> dict:
    fused_cfg = fused_cfg or {}
    _OPTIONS["tp_comm"] = bool(fused_cfg.get("tp_comm", False))
    _OPTIONS["fp8_tp_gemm"] = bool(fused_cfg.get("fp8_tp_gemm", False))
    recipe = str(fused_cfg.get("fp8_recipe", "mx")).lower()
    if recipe not in ("mx", "rowwise"):
        raise ValueError(f"Fused.fp8_recipe must be 'mx' or 'rowwise', got {recipe!r}")
    _OPTIONS["fp8_recipe"] = recipe
    return dict(_OPTIONS)


def _tp_linear(x: torch.Tensor, weight, bias, owner=None) -> torch.Tensor:
    int8 = getattr(owner, "int8", None) if owner is not None else None
    if int8 is not None:                  # serving: W8A8 (weights replaced by ops.quant.quantize_tp_linears_int8)
        y = int8(x)
        return y if bias is None else y + bias
    if _OPTIONS["fp8_tp_gemm"] and x.is_cuda:
        from ..ops.quant import fp8_linear

        return fp8_linear(x, weight, bias, recipe=_OPTIONS["fp8_recipe"])
    return OF.linear(x, weight, bias)


def _mark(p: nn.Parameter, **attrs) -> nn.Parameter:
    for k, v in attrs.items():
        setattr(p, k, v)
    return p


def _init_normal_sharded(weight: torch.Tensor, std: float, full_shape, shard_dim: int, group) -> None:
    """Every TP rank draws its slice from its OWN stream: the tracker's ``local_seed`` (which ``env.set_seed`` derives from the mp
    rank — the reference creates these weights inside the model-parallel RNG tracker, hybrid_model.py:139-196), or, when no tracker
    stream is registered, a generator forked from the default seed by mp rank.  Drawing from the default generator would hand every
    mp rank bit-identical shards (``global_seed`` does not depend on the mp rank and the initial broadcast skips TP-sharded tensors),
    i.e. mp-fold duplicated neurons.  Layouts are equivalent in distribution, not bitwise."""
    from .rng import get_rng_state_tracker

    with torch.no_grad():
        if C.group_size(group) == 1:
            weight.normal_(mean=0.0, std=std)
            return
        tracker = get_rng_state_tracker()
        if tracker.has("local_seed"):
            with tracker.rng_state("local_seed"):
                weight.normal_(mean=0.0, std=std)
        else:
            gen = torch.Generator(device=weight.device)
            gen.manual_seed((torch.initial_seed() + 7919 * (C.group_rank(group) + 1)) & 0x7FFFFFFFFFFFFFFF)
            weight.normal_(mean=0.0, std=std, generator=gen)


class ColumnParallelLinear(nn.Module):
    def __init__(self, in_features: int, out_features: int, mp_group=None, has_bias: bool = True, gather_output: bool = True,
                 init_std: float = 0.02, fuse_matmul_bias: bool = False, dtype=None, device=None):
        super().__init__()
        self.group = mp_group
        self.world = C.group_size(mp_group)
        assert out_features % self.world == 0, f"out_features {out_features} % mp {self.world}"
        self.in_features, self.out_features = in_features, out_features
        self.out_per_rank = out_features // self.world
        self.gather_output = gather_output
        self.weight = nn.Parameter(torch.empty(self.out_per_rank, in_features, dtype=dtype, device=device))
        _init_normal_sharded(self.weight, init_std, (out_features, in_features), 0, mp_group)
        _mark(self.weight, tp_sharded=self.world > 1, split_axis=0)
        if has_bias:
            self.bias = nn.Parameter(torch.zeros(self.out_per_rank, dtype=dtype, device=device))
            _mark(self.bias, tp_sharded=self.world > 1, split_axis=0)
        else:
            self.register_parameter("bias", None)

    def forward(self, x: torch.Tensor, skip_bias: bool = False) -> torch.Tensor:
        x = C.copy_to_group(x, self.group)
        y = _tp_linear(x, self.weight, None if skip_bias else self.bias, self)
        return C.gather_last_dim(y, self.group) if self.gather_output else y


class RowParallelLinear(nn.Module):
    def __init__(self, in_features: int, out_features: int, mp_group=None, has_bias: bool = True, input_is_parallel: bool = False,
                 init_std: float = 0.02, fuse_matmul_bias: bool = False, dtype=None, device=None, skip_bias_add: bool = False):
        super().__init__()
        self.group = mp_group
        self.world = C.group_size(mp_group)
        assert in_features % self.world == 0
        self.in_features, self.out_features = in_features, out_features
        self.in_per_rank = in_features // self.world
        self.input_is_parallel = input_is_parallel
        self.skip_bias_add = skip_bias_add
        self.weight = nn.Parameter(torch.empty(out_features, self.in_per_rank, dtype=dtype, device=device))
        _init_normal_sharded(self.weight, init_std, (out_features, in_features), 1, mp_group)
        _mark(self.weight, tp_sharded=self.world > 1, split_axis=1)
        if has_bias:
            self.bias = nn.Parameter(torch.zeros(out_features, dtype=dtype, device=device))
        else:
            self.register_parameter("bias", None)

    def forward(self, x: torch.Tensor):
        if not self.input_is_parallel:
            x = C.scatter_last_dim(x, self.group)
        if self.world == 1:
            if self.skip_bias_add:
                return _tp_linear(x, self.weight, None, self), self.bias
            return _tp_linear(x, self.weight, self.bias, self)
        y = C.reduce_from_group(_tp_linear(x, self.weight, None, self), self.group)
        if self.skip_bias_add:
            return y, self.bias
        return y if self.bias is None else y + self.bias


class ColumnSequenceParallelLinear(nn.Module):
    """input ``[s/n, b, h]`` -> all-gather along s -> GEMM -> ``[s, b, out/n]``."""

    def __init__(self, in_features: int, out_features: int, mp_group=None, has_bias: bool = True, gather_output: bool = False,
                 init_std: float = 0.02, dtype=None, device=None, fused_comm: bool = False):
        super().__init__()
        assert not gather_output, "sequence-parallel column linear never gathers its output"
        self.group = mp_group
        self.world = C.group_size(mp_group)
        self.out_per_rank = out_features // self.world
        self.fused_comm = fused_comm
        self.weight = nn.Parameter(torch.empty(self.out_per_rank, in_features, dtype=dtype, device=device))
        _init_normal_sharded(self.weight, init_std, (out_features, in_features), 0, mp_group)
        _mark(self.weight, tp_sharded=self.world > 1, split_axis=0)
        if has_bias:
            self.bias = nn.Parameter(torch.zeros(self.out_per_rank, dtype=dtype, device=device))
            _mark(self.bias, tp_sharded=self.world > 1, split_axis=0)
        else:
            self.register_parameter("bias", None)

    def forward(self, x: torch.Tensor, skip_bias: bool = False) -> torch.Tensor:
        bias = None if skip_bias else self.bias
        if (self.fused_comm or _OPTIONS["tp_comm"]) and x.is_cuda and self.world > 1:
            from .fused_tp import all_gather_linear

            return all_gather_linear(x, self.weight, bias, self.group)
        return _tp_linear(C.all_gather_seq(x, self.group), self.weight, bias)


class RowSequenceParallelLinear(nn.Module):
    """input ``[s, b, in/n]`` -> GEMM -> reduce-scatter along s -> ``[s/n, b, out]`` (+ bias)."""

    def __init__(self, in_features: int, out_features: int, mp_group=None, has_bias: bool = True, input_is_parallel: bool = True,
                 init_std: float = 0.02, dtype=None, device=None, fused_comm: bool = False, skip_bias_add: bool = False):
        super().__init__()
        assert input_is_parallel
        self.group = mp_group
        self.world = C.group_size(mp_group)
        self.in_per_rank = in_features // self.world
        self.fused_comm = fused_comm
        self.skip_bias_add = skip_bias_add
        self.weight = nn.Parameter(torch.empty(out_features, self.in_per_rank, dtype=dtype, device=device))
        _init_normal_sharded(self.weight, init_std, (out_features, in_features), 1, mp_group)
        _mark(self.weight, tp_sharded=self.world > 1, split_axis=1)
        if has_bias:
            self.bias = nn.Parameter(torch.zeros(out_features, dtype=dtype, device=device))
            # replicated param whose grad is computed from a sequence shard: needs an mp all-reduce
            _mark(self.bias, sequence_parallel=self.world > 1)
        else:
            self.register_parameter("bias", None)

    def forward(self, x: torch.Tensor):
        if (self.fused_comm or _OPTIONS["tp_comm"]) and x.is_cuda and self.world > 1:
            from .fused_tp import linear_reduce_scatter

            y = linear_reduce_scatter(x, self.weight, self.group)
        else:
            y = C.reduce_scatter_seq(_tp_linear(x, self.weight, None), self.group)
        if self.skip_bias_add:
            return y, self.bias
        return y if self.bias is None else y + self.bias


class VocabParallelEmbedding(nn.Module):
    def __init__(self, num_embeddings: int, embedding_dim: int, mp_group=None, init_std: float = 0.02, dtype=None, device=None):
        super().__init__()
        self.group = mp_group
        self.world = C.group_size(mp_group)
        assert num_embeddings % self.world == 0, f"vocab {num_embeddings} % mp {self.world}"
        self.num_embeddings = num_embeddings
        self.per_rank = num_embeddings // self.world
        self.vocab_start = C.group_rank(mp_group) * self.per_rank
        self.weight = nn.Parameter(torch.empty(self.per_rank, embedding_dim, dtype=dtype, device=device))
        _init_normal_sharded(self.weight, init_std, (num_embeddings, embedding_dim), 0, mp_group)
        _mark(self.weight, tp_sharded=self.world > 1, split_axis=0)

    def forward(self, ids: torch.Tensor, pos_ids=None, pos_weight=None) -> torch.Tensor:
        """``pos_ids`` / ``pos_weight``: optional (replicated) position table added in the same kernel (single-rank vocabulary only: under
        vocabulary parallelism the partial look-ups are summed over the group and the caller adds positions afterwards)."""
        if self.world == 1:
            return OF.embedding(ids, self.weight, 0, pos_ids, pos_weight)
        assert pos_weight is None, "fused position look-up needs an unsharded vocabulary"
        out = OF.embedding(ids, self.weight, self.vocab_start)
        return C.reduce_from_group(out, self.group)


class ParallelCrossEntropy(nn.Module):
    """Un-reduced vocab-parallel CE; logits ``[..., V/n]`` on each rank."""

    def __init__(self, mp_group=None):
        super().__init__()
        self.group = mp_group
        self.world = C.group_size(mp_group)

    def forward(self, logits: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        vocab_start = C.group_rank(self.group) * logits.shape[-1] if self.world > 1 else 0
        return OF.softmax_cross_entropy(logits, labels, self.group if self.world > 1 else None, vocab_start)


def parallel_matmul(x: torch.Tensor, weight: torch.Tensor, mp_group=None, parallel_output: bool = True) -> torch.Tensor:
    """Tied LM head: ``x @ E_shard^T`` with identity-fwd / all-reduce-bwd on x (reference hybrid_model.py:66-87)."""
    world = C.group_size(mp_group)
    if world > 1:
        x = C.copy_to_group(x, mp_group)
    logits = OF.linear(x, weight, None)
    if world > 1 and not parallel_output:
        logits = C.gather_last_dim(logits, mp_group)
    return logits


# ------------------------------------------------------------------ sequence-parallel param hooks
def is_sequence_parallel_parameter(p) -> bool:
    return getattr(p, "sequence_parallel", False)


def mark_as_sequence_parallel_parameter(p) -> None:
    p.sequence_parallel = True


def register_sequence_parallel_allreduce_hooks(model: nn.Module, accumulation_steps: int, fuse: bool, group) -> list:
    """LayerNorm weights/biases and row-linear biases see only a sequence shard under SP, so their grads are
    partial sums: all-reduce them over the mp group once per ``accumulation_steps`` backward passes
    (reference sequence_parallel_utils.py:155-212).  Returns the list of SP params; the engine calls
    ``allreduce_sequence_parallel_grads`` after the last micro-batch (one coalesced all-reduce)."""
    if accumulation_steps <= 0 or C.group_size(group) == 1:
        return []
    params = [p for p in model.parameters() if is_sequence_parallel_parameter(p)]
    model._sp_params = params
    model._sp_group = group
    return params


def allreduce_sequence_parallel_grads(model: nn.Module) -> None:
    params = getattr(model, "_sp_params", None)
    if params:
        C.fused_allreduce_gradients(params, model._sp_group, scale=1.0)


def create_fused_allreduce_gradient_hook(parameter_list, accumulation_steps: int, group=None):
    """A gradient hook shared by ``parameter_list``: once every parameter has produced its gradient ``accumulation_steps`` times, all of
    them are all-reduced over the tensor-parallel group in one coalesced call (reference sequence_parallel_utils.py:155-170).  Register it
    with ``p.register_post_accumulate_grad_hook`` (or ``register_hook``); the engine's default is the equivalent explicit call
    ``allreduce_sequence_parallel_grads`` after the last micro-batch."""
    if group is None:
        from ..distributed.apis import env

        group = env.get_hcg().get_model_parallel_group()
    parameter_list = list(parameter_list)
    fire_at, count = accumulation_steps * len(parameter_list), [0]

    def hook(arg=None):
        count[0] += 1
        if count[0] == fire_at:
            count[0] = 0
            C.fused_allreduce_gradients(parameter_list, group, scale=1.0)
        return None if isinstance(arg, nn.Parameter) else arg

    return hook


def create_non_fused_allreduce_gradient_hook(param, accumulation_steps: int, group=None):
    """Per-parameter variant: every ``accumulation_steps``-th call all-reduces ``param.main_grad`` (or ``param.grad``) over the
    tensor-parallel group (reference sequence_parallel_utils.py:173-188)."""
    if group is None:
        from ..distributed.apis import env

        group = env.get_hcg().get_model_parallel_group()
    count = [0]

    @torch.no_grad()
    def hook(*_):
        count[0] += 1
        if count[0] % accumulation_steps == 0:
            C.fused_allreduce_gradients([param], group, scale=1.0)

    return hook


def is_fused_matmul_bias_supported() -> bool:
    """The reference gates ``fused_linear`` on a cuBLASLt-epilogue capability of the Paddle build (sequence_parallel_utils.py:215-220).  Bias
    (and bias + GELU) always ride in the wgmma GEMM epilogue here when the native library is loaded."""
    from ..ops import _native

    return _native.available()


# sequence-parallel collectives under the reference's names (gpt/dygraph/sequence_parallel_utils.py:30-140)
from .comm_ops import _AllGatherSeq as AllGatherOp  # noqa: E402,F401
from .comm_ops import _GatherSeq as GatherOp  # noqa: E402,F401
from .comm_ops import _ReduceScatterSeq as ReduceScatterOp  # noqa: E402,F401
from .comm_ops import _ScatterSeq as ScatterOp  # noqa: E402,F401
from .comm_ops import all_gather_seq as all_gather  # noqa: E402,F401
from .comm_ops import reduce_scatter_seq as reduce_scatter  # noqa: E402,F401
from .comm_ops import scatter_seq as scatter  # noqa: E402,F401

