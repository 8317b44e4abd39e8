"""Ring context parallelism with packed documents and grouped K/V heads, without a GPU: the per-block document bounds of
``RingDocumentMask`` against a brute-force count, the ring's block schedule replayed in one process against dense float64 document
attention (with G = 1, 2, 4), gloo parity of GPT under ``cp_mode: ring`` with ``reset_attention_mask``, RoPE and GQA (with mp2 and ZeRO
stage 2), and the config rules."""
import os

import numpy as np
import pytest
import torch

from dist_utils import run_distributed
from paddlefleetx_b200.data.dataset.gpt_dataset import document_positions
from paddlefleetx_b200.parallel import ring_attention as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "paddlefleetx_b200", "configs", "nlp", "gpt")


def _positions(lengths, s):
    return torch.tensor(np.asarray(document_positions(lengths, s)), dtype=torch.int64)


def _doc_start(pos):
    """Global first key of every query's document: ``clamp(i - pos, 0, i)`` over the whole sequence."""
    i = torch.arange(pos.shape[-1], device=pos.device)
    return torch.minimum((i - pos).clamp_min(0), i)


def _global_rows(c, r, h):
    return torch.cat([r * h + torch.arange(h), (2 * c - 1 - r) * h + torch.arange(h)])


# ---------------------------------------------------------------------------------------------------------------- bounds
def _layouts(c, h):
    s = 2 * c * h
    return [
        [s],                                             # one document per row
        [h - 1, 1, h, s],                                # shorter than, then equal to a chunk, aligned to the chunk boundaries
        [3, 2 * h + 5, s],                               # longer than a chunk, crossing two chunk boundaries
        [1] * 7 + [h // 2 + 3, s],                       # single-token documents, then one that crosses a boundary
        [max(1, h // 3)] * (3 * c) + [s],                # many short ones, some of them crossing chunk boundaries
    ]


@pytest.mark.parametrize("c", [1, 2, 3, 4])
def test_block_bounds_count_the_keys_before_each_document(c):
    h = 70                                               # two 64-row tiles per chunk, the second ragged
    s = 2 * c * h
    for lengths in _layouts(c, h):
        full = torch.stack([_positions(lengths, s), _positions(list(reversed(lengths[:-1])) + [s], s)])
        start = _doc_start(full)
        for r in range(c):
            rows = _global_rows(c, r, h)
            m = R.RingDocumentMask.from_positions(R.zigzag_slice(full, c, r), c, r)
            for src in range(c):
                qs, ks, _ = R._block_plan(True, r, src, h)
                q_rows = rows[qs]
                keys = _global_rows(c, src, h)[ks]
                want = (keys.view(1, 1, -1) < start[:, q_rows].unsqueeze(-1)).sum(-1).to(torch.int32)
                blk = m.block(src)
                assert torch.equal(blk.key_start, want), (lengths, r, src)
                t = -(-want.shape[1] // 64)
                for j in range(t):
                    part = want[:, 64 * j:64 * (j + 1)]
                    assert torch.equal(blk.tile_min[:, j], part.amin(-1)) and torch.equal(blk.tile_max[:, j], part.amax(-1))
                assert blk.key_start.is_contiguous() and blk.tile_min.shape == (2, t)
                if src == r:                             # the diagonal block is causal and keeps every row's own key
                    assert bool((want <= torch.arange(want.shape[1])).all())


# ---------------------------------------------------------------------------------------------------------------- block schedule
def replay(q, k, v, dout, pos, c, scale):
    """(out, dq, dk, dv) over the full sequence, rank by rank through the ring's block functions with the document masks (the native
    kernels where the blocks reach them)."""
    loc = [[R.zigzag_slice(t, c, r) for t in (q, k, v, dout)] for r in range(c)]
    masks = [R.RingDocumentMask.from_positions(R.zigzag_slice(pos, c, r), c, r) for r in range(c)]
    half = loc[0][0].shape[1] // 2
    outs, lses = [], []
    for r in range(c):
        out = lse = None
        for step in range(c):
            src = (r - step) % c
            qs, ks, bc = R._block_plan(True, r, src, half)
            o_b, l_b = R._block_fwd(loc[r][0][:, qs], loc[src][1][:, ks], loc[src][2][:, ks], bc, scale, 0.0, 0, doc=masks[r].block(src))
            if qs == slice(None):
                out, lse = R._merge(out, lse, o_b, l_b)
            else:
                o2, l2 = R._merge(out[:, qs], lse[:, :, qs], o_b, l_b)
                out, lse = torch.cat([out[:, :half], o2], 1), torch.cat([lse[:, :, :half], l2], 2)
        assert bool(torch.isfinite(lse).all())
        outs.append(out.to(q.dtype))
        lses.append(lse)
    md = R._math_dtype(q)
    dqs = [torch.zeros(loc[r][0].shape, dtype=md, device=q.device) for r in range(c)]
    dks = [torch.zeros(loc[r][1].shape, dtype=md, device=q.device) for r in range(c)]
    dvs = [torch.zeros(loc[r][2].shape, dtype=md, device=q.device) for r in range(c)]
    for r in range(c):
        for step in range(c):
            src = (r - step) % c
            qs, ks, bc = R._block_plan(True, r, src, half)
            gq, gk, gv = R._block_bwd(loc[r][0][:, qs], loc[src][1][:, ks], loc[src][2][:, ks], outs[r][:, qs], loc[r][3][:, qs], lses[r][:, :, qs],
                                      bc, scale, 0.0, 0, doc=masks[r].block(src))
            dqs[r][:, qs] += gq.to(md)
            dks[src][:, ks] += gk.to(md)
            dvs[src][:, ks] += gv.to(md)
    return tuple(R.zigzag_merge(x) for x in (outs, dqs, dks, dvs))


def dense_document_attention(q, k, v, dout, pos, scale):
    """float64 reference: query i attends keys [doc_start(i), i], K / V heads repeated per group; returns (out, dq, dk, dv)."""
    qf, kf, vf = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    g = q.shape[2] // k.shape[2]
    kr, vr = kf.repeat_interleave(g, dim=2), vf.repeat_interleave(g, dim=2)
    s = q.shape[1]
    j = torch.arange(s, device=q.device)
    allowed = (j.view(1, 1, s) >= _doc_start(pos).unsqueeze(-1)) & (j.view(1, 1, s) <= j.view(1, s, 1))
    sc = torch.einsum("bqhd,bkhd->bhqk", qf, kr) * scale
    p = torch.softmax(sc.masked_fill(~allowed.unsqueeze(1), float("-inf")), -1)
    o = torch.einsum("bhqk,bkhd->bqhd", p, vr)
    (o * dout.double()).sum().backward()
    return o.detach(), qf.grad, kf.grad, vf.grad


@pytest.mark.parametrize("c,g", [(2, 1), (3, 2), (4, 4), (4, 1)])
def test_ring_replay_with_documents_matches_dense_float64(c, g):
    torch.manual_seed(3)
    b, h, hkv, d = 2, 4, 4 // g, 8
    half = 5
    s = 2 * c * half
    pos = torch.stack([_positions([3, half, 2 * half + 1, 1, s], s), _positions([2 * half - 1, s], s)])
    q, do = (torch.randn(b, s, h, d, dtype=torch.float64) for _ in range(2))
    k, v = (torch.randn(b, s, hkv, d, dtype=torch.float64) for _ in range(2))
    got = replay(q, k, v, do, pos, c, d ** -0.5)
    for name, a, r_ in zip(("out", "dq", "dk", "dv"), got, dense_document_attention(q, k, v, do, pos, d ** -0.5)):
        torch.testing.assert_close(a, r_, atol=1e-12, rtol=1e-10, msg=name)


def test_empty_rows_give_zero_and_minus_infinity():
    """A non-causal block row whose document starts after the block's keys: out 0, lse -inf, and the merge keeps the accumulator."""
    torch.manual_seed(4)
    q, k, v = (torch.randn(1, 6, 2, 4, dtype=torch.float64) for _ in range(3))
    from paddlefleetx_b200.ops.attention import DocumentMask

    doc = DocumentMask.with_tile_bounds(torch.tensor([[0, 2, 6, 6, 5, 6]], dtype=torch.int32))
    out, lse = R._block_fwd(q, k, v, False, 0.5, 0.0, 0, doc=doc)
    assert torch.equal(out[0, 2], torch.zeros(2, 4, dtype=torch.float64)) and bool((lse[0, :, 2] == float("-inf")).all())
    assert bool(torch.isfinite(lse[0, :, 4]).all())
    acc_o, acc_l = torch.randn(1, 6, 2, 4, dtype=torch.float64), torch.randn(1, 2, 6, dtype=torch.float64)
    mo, ml = R._merge(acc_o, acc_l, out, lse)
    torch.testing.assert_close(mo[:, 2:4], acc_o[:, 2:4], atol=0, rtol=0)
    torch.testing.assert_close(ml[:, :, 2:4], acc_l[:, :, 2:4], atol=0, rtol=0)


# ---------------------------------------------------------------------------------------------------------------- gloo parity
def _doc_batches(cfg, n):
    from helpers import synthetic_batches

    batches = synthetic_batches(cfg, n, seed=21)
    s = batches[0][0].shape[1]
    for i, b in enumerate(batches):
        b[1] = torch.stack([_positions([5 + 3 * i, 9, s], s), _positions([s // 2 + 1, 2, s], s)])
    return batches


def ring_docs_match_single(rank, world, mp, cp, stage, extra):
    """GPT under ring context parallelism (x mp, ZeRO ``stage``) with the document mask: the same losses and weights as one process."""
    import torch.distributed as dist

    from dist_fns import _shard_like
    from helpers import tiny_gpt_config
    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module
    from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

    ov = ["Global.global_batch_size=None", "Global.local_batch_size=2", "Global.micro_batch_size=2", "Model.reset_attention_mask=True",
          "Data.Train.dataset.reset_position_ids=True", "Data.Eval.dataset.reset_position_ids=True"] + list(extra)
    cfg1 = tiny_gpt_config(ov, nranks=1)
    env.set_hcg(HybridCommunicateGroup(world_size=1, rank=0, build_groups=False))
    real_ws = env.world_size
    env.world_size = lambda: 1
    try:
        env.set_seed(cfg1.Global.seed)
        module1 = build_module(cfg1)
        init = {k: v.detach().clone() for k, v in module1.model.state_dict().items()}
        eng1 = EagerEngine(configs=cfg1, module=module1)
        batches = _doc_batches(cfg1, 3)
        ref_losses = [float(eng1.train_step(b)) for b in batches]
        ref_state = {k: v.detach().clone() for k, v in module1.model.state_dict().items()}
    finally:
        env.world_size = real_ws
        env.set_hcg(None)
    data = world // mp
    assert data == cp
    cfg = tiny_gpt_config(ov + [f"Distributed.mp_degree={mp}", f"Model.sequence_parallel={mp > 1}", f"Distributed.sharding.sharding_degree={data}",
                                f"Distributed.sharding.sharding_stage={stage}", f"Distributed.cp_degree={cp}", "Distributed.cp_mode=ring"], nranks=world)
    from paddlefleetx_b200.utils import check

    assert check.check_config(cfg)
    hcg = env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    module = build_module(cfg)
    attn = module.model.gpt.decoder.layers[0].self_attn
    assert attn.cp_mode == "ring" and attn.cp_group.nranks == cp
    with torch.no_grad():
        for k, p in module.model.named_parameters():
            p.copy_(_shard_like(init[k], p, hcg.get_model_parallel_rank(), mp))
    eng = EagerEngine(configs=cfg, module=module)
    built = []
    real_build = R.RingDocumentMask.from_positions.__func__
    R.RingDocumentMask.from_positions = classmethod(lambda cls, *a: built.append(1) or real_build(cls, *a))
    losses = []
    try:
        for b in batches:
            l = eng.train_step(b).detach().clone()
            dist.all_reduce(l)
            losses.append(float(l) / world)
    finally:
        R.RingDocumentMask.from_positions = classmethod(real_build)
    assert len(built) == len(batches), "one ring document mask per step, shared by every layer"
    assert max(abs(a - b) for a, b in zip(losses, ref_losses)) < 3e-4, (losses, ref_losses)
    kvh, grp = attn.local_kv_heads, attn.group
    for k, p in module.model.named_parameters():
        want, got = _shard_like(ref_state[k], p, hcg.get_model_parallel_rank(), mp), p.detach()
        if k.endswith("qkv_proj.bias"):          # K-bias entries: zero gradient in theory, Adam-normalised rounding noise in practice
            keep = [i for i in range(grp + 2) if i != grp]
            want, got = want.view(kvh, grp + 2, -1)[:, keep], got.view(kvh, grp + 2, -1)[:, keep]
        bad = ((got - want).abs() > 1e-4 + 1e-3 * want.abs())
        assert int(bad.sum()) <= max(1, bad.numel() // 1000) and float((got - want).abs().max()) < 1e-3, \
            (k, float((got - want).abs().max()), int(bad.sum()), bad.numel())


@pytest.mark.parametrize("world,mp,cp,stage,extra", [
    (2, 1, 2, 2, ["Model.use_rope=True"]),
    (4, 1, 4, 2, ["Model.use_rope=True", "Model.num_key_value_heads=2"]),
    (4, 2, 2, 2, ["Model.use_rope=True", "Model.num_key_value_heads=2"]),
    (4, 2, 2, 1, []),
], ids=["cp2-rope", "cp4-rope-gqa-zero2", "mp2-cp2-rope-gqa-zero2", "mp2-cp2"])
def test_ring_context_parallel_with_documents_matches_single(world, mp, cp, stage, extra):
    run_distributed("test_ring_doc_attention_cpu:ring_docs_match_single", world, mp, cp, stage, extra)


# ---------------------------------------------------------------------------------------------------------------- config
BASE = ["Model.reset_attention_mask=True", "Data.Train.dataset.reset_position_ids=True", "Data.Eval.dataset.reset_position_ids=True"]


@pytest.mark.parametrize("extra,dist,needle", [
    (BASE, {"cp_degree": 2, "cp_mode": "ring"}, None),
    (["Model.num_key_value_heads=2"], {"cp_degree": 2, "cp_mode": "ring"}, None),
    (BASE + ["Model.num_key_value_heads=2"], {"cp_degree": 4, "cp_mode": "ring"}, None),
    (BASE, {"cp_degree": 2, "cp_mode": "ulysses"}, "cp_mode: ring"),
    (["Model.num_key_value_heads=2"], {"cp_degree": 2}, "cp_mode: ring"),
    (BASE, {"pp_degree": 2, "cp_degree": 2, "cp_mode": "ring"}, "pp_degree"),
    (BASE + ["Data.Train.dataset.max_seq_len=36"], {"cp_degree": 4, "cp_mode": "ring"}, "multiple of"),
])
def test_config_rules(extra, dist, needle):
    from helpers import tiny_gpt_config
    from paddlefleetx_b200.utils import check

    cfg = tiny_gpt_config(extra, nranks=1)
    cfg.Distributed.update(dist)
    if needle is None:
        assert check.check_config(cfg)
    else:
        with pytest.raises(ValueError, match=needle):
            check.check_config(cfg)


def test_recipe_passes_the_config_checks():
    from paddlefleetx_b200.utils import check
    from paddlefleetx_b200.utils import config as C

    cfg = C.get_config(os.path.join(CFG, "pretrain_gpt_1.3B_seq32768_cp8_ring_packed_docs.yaml"), [], show=False, nranks=8)
    assert cfg.Model.reset_attention_mask and cfg.Distributed.cp_mode == "ring" and cfg.Distributed.cp_degree == 8
    assert cfg.Data.Train.dataset.reset_position_ids and cfg.Data.Eval.dataset.reset_position_ids
    assert check.check_config(cfg)
