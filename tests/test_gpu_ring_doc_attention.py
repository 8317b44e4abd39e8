"""Ring context parallelism with packed documents on the sm_90a flash kernels (needs an H100).

The non-causal document kernels at the ring's block shapes (Sq = 2 Sk and Sk = 2 Sq) against float64 within the ``kernel_refs`` budgets
(bf16 / fp16, D 64 / 128, G 1 / 4, dropout, gradients written into NaN-filled buffers); rows that see no key give out 0 and lse -inf and key
tiles that no query reaches give dk = dv = 0, exactly; with every key_start = 0 the kernels equal the plain non-causal ones bit for bit
(dq up to its reduction order).  Then the ring schedule through the kernels against float64 document attention over the whole sequence,
the native bounds launch against the CPU derivation, and, with two GPUs, a two-rank NCCL ring against one GPU.
"""
import math
import os

import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import attention as ATT
from paddlefleetx_b200.ops import functional as OF
from paddlefleetx_b200.parallel import ring_attention as RA
from test_ring_doc_attention_cpu import _global_rows, _positions, dense_document_attention, replay

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]


def _lib():
    return _native.require()


# ---------------------------------------------------------------------------------------------------------------- float64 references
def _logits(q, k, scale, mask):
    """Non-causal logits with ``mask`` (bool [B, Sq, Sk], True = attend) set to -inf: ``doc_attention_refs`` without the causal mask."""
    qh = R._bhsd(q)
    kh = R._bhsd(k, qh.shape[1])
    s = qh @ kh.transpose(-1, -2) * scale
    return qh, kh, s.masked_fill(~mask.to(s.device).unsqueeze(1), -math.inf)


def _attention(q, k, v, scale, mask, keep=None, p=0.0):
    qh, kh, s = _logits(q, k, scale, mask)
    pi, lse = R._softmax_rows(s)
    return ((pi * R._keep_factor(keep, p, pi)) @ R._bhsd(v, qh.shape[1])).transpose(1, 2), lse


def _attention_bwd(q, k, v, dout, scale, mask, keep=None, p=0.0):
    qd, kd, vd = (R._d(t).clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        out, _ = _attention(qd, kd, vd, scale, mask, keep, p)
        return torch.autograd.grad(out, (qd, kd, vd), R._d(dout))


def _bounds(q, k, v, dout, scale, mask, dtype, keep=None, p=0.0):
    """``assert_close`` arguments for out, lse, dq, dk, dv (the budgets of ``doc_attention_refs``)."""
    qh, kh, s = _logits(q, k, scale, mask)
    H, Hkv = qh.shape[1], k.shape[2]
    vh, doh = R._bhsd(v, H), R._bhsd(dout)
    pi, lse = R._softmax_rows(s)
    kw = R._keep_factor(keep, p, pi)
    out_h = (pi * kw) @ vh
    Sq, Sk = s.shape[-2], s.shape[-1]
    ds = R._logit_err(qh, kh, s, pi, lse, scale)
    E_o = R._fwd_budget(pi, kw, vh, out_h, ds, dtype, -(-Sk // 128))
    E_lse = ds.squeeze(-1) + R.EX2_APPROX + R.LG2_APPROX + R.FP32_U * math.sqrt(Sk)
    rel_p = 2 * ds + R.EX2_APPROX + R.LG2_APPROX + R.FP32_U * math.sqrt(Sk) + R.EX2_APPROX
    E_dq, E_dk, E_dv = R._bwd_budget(qh, kh, vh, doh, pi, kw, rel_p, E_o, out_h, dtype, scale, -(-Sq // 64), -(-Sk // 64))
    return (R._abs_bound(E_o.transpose(1, 2)), R._abs_bound(E_lse), R._abs_bound(E_dq.transpose(1, 2)),
            R._abs_bound(R._group_sum(E_dk, Hkv).transpose(1, 2)), R._abs_bound(R._group_sum(E_dv, Hkv).transpose(1, 2)))


def _ring_block(c, r, src, h, lengths):
    """The document mask of rank r's block from rank src (native bounds) for two rows of documents, and its dense bool form."""
    s = 2 * c * h
    full = torch.stack([_positions(lengths, s), _positions(list(reversed(lengths[:-1])) + [s], s)]).cuda()
    doc = RA.RingDocumentMask.from_positions(RA.zigzag_slice(full, c, r), c, r).block(src)
    qs, ks, causal = RA._block_plan(True, r, src, h)
    sk = len(_global_rows(c, src, h)[ks])
    assert not causal
    mask = torch.arange(sk, device="cuda").view(1, 1, sk) >= doc.key_start.long().unsqueeze(-1)
    return doc, mask, sk


# ---------------------------------------------------------------------------------------------------------------- kernels
CASES = [   # (c, r, src, chunk h, document lengths): src < r gives Sq = 2 Sk, src > r gives Sk = 2 Sq
    (4, 2, 1, 256, [100, 300, 64, 129, 1, 4000, 8192]),
    (4, 1, 3, 256, [77, 520, 1, 1, 1000, 8192]),
    (2, 1, 0, 1088, [900, 700, 1300, 8192]),
    (2, 0, 1, 1088, [1500, 64, 2000, 8192]),
    (4, 3, 0, 4096, [5000, 3000, 12000, 70000]),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: f"c{c[0]}-r{c[1]}-src{c[2]}-h{c[3]}")
@pytest.mark.parametrize("D,G", [(128, 1), (64, 1), (64, 4), (128, 4)])
@pytest.mark.parametrize("p", [0.0, 0.2])
def test_noncausal_document_kernels_match_float64(case, D, G, p):
    c, r, src, h, lengths = case
    if h == 4096 and (D, G, p) != (128, 1, 0.0):
        pytest.skip("the largest chunk runs once: its float64 reference is the expensive part")
    doc, mask, sk = _ring_block(c, r, src, h, lengths)
    B, sq = doc.key_start.shape
    H = 2 if h == 4096 else 8
    masters = R.attention_inputs(B, sq, sk, H, D, H // G, seed=h + src, device="cuda")
    scale, dseed = D ** -0.5, 0xD0C + sq
    keep = ATT.attn_keep_mask(dseed, B, H, sq, sk, p, "cuda") if p > 0 else None
    empty = (doc.key_start == sk)
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        out, lse = _lib().attention_fwd_doc(q, k, v, *doc.bounds(), scale, p, dseed, False)
        dq, dk, dv = (torch.full_like(t, math.nan) for t in (q, k, v))
        _lib().attention_bwd_doc(q, k, v, out, do, lse, dq, dk, dv, *doc.bounds(), scale, p, dseed, False)
        ref, ref_lse = _attention(q, k, v, scale, mask, keep, p)
        okw, lkw, qkw, kkw, vkw = _bounds(q, k, v, do, scale, mask, dt, keep, p)
        R.assert_close(out, ref, dt, what="out", **okw)
        live = ~empty.unsqueeze(1).expand_as(lse)
        R.assert_close(lse[live], ref_lse[live].float(), torch.float32, scale=lkw["scale"][live], approx=1.0, what="lse")
        assert bool((out[empty] == 0).all()) and bool((lse.transpose(1, 2)[empty] == -math.inf).all())
        rdq, rdk, rdv = _attention_bwd(q, k, v, do, scale, mask, keep, p)
        for name, got, want, kw in (("dq", dq, rdq, qkw), ("dk", dk, rdk, kkw), ("dv", dv, rdv, vkw)):
            R.assert_close(got, want, dt, what=name, **kw)


def test_empty_blocks_write_zeros():
    """Documents shorter than a chunk: the block of an earlier, non-adjacent rank holds no key of any local document.  Every row is empty
    (out 0, lse -inf) and no query tile reaches any key tile (dk = dv = 0, written over NaN)."""
    c, r, src, h = 4, 2, 0, 512
    doc, mask, sk = _ring_block(c, r, src, h, [128] * 64 + [8192])
    assert bool((doc.key_start == sk).all())
    for dt in DTYPES:
        q, do = (torch.randn(2, 2 * h, 8, 128, device="cuda", dtype=dt) for _ in range(2))
        k, v = (torch.randn(2, sk, 2, 128, device="cuda", dtype=dt) for _ in range(2))
        out, lse = _lib().attention_fwd_doc(q, k, v, *doc.bounds(), 0.1, 0.0, 0, False)
        assert bool((out == 0).all()) and bool((lse == -math.inf).all())
        dq, dk, dv = (torch.full_like(t, math.nan) for t in (q, k, v))
        _lib().attention_bwd_doc(q, k, v, out, do, lse, dq, dk, dv, *doc.bounds(), 0.1, 0.0, 0, False)
        assert bool((dq == 0).all()) and bool((dk == 0).all()) and bool((dv == 0).all())


@pytest.mark.parametrize("sq,sk,G", [(1024, 512, 1), (512, 1024, 4), (640, 2176, 2)])
@pytest.mark.parametrize("D", [64, 128])
def test_zero_key_start_equals_the_noncausal_kernels_bitwise(sq, sk, G, D):
    B, H = 2, 8
    doc = ATT.DocumentMask.with_tile_bounds(torch.zeros(B, sq, dtype=torch.int32, device="cuda"))
    masters = R.attention_inputs(B, sq, sk, H, D, H // G, seed=7, device="cuda")
    for dt in DTYPES:
        for p in (0.0, 0.1):
            q, k, v, do = (m.to(dt) for m in masters)
            out, lse = _lib().attention_fwd_doc(q, k, v, *doc.bounds(), D ** -0.5, p, 99, False)
            out0, lse0 = _lib().attention_fwd_v2(q, k, v, False, D ** -0.5, p, 99)
            assert torch.equal(out, out0) and torch.equal(lse, lse0)
            g = [torch.empty_like(t) for t in (q, k, v)]
            g0 = [torch.empty_like(t) for t in (q, k, v)]
            _lib().attention_bwd_doc(q, k, v, out, do, lse, *g, *doc.bounds(), D ** -0.5, p, 99, False)
            _lib().attention_bwd(q, k, v, out0, do, lse0, *g0, False, D ** -0.5, p, 99)
            assert torch.equal(g[1], g0[1]) and torch.equal(g[2], g0[2])
            torch.testing.assert_close(g[0], g0[0], atol=2e-2, rtol=2e-2)


# ---------------------------------------------------------------------------------------------------------------- ring schedule
@pytest.mark.parametrize("c,h,G", [(2, 512, 1), (4, 256, 4), (8, 128, 2), (8, 192, 1)])
def test_ring_replay_on_the_kernels_matches_float64(c, h, G):
    torch.manual_seed(c + h)
    b, H, d = 2, 8, 128
    s = 2 * c * h
    pos = torch.stack([_positions([h // 2 + 3, 3 * h + 1, 70, 1, 1, 2 * h, s], s), _positions([5 * h - 7, 200, s], s)]).cuda()
    q, do = (torch.randn(b, s, H, d, device="cuda").bfloat16() for _ in range(2))
    k, v = (torch.randn(b, s, H // G, d, device="cuda").bfloat16() for _ in range(2))
    loc = RA.zigzag_slice(q, c, 1)
    kl = RA.zigzag_slice(k, c, 1)
    m = RA.RingDocumentMask.from_positions(RA.zigzag_slice(pos, c, 1), c, 1)
    assert ATT._native_ok(loc, kl, kl, None, True, True, m.block(1)) and ATT._native_ok(loc, kl[:, :h], kl[:, :h], None, False, True, m.block(0))
    got = replay(q, k, v, do, pos, c, d ** -0.5)
    ref = dense_document_attention(q, k, v, do, pos, d ** -0.5)
    for name, a, r_ in zip(("out", "dq", "dk", "dv"), got, ref):
        err = float((a.double() - r_).norm() / r_.norm())
        assert err < 2e-2, (name, err)


@pytest.mark.parametrize("c", [1, 2, 3, 8])
def test_native_bounds_equal_the_cpu_derivation_in_one_launch(c):
    h = 200
    s = 2 * c * h
    full = torch.stack([_positions([3, h, 2 * h + 5, 1, 1, 130, s], s), _positions([s], s), _positions([64] * (s // 64 + 1), s)])
    for r in range(c):
        local = RA.zigzag_slice(full, c, r)
        OF.reset_launch_count()
        gpu = RA.RingDocumentMask.from_positions(local.cuda(), c, r)
        assert OF.native_launch_count() == 1
        cpu = RA.RingDocumentMask.from_positions(local, c, r)
        for src in range(c):
            for a, b_ in zip(gpu.block(src).bounds(), cpu.block(src).bounds()):
                assert a.is_contiguous() and torch.equal(a.cpu(), b_), (r, src)


# ---------------------------------------------------------------------------------------------------------------- two GPUs
def _nccl_rank(rank, world, port, q, k, v, do, pos, res):
    import torch.distributed as dist

    from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    try:
        group = HybridCommunicateGroup(dp=world, cp=world, cp_mode="ring").get_context_parallel_group()
        loc = [RA.zigzag_slice(t, world, rank).cuda().requires_grad_(True) for t in (q, k, v)]
        m = RA.RingDocumentMask.from_positions(RA.zigzag_slice(pos, world, rank).cuda(), world, rank)
        out = RA.ring_attention(*loc, group, causal=True, doc=m)
        out.backward(RA.zigzag_slice(do, world, rank).cuda())
        res[rank] = [t.detach().cpu() for t in (out, loc[0].grad, loc[1].grad, loc[2].grad)]
    finally:
        dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_gpu_nccl_ring_matches_one_gpu():
    import socket

    import torch.multiprocessing as mp

    c, h, H, d = 2, 512, 8, 128
    s = 2 * c * h
    torch.manual_seed(5)
    q, do = (torch.randn(2, s, H, d).bfloat16() for _ in range(2))
    k, v = (torch.randn(2, s, 2, d).bfloat16() for _ in range(2))
    pos = torch.stack([_positions([300, 900, 64, s], s), _positions([s], s)])
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    res = mp.Manager().dict()
    mp.spawn(_nccl_rank, args=(c, port, q, k, v, do, pos, res), nprocs=c, join=True)
    got = [RA.zigzag_merge([res[r][i] for r in range(c)]) for i in range(4)]
    want = replay(q.cuda(), k.cuda(), v.cuda(), do.cuda(), pos.cuda(), c, d ** -0.5)
    for name, a, b_ in zip(("out", "dq", "dk", "dv"), got, want):
        torch.testing.assert_close(a.float(), b_.float().cpu(), atol=2e-2, rtol=2e-2, msg=name)
