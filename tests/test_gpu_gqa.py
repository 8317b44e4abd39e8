"""Grouped-query attention on the sm_90a flash, decode and KV-cache paths (needs an H100).

Every kernel case is checked against an fp32 reference that repeats K/V per group (``repeat_interleave``: query head h reads K/V head
h // G) and drops the elements ``attn_keep_mask`` names, with the bounds of test_gpu_fp16.py: bf16 within 3e-2 of the reference and
fp16 closer than half of bf16's error."""
import os
import re

import numpy as np
import pytest
import torch

from paddlefleetx_b200.ops import attention as ATT
from paddlefleetx_b200.ops import functional as OF
from paddlefleetx_b200.ops import _native

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16


def _lib():
    return _native.require()


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _assert_fp16_closer(errs, bf16_bound=3e-2):
    for i, (e16, eb) in enumerate(zip(errs[F16], errs[B16])):
        assert eb < bf16_bound, ("bf16 result is off", i, errs)
        assert e16 < 0.5 * eb, ("fp16 result is not closer to fp32 than bf16's", i, errs)


def _reference(q, k, v, go, causal, scale, keep, p):
    """fp32 attention with K/V repeated to the query heads; returns (out, lse, dq, dk, dv)."""
    g = q.shape[2] // k.shape[2]
    Sq, Sk = q.shape[1], k.shape[1]
    q, k, v = (t.detach().float().clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        kr, vr = k.repeat_interleave(g, 2), v.repeat_interleave(g, 2)
        s = torch.einsum("bqhd,bkhd->bhqk", q, kr) * scale
        if causal:
            s = s.masked_fill(~torch.ones(Sq, Sk, dtype=torch.bool, device="cuda").tril(Sk - Sq), float("-inf"))
        pr = torch.softmax(s, -1)
        if keep is not None:
            pr = pr * keep.float() / (1.0 - p)
        o = torch.einsum("bhqk,bkhd->bqhd", pr, vr)
        o.backward(go.float())
    return o.detach(), torch.logsumexp(s.detach(), -1), q.grad, k.grad, v.grad


# B, Sq, Sk, H, Hkv, causal, p, layout, D   (G = H / Hkv covers 1, 2, 4, 8 and H)
CASES = [(2, 256, 256, 8, 8, True, 0.0, "plain", 128), (2, 200, 200, 8, 4, False, 0.0, "plain", 128), (1, 128, 320, 8, 2, True, 0.0, "plain", 64),
         (2, 577, 577, 8, 1, False, 0.1, "plain", 64), (1, 192, 320, 4, 2, False, 0.1, "plain", 128),
         (2, 384, 384, 8, 2, True, 0.1, "packed", 128), (1, 300, 300, 4, 1, True, 0.0, "packed", 64), (2, 256, 256, 4, 2, False, 0.0, "packed", 128),
         (2, 260, 260, 8, 1, True, 0.0, "packed", 128),
         (2, 384, 384, 8, 1, True, 0.1, "seq_major", 128), (2, 197, 260, 6, 3, False, 0.0, "seq_major", 64), (1, 256, 256, 16, 2, True, 0.0, "seq_major", 64)]


def _views(masters, Hkv, layout, dt):
    """q ([B,S,H,D] or the [B,S,Hkv,G,D] slice of a packed projection), k, v in the requested storage, and matching gradient views."""
    q, k, v = (m.to(dt) for m in masters)
    B, S, H, D = q.shape
    G = H // Hkv
    if layout == "plain":
        return (q, k, v), (torch.empty_like(q), torch.empty_like(k), torch.empty_like(v))
    if layout == "seq_major":
        qs, ks, vs = (t.transpose(0, 1).contiguous().transpose(0, 1) for t in (q, k, v))
        return (qs, ks, vs), tuple(torch.empty_like(t.transpose(0, 1)).transpose(0, 1) for t in (q, k, v))
    mix = torch.cat([q.view(B, S, Hkv, G, D), k.unsqueeze(3), v.unsqueeze(3)], dim=3)      # [B, S, Hkv, G + 2, D]
    dmix = torch.empty_like(mix)
    split = (lambda m: m.unbind(3)) if G == 1 else (lambda m: (m[:, :, :, :G], m[:, :, :, G], m[:, :, :, G + 1]))
    return split(mix), split(dmix)


@pytest.mark.parametrize("case", CASES, ids=lambda c: "B{}_Sq{}_Sk{}_H{}_Hkv{}_{}_p{}_{}_D{}".format(*c[:5], "causal" if c[5] else "full", *c[6:]))
def test_flash_attention_grouped_kv(case):
    B, Sq, Sk, H, Hkv, causal, p, layout, D = case
    torch.manual_seed(11)
    scale = D ** -0.5
    seed = 0x2468ACE + 31 * Sq
    keep = ATT.attn_keep_mask(seed, B, H, Sq, Sk, p, "cuda") if p > 0 else None
    masters = [torch.randn(B, Sq, H, D, device="cuda"), torch.randn(B, Sk, Hkv, D, device="cuda"), torch.randn(B, Sk, Hkv, D, device="cuda"),
               torch.randn(B, Sq, H, D, device="cuda") * 0.5]
    errs = {}
    for dt in (F16, B16):
        (q, k, v), (dq, dk, dv) = _views(masters[:3], Hkv, layout, dt)
        go = masters[3].to(dt)
        out, lse = _lib().attention_fwd_v2(q, k, v, causal, scale, p, seed)
        assert out.shape == (B, Sq, H, D) and lse.shape == (B, H, Sq)
        _lib().attention_bwd(q, k, v, out, go, lse, dq, dk, dv, causal, scale, p, seed)
        dk1, dv1 = dk.clone(), dv.clone()
        _lib().attention_bwd(q, k, v, out, go, lse, dq, dk, dv, causal, scale, p, seed)
        torch.cuda.synchronize()
        assert torch.equal(dk, dk1) and torch.equal(dv, dv1), "dK / dV differ between two backward runs"
        dq_full = dq.reshape(B, Sq, H, D) if dq.dim() == 5 else dq
        qr = q.reshape(B, Sq, H, D) if q.dim() == 5 else q
        own = _reference(qr, k, v, go, causal, scale, keep, p)
        master_lse = _reference(*masters, causal, scale, keep, p)[1]
        errs[dt] = [_rel(out, own[0]), _rel(lse, master_lse), _rel(dq_full, own[2]), _rel(dk, own[3]), _rel(dv, own[4])]
    _assert_fp16_closer(errs)


def test_grouped_dropout_keeps_the_pairs_of_the_repeated_kv_call():
    """Same seed: a grouped call drops exactly the elements an H-head call with K/V repeated drops (the key is per query head)."""
    B, Sq, Sk, H, Hkv, D, p, seed = 2, 100, 128, 8, 2, 128, 0.25, 123456789
    q = torch.zeros(B, Sq, H, D, device="cuda", dtype=B16)
    k = torch.zeros(B, Sk, Hkv, D, device="cuda", dtype=B16)
    v = torch.eye(Sk, D, device="cuda", dtype=B16).view(1, Sk, 1, D).expand(B, Sk, Hkv, D).contiguous()
    out, _ = _lib().attention_fwd_v2(q, k, v, False, D ** -0.5, p, seed)
    got = (out.float() > 0).permute(0, 2, 1, 3)
    assert torch.equal(got, ATT.attn_keep_mask(seed, B, H, Sq, Sk, p, "cuda"))


@pytest.mark.parametrize("Hkv,dt", [(2, B16), (1, F16), (4, B16)])
def test_packed_and_unpacked_autograd_front_ends(Hkv, dt):
    """flash_attention_packed takes [b, s, Hkv, G + 2, d] and returns ONE packed gradient; attention(q, k, v) takes fewer K/V heads."""
    torch.manual_seed(3)
    B, S, H, D = 2, 256, 8, 128
    G = H // Hkv
    mix = (torch.randn(B, S, Hkv, G + 2, D, device="cuda") * 0.7).to(dt).requires_grad_(True)
    go = torch.randn(B, S, H, D, device="cuda", dtype=dt)
    out = ATT.flash_attention_packed(mix, causal=True)
    assert out is not None and out.shape == (B, S, H, D)
    out.backward(go)
    assert mix.grad is not None and mix.grad.shape == mix.shape and mix.grad.dtype == dt
    m = mix.detach()
    q, k, v = m[:, :, :, :G].reshape(B, S, H, D), m[:, :, :, G], m[:, :, :, G + 1]
    ro, _, rdq, rdk, rdv = _reference(q, k, v, go, True, D ** -0.5, None, 0.0)
    bound = 2e-3 if dt == F16 else 1.5e-2
    assert _rel(out, ro) < bound
    ref_grad = torch.cat([rdq.view(B, S, Hkv, G, D), rdk.unsqueeze(3), rdv.unsqueeze(3)], 3)
    assert _rel(mix.grad, ref_grad) < 2.5 * bound
    qa, ka, va = (t.clone().requires_grad_(True) for t in (q, k, v))
    out2 = ATT.attention(qa, ka, va, causal=True)
    out2.backward(go)
    assert torch.equal(out2, out)
    assert _rel(qa.grad, rdq) < 2.5 * bound and _rel(ka.grad, rdk) < 2.5 * bound and _rel(va.grad, rdv) < 2.5 * bound


def _decode_ref(q, k, v, mask, scale):
    g = q.shape[2] // k.shape[2]
    k, v = k.float().repeat_interleave(g, 2), v.float().repeat_interleave(g, 2)
    s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k) * scale + mask.reshape(q.shape[0], 1, 1, -1).float()
    return torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v)


@pytest.mark.parametrize("G", [1, 4, 8])
@pytest.mark.parametrize("D", [64, 128])
def test_decode_grouped_kv(G, D):
    torch.manual_seed(5)
    B, H, L = 3, 8, 700
    Hkv = H // G
    scale = D ** -0.5
    for dt in (B16, F16):
        q = torch.randn(B, 1, H, D, device="cuda", dtype=dt)
        kc = torch.randn(B, L, Hkv, D, device="cuda", dtype=dt)
        vc = torch.randn(B, L, Hkv, D, device="cuda", dtype=dt)
        valid = torch.rand(B, L, device="cuda") > 0.2
        valid[:, 0] = True
        mask = torch.where(valid, 0.0, -1e4).to(dt)
        out = OF.attention_decode(q, kc, vc, mask, scale)
        assert _rel(out, _decode_ref(q, kc, vc, mask, scale)) < 1e-2
        # packed step: qkv [B, 1, Hkv, G + 2, D]; the new K/V land at write_idx and every query head attends to them
        pos = 517
        qkv = torch.randn(B, 1, Hkv, G + 2, D, device="cuda", dtype=dt)
        k2, v2 = kc.clone(), vc.clone()
        want_k, want_v = kc.clone(), vc.clone()
        want_k[:, pos], want_v[:, pos] = qkv[:, 0, :, G], qkv[:, 0, :, G + 1]
        o2 = OF.attention_decode_packed(qkv, k2, v2, mask, torch.tensor([pos], device="cuda"), scale)
        torch.cuda.synchronize()
        assert torch.equal(k2, want_k) and torch.equal(v2, want_v)
        qf = qkv[:, :, :, :G].reshape(B, 1, H, D)
        assert _rel(o2, _decode_ref(qf, want_k, want_v, mask, scale)) < 1e-2


# ---------------------------------------------------------------------------------------------------------------- GPT
def _gpt_cfg(extra=()):
    from test_gpu_models import CFG, SMALL_GPT
    from paddlefleetx_b200.utils import config as C

    return C.get_config(os.path.join(CFG, "nlp/gpt/pretrain_gpt_345M_single_card.yaml"), SMALL_GPT + list(extra), nranks=1)


def _reset_tp():
    from paddlefleetx_b200.parallel import tp_layers as _tp
    _tp.configure({})


@pytest.mark.parametrize("kv", [2, 1])
def test_gqa_gpt_trains_without_library_kernels(kv, monkeypatch):
    from test_gpu_models import _engine, _gpt_batches

    def refuse(name):
        def f(*a, **k):
            raise AssertionError(f"torch.nn.functional.{name} was called")
        return f
    monkeypatch.setattr(torch.nn.functional, "linear", refuse("linear"))
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", refuse("scaled_dot_product_attention"))
    cfg = _gpt_cfg([f"Model.num_key_value_heads={kv}"])
    eng = _engine(cfg)
    attn = eng._module.model.gpt.decoder.layers[0].self_attn
    assert (attn.local_heads, attn.local_kv_heads) == (4, kv)
    batch = _gpt_batches(cfg, 1)[0]
    OF.reset_launch_count()
    losses = [float(eng.train_step(batch)) for _ in range(12)]
    assert OF.native_launch_count() > 100
    assert np.isfinite(losses).all() and losses[-1] < losses[0] - 0.3, losses
    _reset_tp()


_COPY = re.compile(r"copy|cat|memcpy|memset|gather|index", re.I)


def _copy_kernels_per_step(extra):
    from test_gpu_models import _engine, _gpt_batches

    cfg = _gpt_cfg(extra)
    eng = _engine(cfg)
    batch = _gpt_batches(cfg, 1)[0]
    eng.train_step(batch)
    eng.train_step(batch)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.train_step(batch)
        torch.cuda.synchronize()
    _reset_tp()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sorted(n for n in names if _COPY.search(n))


def test_gqa_step_launches_no_extra_copies():
    mha = _copy_kernels_per_step([])
    for kv in (2, 1):
        gqa = _copy_kernels_per_step([f"Model.num_key_value_heads={kv}"])
        assert len(gqa) <= len(mha), (kv, gqa, mha)


@pytest.mark.parametrize("kv", [2, 1])
def test_gqa_generation_graph_eager_and_recompute_agree(kv):
    from paddlefleetx_b200.models.language_model.gpt import model as gpt
    from paddlefleetx_b200.models.language_model.gpt.generation import GPTForGeneration

    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=1024, hidden_size=256, num_layers=2, num_attention_heads=4, ffn_hidden_size=1024, max_position_embeddings=128,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, num_key_value_heads=kv, dtype=B16, device="cuda")
    assert core.new_caches(1, 8)[0].k.shape[2] == kv
    cfg = dict(max_dec_len=10, decode_strategy="greedy_search", eos_token_id=None, pad_token_id=0)
    eager = GPTForGeneration(core, dict(cfg, use_cuda_graph=False))
    graph = GPTForGeneration(core, dict(cfg, use_cuda_graph=True))
    for bs in (1, 3, 12):
        ids = torch.randint(1, 1000, (bs, 9), device="cuda")
        a, _ = eager.generate(ids)
        b, _ = graph.generate(ids)
        c, _ = graph.generate(ids)
        assert torch.equal(b, c)
        assert (a == b).float().mean() > 0.9, (a, b)       # bf16 ties may flip an argmax; sequences must essentially agree
        seq = ids
        with torch.no_grad():
            for _ in range(a.shape[1]):
                h = core(seq)[:, -1]
                seq = torch.cat([seq, (h @ core.embeddings.word_embeddings.weight.t()).argmax(-1, keepdim=True)], 1)
        assert (seq[:, ids.shape[1]:] == a).float().mean() > 0.9, (seq, a)
