"""Intra-document causal attention (``DocumentMask``) on the sm_90a flash kernels (needs an H100).

Forward (out, lse) and backward (dq, dk, dv) against float64 within the ``kernel_refs`` bounds (``doc_attention_refs``: the same budgets under the mask) for bf16 and fp16, D 64 / 128, G 1 / 4,
dropout, and packed / sequence-major / grouped-packed views, with gradients written into NaN-filled buffers; documents of 1, 63, 64, 65,
127, 128, 129 tokens and random mixes.  With every key_start = 0 the kernels must reproduce the causal kernels bit for bit (dq up to its
reduction order), and a document's results must not change by a single bit when the other documents' q / k / v do.  Then the GPT
training step with ``reset_attention_mask`` (no SDPA, no F.linear, one bounds launch per step) and left-padded generation prefill.

Run with ``-s`` to print the largest error/bound ratio seen per kernel and dtype.
"""
import math
from collections import defaultdict

import numpy as np
import pytest
import torch

import doc_attention_refs as DR
import kernel_refs as R
from paddlefleetx_b200.data.dataset.gpt_dataset import document_positions
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import attention as ATT

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16
DTYPES = [B16, F16]
RATIOS = defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(RATIOS, key=str):
        print(f"max error/bound {key[0]:<28} {str(key[1]):<15} {RATIOS[key]:.3f}")


def _lib():
    return _native.require()


def _close(kernel, got, ref, dtype, kw):
    RATIOS[(kernel, dtype)] = max(RATIOS[(kernel, dtype)], R.assert_close(got, ref, dtype, what=kernel, **kw))


def _nan_like(t):
    return torch.full_like(t, math.nan)


def _positions(B, S, lengths, seed=0):
    """[B, S] position ids: ``lengths`` a document length repeated along the rows, or "mix" for random lengths per row."""
    rng = np.random.default_rng(seed)
    rows = []
    for b in range(B):
        if lengths == "mix":
            lens = rng.integers(1, 300, size=S).tolist()
        else:
            lens = [lengths] * (S // lengths + 1)
        rows.append(document_positions(lens, S))
    return torch.tensor(np.stack(rows), device="cuda")


def _doc_case(kernel, B, S, H, D, Hkv, lengths, p=0.0, seed=0):
    masters = R.attention_inputs(B, S, S, H, D, Hkv, seed=seed, device="cuda")
    pos = _positions(B, S, lengths, seed)
    doc = ATT.DocumentMask.from_positions(pos)
    for a, b in zip(doc.bounds(), ATT.DocumentMask.from_positions(pos.cpu()).bounds()):
        assert torch.equal(a.cpu(), b), "native bounds differ from the CPU derivation"
    mask = doc.dense()[:, 0]
    scale = D ** -0.5
    dseed = 0xD0C + S
    keep = ATT.attn_keep_mask(dseed, B, H, S, S, p, "cuda") if p > 0 else None
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        out, lse = _lib().attention_fwd_doc(q, k, v, *doc.bounds(), scale, p, dseed)
        dq, dk, dv = _nan_like(q), _nan_like(k), _nan_like(v)
        _lib().attention_bwd_doc(q, k, v, out, do, lse, dq, dk, dv, *doc.bounds(), scale, p, dseed)
        ref, ref_lse = DR.attention(q, k, v, scale, mask, keep, p)
        okw, lkw = DR.attention_bounds(q, k, v, scale, mask, dt, keep, p)
        _close(kernel + " out", out, ref, dt, okw)
        RATIOS[(kernel + " lse", dt)] = max(RATIOS[(kernel + " lse", dt)], R.assert_close(lse, ref_lse, torch.float32, what=kernel, **lkw))
        grads = DR.attention_bwd(q, k, v, do, scale, mask, keep, p)
        bkw = DR.attention_bwd_bounds(q, k, v, do, scale, mask, dt, keep, p)
        for n, g, r, kw in zip(("dq", "dk", "dv"), (dq, dk, dv), grads, bkw):
            _close(f"{kernel} {n}", g, r, dt, kw)


@pytest.mark.parametrize("lengths", [1, 63, 64, 65, 127, 128, 129, "mix"])
@pytest.mark.parametrize("D,Hkv", [(64, 4), (128, 4), (64, 1), (128, 1)])
def test_doc_attention_against_float64(lengths, D, Hkv):
    _doc_case("doc" if Hkv == 4 else "doc gqa", 2, 300, 4, D, Hkv, lengths)


def test_doc_attention_long_rows_against_float64():
    _doc_case("doc long", 1, 2048, 2, 128, 2, "mix", seed=3)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_doc_attention_dropout_against_float64(p):
    _doc_case("doc dropout", 2, 300, 4, 64, 4, "mix", p=p, seed=1)


@pytest.mark.parametrize("layout", ["packed", "seq_major", "grouped_packed"])
def test_doc_attention_views_against_float64(layout):
    """``flash_attention_packed`` with a document mask on a [b, s, h, 3, d] projection (batch- or sequence-major storage) or its grouped
    [b, s, 1, G + 2, d] form: q / k / v read in place, one packed gradient."""
    B, S, D = 2, 257, 128
    G = 4 if layout == "grouped_packed" else 1
    H = G if layout == "grouped_packed" else 3
    masters = R.attention_inputs(B, S, S, H, D, 1 if G > 1 else None, seed=2, device="cuda")
    doc = ATT.DocumentMask.from_positions(_positions(B, S, "mix", seed=2))
    mask = doc.dense()[:, 0]
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        if G > 1:
            mix = torch.cat([q.view(B, S, 1, G, D), k.view(B, S, 1, 1, D), v.view(B, S, 1, 1, D)], dim=3)
        else:
            mix = torch.stack([q, k, v], dim=3)
        if layout == "seq_major":
            mix = mix.transpose(0, 1).contiguous().transpose(0, 1)
        mix.requires_grad_(True)
        out = ATT.flash_attention_packed(mix, causal=True, doc=doc)
        assert out is not None
        out.backward(do)
        if G > 1:
            got = (mix.grad[:, :, :, :G].reshape(B, S, G, D), mix.grad[:, :, :, G], mix.grad[:, :, :, G + 1])
        else:
            got = mix.grad.unbind(3)
        ref, _ = DR.attention(q, k, v, D ** -0.5, mask)
        okw, _ = DR.attention_bounds(q, k, v, D ** -0.5, mask, dt)
        _close("doc " + layout, out, ref, dt, okw)
        grads = DR.attention_bwd(q, k, v, do, D ** -0.5, mask)
        bkw = DR.attention_bwd_bounds(q, k, v, do, D ** -0.5, mask, dt)
        for n, g, r, kw in zip(("dq", "dk", "dv"), got, grads, bkw):
            _close(f"doc {layout} {n}", g, r, dt, kw)


@pytest.mark.parametrize("D,Hkv", [(64, 4), (128, 4), (128, 1)])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_zero_key_start_is_the_causal_kernel(D, Hkv, p):
    """One document per row: out, lse, dk and dv bit-identical to the causal kernels; dq equal up to the order of its fp32 reduction."""
    B, S, H = 2, 333, 4
    masters = R.attention_inputs(B, S, S, H, D, Hkv, seed=4, device="cuda")
    doc = ATT.DocumentMask.from_key_start(torch.zeros(B, S, dtype=torch.long, device="cuda"))
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        o1, l1 = _lib().attention_fwd_v2(q, k, v, True, D ** -0.5, p, 11)
        o2, l2 = _lib().attention_fwd_doc(q, k, v, *doc.bounds(), D ** -0.5, p, 11)
        assert torch.equal(o1, o2) and torch.equal(l1, l2)
        g1 = [_nan_like(t) for t in (q, k, v)]
        g2 = [_nan_like(t) for t in (q, k, v)]
        _lib().attention_bwd(q, k, v, o1, do, l1, *g1, True, D ** -0.5, p, 11)
        _lib().attention_bwd_doc(q, k, v, o1, do, l1, *g2, *doc.bounds(), D ** -0.5, p, 11)
        assert torch.equal(g1[1], g2[1]) and torch.equal(g1[2], g2[2])
        torch.testing.assert_close(g1[0].float(), g2[0].float(), rtol=1e-2, atol=1e-3)


@pytest.mark.parametrize("D,Hkv", [(64, 4), (128, 1)])
def test_documents_are_isolated(D, Hkv):
    """Changing the q / k / v of every other document leaves a document's out, dk and dv bit-identical."""
    B, S, H = 2, 400, 4
    pos = _positions(B, S, "mix", seed=5)
    doc = ATT.DocumentMask.from_positions(pos)
    starts = (torch.arange(S, device="cuda") - pos)                     # document id of each token = its start index
    masters = R.attention_inputs(B, S, S, H, D, Hkv, seed=5, device="cuda")
    target = starts == starts[:, S // 2: S // 2 + 1]                  # the document holding the middle token of each row
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        res = []
        for perturb in (False, True):
            if perturb:
                noise = [torch.randn_like(t) for t in (q, k, v)]
                q2, k2, v2 = (torch.where(target[:, :, None, None], t, n) for t, n in zip((q, k, v), noise))
            else:
                q2, k2, v2 = q, k, v
            out, lse = _lib().attention_fwd_doc(q2, k2, v2, *doc.bounds(), D ** -0.5, 0.0, 0)
            dq, dk, dv = _nan_like(q2), _nan_like(k2), _nan_like(v2)
            _lib().attention_bwd_doc(q2, k2, v2, out, do, lse, dq, dk, dv, *doc.bounds(), D ** -0.5, 0.0, 0)
            sel = target[:, :, None, None]
            res.append([torch.where(sel, t, torch.zeros_like(t)) for t in (out, dk, dv)])
        for a, b in zip(*res):
            assert torch.equal(a, b)


def test_bounds_from_positions_clamp():
    pos = torch.tensor([[0, 1, 2, 0, 1, 9, 0, -3] + list(range(100))], device="cuda")
    doc = ATT.DocumentMask.from_positions(pos)
    cpu = ATT.DocumentMask.from_positions(pos.cpu())
    for a, b in zip(doc.bounds(), cpu.bounds()):
        assert torch.equal(a.cpu(), b)
    assert doc.key_start[0, :8].tolist() == [0, 0, 0, 3, 3, 0, 6, 7]


# ---------------------------------------------------------------------------------------------------------------- GPT
def _gpt(dtype, device, use_rope=False, kv=None):
    from paddlefleetx_b200.models.language_model.gpt import model as gpt

    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=1024, hidden_size=256, num_layers=2, num_attention_heads=4, ffn_hidden_size=1024, max_position_embeddings=256,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, use_rope=use_rope, num_key_value_heads=kv,
                        reset_attention_mask=True, dtype=dtype, device=device)
    return gpt.GPTForPretraining(core), gpt.GPTPretrainingCriterion()


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("use_rope,kv", [(False, None), (True, 2)])
def test_gpt_step_with_document_mask(monkeypatch, dtype, use_rope, kv):
    """One training step with 16-bit parameters (O2) runs on our kernels only and its loss matches the fp32 CPU dense path."""
    from paddlefleetx_b200.ops import functional as OF
    from paddlefleetx_b200.optims import FusedAdamW

    model, crit = _gpt(dtype, "cuda", use_rope, kv)
    ref_model, ref_crit = _gpt(torch.float32, "cpu", use_rope, kv)
    ref_model.load_state_dict({k: v.float().cpu() for k, v in model.state_dict().items()})
    tokens = torch.randint(0, 1024, (2, 257))
    x, y = tokens[:, :-1], tokens[:, 1:]
    pos = _positions(2, 256, "mix", seed=6).cpu()
    mask = torch.ones(2, 256)
    with torch.no_grad():
        want = float(ref_crit(ref_model(x, pos), y, mask))

    def refuse(name):
        def f(*a, **k):
            raise AssertionError(f"torch.nn.functional.{name} was called")
        return f
    monkeypatch.setattr(torch.nn.functional, "linear", refuse("linear"))
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", refuse("scaled_dot_product_attention"))
    opt = FusedAdamW(1e-3, named_parameters=list(model.named_parameters()), multi_precision=True)
    OF.reset_launch_count()
    loss = crit(model(x.cuda(), pos.cuda()), y.cuda(), mask.cuda())
    loss.backward()
    opt.step()
    opt.clear_grad()
    assert OF.native_launch_count() > 0
    assert abs(float(loss) - want) < 2e-2 * abs(want), (float(loss), want)
    assert all(torch.isfinite(p).all() for p in model.parameters())


def test_gpt_step_adds_one_bounds_launch_and_no_library_kernel():
    def kernels(flag):
        model, crit = _gpt(B16, "cuda")
        model.gpt.reset_attention_mask = flag
        tokens = torch.randint(0, 1024, (2, 257), device="cuda")
        pos = _positions(2, 256, 100, seed=7)
        args = (tokens[:, :-1], pos)
        crit(model(*args), tokens[:, 1:], torch.ones(2, 256, device="cuda")).backward()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            crit(model(*args), tokens[:, 1:], torch.ones(2, 256, device="cuda")).backward()
            torch.cuda.synchronize()
        return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]

    on, off = kernels(True), kernels(False)
    assert sum("attn_doc_bounds_kernel" in n for n in on) == 1, sorted(set(on))
    other = lambda names: sorted(n for n in names if "attn_doc_bounds_kernel" not in n and "attention_" not in n)
    assert other(on) == other(off), (set(other(on)) ^ set(other(off)))


def test_left_padded_generation_prefill_is_native(monkeypatch):
    from paddlefleetx_b200.models.language_model.gpt import model as gpt
    from paddlefleetx_b200.models.language_model.gpt.generation import GPTForGeneration, _left_padded_mask, _to_additive

    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=1024, hidden_size=256, num_layers=2, num_attention_heads=4, ffn_hidden_size=1024, max_position_embeddings=128,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, dtype=B16, device="cuda").eval()
    b, s = 3, 40
    ids = torch.randint(1, 1000, (b, s), device="cuda")
    valid = torch.ones(b, s, dtype=torch.bool, device="cuda")
    valid[1, :7] = False
    valid[2, :33] = False
    ids[~valid] = 0
    pos = (valid.long().cumsum(-1) - 1).clamp(min=0)
    causal = torch.ones(s, s, dtype=torch.bool, device="cuda").tril()
    dense = ((causal.unsqueeze(0) & valid.unsqueeze(1)).unsqueeze(1)) | torch.eye(s, dtype=torch.bool, device="cuda")
    with torch.no_grad():
        want = core(ids, pos, _to_additive(dense, B16), core.new_caches(b, s + 4))
        doc = _left_padded_mask(valid)
        assert torch.equal(doc.dense(), dense)

        def refuse(*a, **k):
            raise AssertionError("scaled_dot_product_attention was called")
        monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", refuse)
        got = core(ids, pos, doc, core.new_caches(b, s + 4))
        monkeypatch.undo()
        gen = GPTForGeneration(core, dict(max_dec_len=4, decode_strategy="greedy_search", eos_token_id=None, pad_token_id=0))
        out, _ = gen.generate(ids)
    live = valid[:, :, None]
    torch.testing.assert_close(torch.where(live, got, 0).float(), torch.where(live, want, 0).float(), rtol=2e-2, atol=2e-2)
    assert out.shape == (b, 4)
