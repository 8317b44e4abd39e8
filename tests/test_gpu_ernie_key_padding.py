"""Bidirectional key padding (``KeyPaddingMask``) on the sm_90a flash kernels (needs an H100).

Forward (out, lse) and backward (dq, dk, dv) against float64 within the ``kernel_refs`` budgets for bf16 and fp16, D 64 / 128: valid lengths
1, 63, 64, 65, 127, 128, 129 and s, random interior patterns, all-padding rows, dropout (``attn_keep_mask``), gradients written into
NaN-filled buffers, contiguous and sequence-major views.  Padded keys carry exactly zero weight: other K / V there leave out and lse
bit-identical (dq up to its reduction order), and dk = dv = 0 there, also on key tiles past key_end.  With every bit set the kernels equal the plain non-causal ones bit
for bit (dq up to its reduction order).  The native bounds take one launch and match the CPU derivation.  Then ERNIE-base training steps
on padded batches: no SDPA, one bounds launch per step, and the loss and gradients of the unfused ``use_flash_attn: False`` path.
"""
import math

import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import attention as ATT
from test_gpu_ring_doc_attention import _attention, _attention_bwd, _bounds

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]


def _lib():
    return _native.require()


def _nan_like(t):
    return torch.full_like(t, math.nan)


def _mask(valid):
    pad = ATT.KeyPaddingMask.from_valid(valid.cuda())
    for a, b in zip(pad.bounds(), ATT.KeyPaddingMask.from_valid(valid.cpu()).bounds()):
        assert torch.equal(a.cpu(), b), "native bounds differ from the CPU derivation"
    return pad


def _check(tag, pad, masters, D, p=0.0, seed=0, views=lambda t: t):
    """Kernels against float64 for both dtypes; ``views`` maps a contiguous tensor to the layout the kernels read."""
    B, S, H = masters[0].shape[:3]
    scale = D ** -0.5
    mask = pad.dense()[:, 0].expand(B, S, S)
    keep = ATT.attn_keep_mask(seed, B, H, S, S, p, "cuda") if p > 0 else None
    for dt in DTYPES:
        q, k, v, do = (views(m.to(dt)) for m in masters)
        out, lse = _lib().attention_fwd_keypad(q, k, v, *pad.bounds(), scale, p, seed)
        dq, dk, dv = (views(_nan_like(t)) for t in (q, k, v))
        _lib().attention_bwd_keypad(q, k, v, out, do, lse, dq, dk, dv, *pad.bounds(), scale, p, seed)
        ref, ref_lse = _attention(q, k, v, scale, mask, keep, p)
        grads = _attention_bwd(q, k, v, do, scale, mask, keep, p)
        kws = _bounds(q, k, v, do, scale, mask, dt, keep, p)
        for n, got, want, kw, t in zip(("out", "lse", "dq", "dk", "dv"), (out, lse) + (dq, dk, dv), (ref, ref_lse) + tuple(grads), kws,
                                       (dt, torch.float32, dt, dt, dt)):
            R.assert_close(got, want, t, what=f"{tag} {n} {dt}", **kw)


def _right_padded(B, S, lengths):
    valid = torch.zeros(B, S, dtype=torch.bool)
    for b, n in enumerate(lengths):
        valid[b, :n] = True
    return valid


@pytest.mark.parametrize("length", [1, 63, 64, 65, 127, 128, 129, 300])
@pytest.mark.parametrize("D", [64, 128])
def test_right_padding_against_float64(length, D):
    B, S, H = 2, 300, 4
    masters = R.attention_inputs(B, S, S, H, D, seed=length, device="cuda")
    _check(f"len {length}", _mask(_right_padded(B, S, [length, S - length // 2])), masters, D)


@pytest.mark.parametrize("D", [64, 128])
def test_interior_patterns_and_empty_rows_against_float64(D):
    B, S, H = 4, 333, 2
    g = torch.Generator().manual_seed(D)
    valid = torch.rand(B, S, generator=g) > 0.4
    valid[1, 200:] = False
    valid[2] = False                                   # no valid key: attends every key
    valid[3, :] = False
    valid[3, [0, 130, 257]] = True
    masters = R.attention_inputs(B, S, S, H, D, seed=7, device="cuda")
    _check("interior", _mask(valid), masters, D)


@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("D", [64, 128])
def test_dropout_against_float64(p, D):
    B, S, H = 2, 260, 4
    valid = _right_padded(B, S, [190, 77])
    valid[0, 5:9] = False
    masters = R.attention_inputs(B, S, S, H, D, seed=3, device="cuda")
    _check(f"dropout {p}", _mask(valid), masters, D, p=p, seed=0x5EED + S)


@pytest.mark.parametrize("D", [64, 128])
def test_sequence_major_views_against_float64(D):
    """[s, b, h, d] storage read as [b, s, h, d] views, as under sequence parallelism."""
    B, S, H = 3, 200, 4
    masters = R.attention_inputs(B, S, S, H, D, seed=11, device="cuda")
    _check("seq-major", _mask(_right_padded(B, S, [200, 131, 40])), masters, D,
           views=lambda t: t.transpose(0, 1).contiguous().transpose(0, 1))


@pytest.mark.parametrize("D", [64, 128])
def test_autograd_path_against_float64(D):
    """``ATT.attention`` with a ``KeyPaddingMask``: native forward and backward, no SDPA."""
    B, S, H = 2, 192, 4
    pad = _mask(_right_padded(B, S, [192, 100]))
    masters = R.attention_inputs(B, S, S, H, D, seed=13, device="cuda")
    mask = pad.dense()[:, 0].expand(B, S, S)
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        qs, ks, vs = (t.clone().requires_grad_(True) for t in (q, k, v))
        out = ATT.attention(qs, ks, vs, causal=False, attn_mask=pad)
        out.backward(do)
        okw, _, qkw, kkw, vkw = _bounds(q, k, v, do, D ** -0.5, mask, dt)
        R.assert_close(out, _attention(q, k, v, D ** -0.5, mask)[0], dt, what="autograd out", **okw)
        for g, r, kw in zip((qs.grad, ks.grad, vs.grad), _attention_bwd(q, k, v, do, D ** -0.5, mask), (qkw, kkw, vkw)):
            R.assert_close(g, r, dt, what="autograd grad", **kw)


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_padded_keys_carry_zero_weight(D, p):
    """Other K / V at padded keys: out and lse bit-identical, dq up to the order of its reduction; dk = dv = 0 there, also on key tiles
    past key_end (rows 256-399)."""
    B, S, H = 2, 400, 4
    valid = _right_padded(B, S, [250, 130])
    valid[0, [3, 64, 200]] = False
    pad = _mask(valid)
    assert pad.key_end.tolist() == [250, 130]
    masters = R.attention_inputs(B, S, S, H, D, seed=17, device="cuda")
    inv = (~valid).cuda()[:, :, None, None]
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        res = []
        for perturb in (False, True):
            k2, v2 = k, v
            if perturb:
                k2, v2 = (torch.where(inv, torch.randn_like(t) * 4, t) for t in (k, v))
            out, lse = _lib().attention_fwd_keypad(q, k2, v2, *pad.bounds(), D ** -0.5, p, 99)
            dq, dk, dv = _nan_like(q), _nan_like(k), _nan_like(v)
            _lib().attention_bwd_keypad(q, k2, v2, out, do, lse, dq, dk, dv, *pad.bounds(), D ** -0.5, p, 99)
            assert not dq.isnan().any() and not dk.isnan().any() and not dv.isnan().any()
            inv_b = inv.expand_as(dk)
            assert torch.equal(dk[inv_b], torch.zeros_like(dk[inv_b])) and torch.equal(dv[inv_b], torch.zeros_like(dv[inv_b]))
            res.append((out, lse, dq))
        (o1, l1, dq1), (o2, l2, dq2) = res
        assert torch.equal(o1, o2) and torch.equal(l1, l2)
        torch.testing.assert_close(dq1.float(), dq2.float(), rtol=1e-2, atol=1e-3)      # fp32 reduce-adds across key tiles: any order


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("p", [0.0, 0.1])
def test_all_valid_is_the_non_causal_kernel(D, p):
    B, S, H = 2, 333, 4
    pad = _mask(torch.ones(B, S, dtype=torch.bool))
    masters = R.attention_inputs(B, S, S, H, D, seed=19, device="cuda")
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        o1, l1 = _lib().attention_fwd_v2(q, k, v, False, D ** -0.5, p, 23)
        o2, l2 = _lib().attention_fwd_keypad(q, k, v, *pad.bounds(), D ** -0.5, p, 23)
        assert torch.equal(o1, o2) and torch.equal(l1, l2)
        g1 = [_nan_like(t) for t in (q, k, v)]
        g2 = [_nan_like(t) for t in (q, k, v)]
        _lib().attention_bwd(q, k, v, o1, do, l1, *g1, False, D ** -0.5, p, 23)
        _lib().attention_bwd_keypad(q, k, v, o1, do, l1, *g2, *pad.bounds(), D ** -0.5, p, 23)
        assert torch.equal(g1[1], g2[1]) and torch.equal(g1[2], g2[2])
        torch.testing.assert_close(g1[0].float(), g2[0].float(), rtol=1e-2, atol=1e-3)


def _kernel_names(fn):
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


@pytest.mark.parametrize("dtype", [torch.bool, torch.int32, torch.int64, torch.float32, torch.float16, torch.bfloat16])
def test_native_bounds_in_one_launch(dtype):
    g = torch.Generator().manual_seed(1)
    valid = torch.rand(5, 1000, generator=g) > 0.5
    valid[1, 700:] = False
    valid[2] = False
    valid[3] = True
    src = valid.to(dtype).cuda()
    ATT.KeyPaddingMask.from_valid(src)
    names = _kernel_names(lambda: ATT.KeyPaddingMask.from_valid(src))
    assert len(names) == 1 and "attn_key_pad_bounds_kernel" in names[0], names
    _mask(valid.to(dtype))
    ids = torch.where(valid, torch.randint(1, 999, valid.shape, generator=g), torch.full_like(valid, 7, dtype=torch.long))
    a = ATT.KeyPaddingMask.from_ids(ids.cuda(), 7)
    for x, y in zip(a.bounds(), ATT.KeyPaddingMask.from_ids(ids, 7).bounds()):
        assert torch.equal(x.cpu(), y)


# ---------------------------------------------------------------------------------------------------------------- ERNIE
def _ernie_base(dtype, use_flash_attn):
    from paddlefleetx_b200.models.language_model.ernie import model as E

    torch.manual_seed(0)
    core = E.ErnieModel(vocab_size=8192, hidden_size=768, num_hidden_layers=4, num_attention_heads=12, intermediate_size=3072,
                        max_position_embeddings=512, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, use_flash_attn=use_flash_attn,
                        dtype=dtype, device="cuda")
    return E.ErnieForPretraining(core), E.ErniePretrainingCriterion()


def _ernie_batch(seed=0):
    g = torch.Generator().manual_seed(seed)
    b, s = 4, 256
    ids = torch.randint(1, 8192, (b, s), generator=g)
    lengths = [256, 190, 129, 40]
    mask = torch.zeros(b, s)
    for i, n in enumerate(lengths):
        mask[i, :n] = 1.0
    ids[mask == 0] = 0
    seg = torch.randint(0, 2, (b, s), generator=g)
    pos = torch.cat([torch.randperm(n, generator=g)[:10] + i * s for i, n in enumerate(lengths)])
    labels = torch.randint(0, 8192, (pos.numel(),), generator=g)
    nsp = torch.randint(0, 2, (b,), generator=g)
    return [t.cuda() for t in (ids, seg, mask, pos, labels, nsp)]


def _step(model, crit, batch):
    ids, seg, mask, pos, labels, nsp = batch
    scores, rel = model(ids, seg, None, mask, pos)
    loss = crit(scores, rel, labels, nsp)[0]
    loss.backward()
    return loss.detach()


@pytest.mark.parametrize("dtype", DTYPES)
def test_ernie_base_step_on_padded_batches(monkeypatch, dtype):
    """Loss within 1 % and every parameter gradient within 10 % (relative Frobenius norm) of the unfused path, with no SDPA call.  The
    two paths differ by 16-bit rounding only: the unfused one rounds the logits and P to the parameter dtype."""
    model, crit = _ernie_base(dtype, True)
    ref, _ = _ernie_base(dtype, False)
    ref.load_state_dict(model.state_dict())
    batch = _ernie_batch()
    want = _step(ref, crit, batch)

    def refuse(*a, **k):
        raise AssertionError("scaled_dot_product_attention was called")
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", refuse)
    got = _step(model, crit, batch)
    assert abs(float(got) - float(want)) < 1e-2 * abs(float(want)), (float(got), float(want))
    ref_grads = dict(ref.named_parameters())
    for n, p in model.named_parameters():
        g, r = p.grad.float(), ref_grads[n].grad.float()
        assert torch.isfinite(g).all(), n
        if n.endswith("k_proj.bias"):
            continue                  # adds one constant to every logit of a row: its exact gradient is 0, both paths give rounding noise
        assert (g - r).norm() <= 1e-1 * r.norm() + 1e-6, (n, float((g - r).norm() / r.norm()))


def test_ernie_step_adds_one_bounds_launch_and_no_library_attention():
    model, crit = _ernie_base(torch.bfloat16, True)
    batch = _ernie_batch(1)
    _step(model, crit, batch)
    names = _kernel_names(lambda: _step(model, crit, batch))
    assert sum("attn_key_pad_bounds_kernel" in n for n in names) == 1, sorted(set(names))
    assert sum("attention_fwd_kernel" in n for n in names) == 4 and sum("attention_bwd_kernel" in n for n in names) == 4
    assert not any("fmha" in n or "flash" in n.lower() or "efficient_attention" in n for n in names), sorted(set(names))
