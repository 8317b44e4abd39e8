"""The attention kernels against float64, element by element (needs an H100).

Flash forward / backward (bf16 and fp16, D 64 and 128, causal and full, ragged and long rows, rows whose maximum moves into every later key
tile, dropout, grouped K/V heads, packed / sequence-major / grouped-packed views), the single-query decode kernel and its packed form with
the cache append, and the Evoformer gated attention forward / backward (bf16).  References and bounds come from ``kernel_refs`` (see the
attention section of its docstring); ``test_attention_tolerances_cpu.py`` shows on the same inputs that the bounds reject the plausible
mistakes.  Each 16-bit case runs in both dtypes on the same masters and the fp16 error must be well under the bf16 one.

Run with ``-s`` to print the largest error/bound ratio seen per kernel and dtype.
"""
import math
from collections import defaultdict

import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import attention as ATT
from paddlefleetx_b200.ops import evoformer_attention as EA

pytestmark = pytest.mark.gpu

F16, B16, F32 = torch.float16, torch.bfloat16, torch.float32
DTYPES = [B16, F16]
RATIOS = defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(RATIOS, key=str):
        print(f"max error/bound {key[0]:<24} {str(key[1]):<15} {RATIOS[key]:.3f}")


def _lib():
    return _native.require()


def _close(kernel, got, ref, dtype, kw, check_dtype=None):
    r = R.assert_close(got, ref, check_dtype or dtype, what=kernel, **kw)
    RATIOS[(kernel, dtype)] = max(RATIOS[(kernel, dtype)], r)
    return R.rel_err(got, ref) if float(ref.norm()) > 0 else None        # an exact zero (a one-key row's dq) has no relative error


def _fp16_closer(errs, what):
    """errs: {dtype: [relative errors of the same results on the same masters]}."""
    for i, (e16, eb) in enumerate(zip(errs[F16], errs[B16])):
        assert e16 is None or e16 <= 0.5 * eb, (what, i, "fp16 is not closer to the reference than bf16", errs)


def _nan_like(t):
    return torch.full_like(t, math.nan)


# ================================================================================================================ flash
FLASH_SHAPES = [(1, 1, False), (1, 300, True), (63, 63, False), (64, 64, True), (65, 65, False), (127, 129, True), (129, 257, True),
                (200, 1000, True), (257, 257, False), (1000, 1000, True)]


def _flash_case(kernel, B, Sq, Sk, H, D, causal, Hkv=None, p=0.0, rising=False, seed=0):
    """Bindings directly: forward, then backward into NaN-filled gradients; every output against float64 in both dtypes."""
    masters = R.attention_inputs(B, Sq, Sk, H, D, Hkv, seed=seed, rising=rising, device="cuda")
    scale = D ** -0.5
    dseed = 0x5EED + Sq
    keep = ATT.attn_keep_mask(dseed, B, H, Sq, Sk, p, "cuda") if p > 0 else None
    errs = {}
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        out, lse = _lib().attention_fwd_v2(q, k, v, causal, scale, p, dseed)
        dq, dk, dv = _nan_like(q), _nan_like(k), _nan_like(v)
        _lib().attention_bwd(q, k, v, out, do, lse, dq, dk, dv, causal, scale, p, dseed)
        ref, ref_lse = R.attention(q, k, v, scale, causal, keep, p)
        okw, lkw = R.attention_bounds(q, k, v, scale, causal, dt, keep, p)
        errs[dt] = [_close(kernel + " out", out, ref, dt, okw)]
        _close(kernel + " lse", lse, ref_lse, dt, lkw, check_dtype=F32)
        grads = R.attention_bwd(q, k, v, do, scale, causal, keep, p)
        bkw = R.attention_bwd_bounds(q, k, v, do, scale, causal, dt, keep, p)
        errs[dt] += [_close(f"{kernel} {n}", g, r, dt, kw) for n, g, r, kw in zip(("dq", "dk", "dv"), (dq, dk, dv), grads, bkw)]
    _fp16_closer(errs, (kernel, B, Sq, Sk, H, D, causal, Hkv, p))


@pytest.mark.parametrize("D", [64, 128])
@pytest.mark.parametrize("Sq,Sk,causal", FLASH_SHAPES)
def test_flash_attention_against_float64(Sq, Sk, causal, D):
    _flash_case("flash", 2, Sq, Sk, 3, D, causal)


@pytest.mark.parametrize("D", [64, 128])
def test_flash_attention_long_rows_with_a_moving_maximum(D):
    """4096 keys: 32 rescales per row, and the row maximum moves into every later key tile."""
    _flash_case("flash long", 1, 4096, 4096, 2, D, True, rising=True)


@pytest.mark.parametrize("D", [64, 128])
def test_flash_attention_moving_maximum(D):
    _flash_case("flash rising", 2, 1000, 1000, 3, D, False, rising=True)


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_flash_attention_dropout_against_float64(p):
    _flash_case("flash dropout", 2, 200, 1000, 3, 64, True, p=p)


@pytest.mark.parametrize("Hkv,D", [(2, 64), (1, 128)])
def test_flash_attention_grouped_heads_against_float64(Hkv, D):
    _flash_case("flash gqa", 2, 129, 257, 4, D, True, Hkv=Hkv)


@pytest.mark.parametrize("layout", ["packed", "seq_major"])
def test_flash_attention_packed_views_against_float64(layout):
    """q / k / v as slices of one [b, s, h, 3, d] tensor, in batch-major and sequence-major storage, gradients into NaN-filled views."""
    B, S, H, D = 2, 257, 3, 128
    masters = R.attention_inputs(B, S, S, H, D, seed=1, device="cuda")
    errs = {}
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        mix = torch.stack([q, k, v], dim=3)
        dmix = _nan_like(mix)
        if layout == "seq_major":
            mix = mix.transpose(0, 1).contiguous().transpose(0, 1)
            dmix = _nan_like(mix.transpose(0, 1)).transpose(0, 1)
        qv, kv, vv = mix.unbind(3)
        out, lse = _lib().attention_fwd_v2(qv, kv, vv, True, D ** -0.5, 0.0, 0)
        dq, dk, dv = dmix.unbind(3)
        _lib().attention_bwd(qv, kv, vv, out, do, lse, dq, dk, dv, True, D ** -0.5, 0.0, 0)
        ref, _ = R.attention(q, k, v, D ** -0.5, True)
        okw, _ = R.attention_bounds(q, k, v, D ** -0.5, True, dt)
        errs[dt] = [_close("flash " + layout, out, ref, dt, okw)]
        grads = R.attention_bwd(q, k, v, do, D ** -0.5, True)
        bkw = R.attention_bwd_bounds(q, k, v, do, D ** -0.5, True, dt)
        errs[dt] += [_close(f"flash {layout} grad", g, r, dt, kw) for g, r, kw in zip((dq, dk, dv), grads, bkw)]
    _fp16_closer(errs, layout)


@pytest.mark.parametrize("G", [2, 4])
def test_flash_attention_packed_grouped_front_end(G):
    """``flash_attention_packed`` on a [b, s, 1, G + 2, d] grouped projection: one packed gradient."""
    B, S, D = 2, 200, 64
    masters = R.attention_inputs(B, S, S, G, D, 1, seed=2, device="cuda")
    errs = {}
    for dt in DTYPES:
        q, k, v, do = (m.to(dt) for m in masters)
        mix = torch.cat([q.view(B, S, 1, G, D), k.view(B, S, 1, 1, D), v.view(B, S, 1, 1, D)], dim=3).requires_grad_(True)
        out = ATT.flash_attention_packed(mix, causal=True)
        out.backward(do)
        ref, _ = R.attention(q, k, v, D ** -0.5, True)
        okw, _ = R.attention_bounds(q, k, v, D ** -0.5, True, dt)
        errs[dt] = [_close("flash grouped packed", out, ref, dt, okw)]
        grads = R.attention_bwd(q, k, v, do, D ** -0.5, True)
        bkw = R.attention_bwd_bounds(q, k, v, do, D ** -0.5, True, dt)
        got = (mix.grad[:, :, :, :G].reshape(B, S, G, D), mix.grad[:, :, :, G], mix.grad[:, :, :, G + 1])
        errs[dt] += [_close("flash grouped packed grad", g, r, dt, kw) for g, r, kw in zip(got, grads, bkw)]
    _fp16_closer(errs, G)


def test_flash_attention_front_end():
    B, S, H, D = 2, 129, 3, 128
    masters = R.attention_inputs(B, S, S, H, D, seed=3, device="cuda")
    for dt in DTYPES:
        q, k, v, do = (m.to(dt).requires_grad_(True) for m in masters)
        out = ATT.attention(q, k, v, causal=True)
        out.backward(do)
        ref, _ = R.attention(q, k, v, D ** -0.5, True)
        okw, _ = R.attention_bounds(q, k, v, D ** -0.5, True, dt)
        _close("attention front end", out, ref, dt, okw)
        grads = R.attention_bwd(q, k, v, do, D ** -0.5, True)
        for g, r, kw in zip((q.grad, k.grad, v.grad), grads, R.attention_bwd_bounds(q, k, v, do, D ** -0.5, True, dt)):
            _close("attention front end grad", g, r, dt, kw)


# ================================================================================================================ decode
def _pad_mask(B, Lmax, fill, dt):
    mask = torch.zeros(B, Lmax, device="cuda")
    mask[1, : Lmax // 3] = fill                         # left padding of the second sequence
    return mask.to(dt)


@pytest.mark.parametrize("fill", [-1e4, -math.inf], ids=["pad_1e4", "neg_inf"])
@pytest.mark.parametrize("Lmax", [1, 7, 9, 136, 1000, 4097])
@pytest.mark.parametrize("D,G", [(64, 1), (128, 4), (64, 8), (128, 1)])
def test_decode_against_float64(D, G, Lmax, fill):
    B, Hkv = 2, 2
    masters = R.attention_inputs(B, 1, Lmax, Hkv * G, D, Hkv, seed=Lmax, device="cuda")
    errs = {}
    for dt in DTYPES:
        q, k, v = (m.to(dt) for m in masters[:3])
        mask = _pad_mask(B, Lmax, fill, dt)
        errs[dt] = []
        for L in sorted({Lmax, max(1, Lmax - 5)}):
            out = _lib().attention_decode(q, k, v, mask, L, D ** -0.5)
            ref = R.attention_decode(q, k, v, mask, L, D ** -0.5)
            errs[dt].append(_close("decode", out, ref, dt, R.attention_decode_bound(q, k, v, mask, L, D ** -0.5)))
    if Lmax > 1:
        _fp16_closer(errs, (D, G, Lmax))


def test_decode_neg_inf_on_every_key_returns_zero():
    """Every key masked with -inf: 0, the flash kernels' l = 0 convention (no NaN)."""
    for D, G in ((64, 1), (128, 4)):
        q, k, v = (m.to(B16) for m in R.attention_inputs(1, 1, 300, 2 * G, D, 2, device="cuda")[:3])
        out = _lib().attention_decode(q, k, v, torch.full((1, 300), -math.inf, device="cuda", dtype=B16), 300, D ** -0.5)
        assert torch.equal(out, torch.zeros_like(out))


@pytest.mark.parametrize("Lmax,pos", [(9, 0), (136, 70), (1000, 999)])
@pytest.mark.parametrize("D,G", [(64, 1), (128, 4), (64, 8)])
def test_decode_packed_appends_and_attends(D, G, Lmax, pos):
    """The cache row at write_idx becomes this step's K / V bit for bit, every other row is untouched, and the output attends over the
    appended cache (rows past write_idx masked, as the model does)."""
    B, Hkv = 2, 2
    masters = R.attention_inputs(B, 1, Lmax, Hkv * G, D, Hkv, seed=pos, device="cuda")
    k_new, v_new = R.decode_new_kv(masters[0], Hkv, seed=pos)
    for dt in DTYPES:
        q, k, v = (m.to(dt) for m in masters[:3])
        kn, vn = k_new.to(dt), v_new.to(dt)
        qkv = torch.cat([q.view(B, 1, Hkv, G, D), kn.view(B, 1, Hkv, 1, D), vn.view(B, 1, Hkv, 1, D)], dim=3).contiguous()
        mask = torch.zeros(B, Lmax, device="cuda")
        mask[:, pos + 1:] = -1e4
        mask = mask.to(dt)
        kc, vc = k.clone(), v.clone()
        out = _lib().attention_decode_packed(qkv, kc, vc, mask, torch.tensor([pos], device="cuda"), D ** -0.5)
        torch.cuda.synchronize()
        assert torch.equal(kc[:, pos], kn) and torch.equal(vc[:, pos], vn)
        others = torch.arange(Lmax, device="cuda") != pos
        assert torch.equal(kc[:, others], k[:, others]) and torch.equal(vc[:, others], v[:, others])
        k2, v2 = k.clone(), v.clone()
        k2[:, pos], v2[:, pos] = kn, vn
        ref = R.attention_decode(q, k2, v2, mask, Lmax, D ** -0.5)
        _close("decode packed", out, ref, dt, R.attention_decode_bound(q, k2, v2, mask, Lmax, D ** -0.5))
    # no fp16-closer check here: the appended key carries nearly all the weight, so O is close to one 16-bit V row in both dtypes


# ================================================================================================================ Evoformer
EVO_SHAPES = [(1, 1), (63, 65), (128, 128), (129, 257), (300, 77), (96, 96)]
# (H, G, gpp, mask, pair, gate): every head count, gpp in {1, 3, G}, each operand on and off
EVO_OPTS = [(2, 3, 1, True, True, True), (4, 3, 3, True, True, False), (8, 6, 3, False, True, True), (4, 6, 6, True, True, True),
            (2, 2, 1, False, False, False), (8, 3, 1, True, False, True)]


def _evo_run(q, k, v, mb, pb, gate, do, gpp, scale):
    out, stats = _lib().evoformer_attention_fwd(q, k, v, mb, pb, gate, gpp, scale)
    grads = _lib().evoformer_attention_bwd(q, k, v, out, do, stats, mb, pb, gate, gpp, scale, pb is not None)
    return out, grads


def _evo_check(kernel, got_out, grads, ins, gpp, scale, uniform=None, dpair_dtype=F32):
    q, k, v, mb, pb, gate, do = ins
    ref = R.evoformer(q, k, v, mb, pb, gate, gpp, scale, uniform)
    kws = R.evoformer_bounds(q, k, v, mb, pb, gate, gpp, scale, do, uniform)
    _close(kernel + " out", got_out, ref, B16, kws[0])
    rg = R.evoformer_bwd(q, k, v, mb, pb, gate, gpp, scale, do, uniform)
    for name, g, r, kw in zip(("dq", "dk", "dv"), grads[:3], rg[:3], kws[1:4]):
        _close(f"{kernel} {name}", g, r, B16, kw)
    if gate is not None:
        _close(kernel + " dgate", grads[3], rg[3], B16, kws[4])
    if pb is not None and grads[4] is not None and grads[4].numel():
        _close(kernel + " dpair", grads[4], rg[4], B16, kws[5], check_dtype=dpair_dtype)


def _evo_inputs(G, Sq, Sk, H, gpp, wm, wp, wg, seed=0):
    ms = R.evoformer_inputs(G, Sq, Sk, H, gpp, wm, wp, wg, seed=seed, device="cuda")
    return [None if t is None else (t if i == 3 else t.to(B16)) for i, t in enumerate(ms)]


@pytest.mark.parametrize("opts", EVO_OPTS, ids=lambda o: "H{}_G{}_gpp{}{}{}{}".format(*o[:3], "_mask" * o[3], "_pair" * o[4], "_gate" * o[5]))
@pytest.mark.parametrize("Sq,Sk", EVO_SHAPES)
def test_evoformer_against_float64(Sq, Sk, opts):
    H, G, gpp, wm, wp, wg = opts
    ins = _evo_inputs(G, Sq, Sk, H, gpp, wm, wp, wg, seed=Sq + Sk)
    q, k, v, mb, pb, gate, do = ins
    out, grads = _evo_run(q, k, v, mb, pb, gate, do, gpp, 32 ** -0.5)
    _evo_check("evoformer", out, grads, ins, gpp, 32 ** -0.5)


@pytest.mark.parametrize("bwd", ["native", "torch", "mask_grad"])
def test_evoformer_front_end(bwd, monkeypatch):
    """``evoformer_attention`` with its native backward, the chunked torch backward, and the path taken when the mask bias needs a gradient."""
    G, Sq, Sk, H, gpp = 6, 129, 77, 4, 3
    ins = _evo_inputs(G, Sq, Sk, H, gpp, True, True, True, seed=7)
    q, k, v, mb, pb, gate, do = ins
    if bwd == "torch":
        monkeypatch.setattr(EA, "_BWD", "torch")
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v, pb, gate)]
    mbl = mb.clone().requires_grad_(bwd == "mask_grad")
    out = EA.evoformer_attention(leaves[0], leaves[1], leaves[2], mbl, leaves[3], leaves[4], gpp, 32 ** -0.5)
    out.backward(do)
    grads = (leaves[0].grad, leaves[1].grad, leaves[2].grad, leaves[4].grad, leaves[3].grad)
    _evo_check("evoformer " + bwd, out, grads, ins, gpp, 32 ** -0.5, dpair_dtype=B16)       # the front end returns dpair in the bias dtype


@pytest.mark.parametrize("bwd", ["native", "torch"])
def test_evoformer_fully_masked_groups(bwd, monkeypatch):
    """Groups whose every key carries the model's -1e9: the fp32 contract (kernels and ``EA.reference``) is the gated mean of V, with the
    softmax derivative taken at those uniform probabilities.  float64 would keep the scores; the general bound is not loosened for it."""
    G, Sq, Sk, H, gpp = 4, 63, 96, 4, 2
    ins = _evo_inputs(G, Sq, Sk, H, gpp, True, True, True, seed=11)
    q, k, v, mb, pb, gate, do = ins
    mb[1] = -1e9
    mb[2] = -1e9
    uniform = torch.tensor([False, True, True, False], device="cuda")
    if bwd == "torch":
        monkeypatch.setattr(EA, "_BWD", "torch")
    leaves = [t.clone().requires_grad_(True) for t in (q, k, v, pb, gate)]
    out = EA.evoformer_attention(leaves[0], leaves[1], leaves[2], mb, leaves[3], leaves[4], gpp, 32 ** -0.5)
    out.backward(do)
    mean = (v.double().mean(1, keepdim=True) * torch.sigmoid(gate.double()))[1:3]
    kw = R.evoformer_bounds(q, k, v, mb, pb, gate, gpp, 32 ** -0.5, uniform=uniform)
    R.assert_close(out[1:3], mean, B16, scale=kw["scale"][1:3], approx=1.0, what="fully masked: gated mean of V")
    grads = (leaves[0].grad, leaves[1].grad, leaves[2].grad, leaves[4].grad, leaves[3].grad)
    _evo_check("evoformer fully masked", out, grads, ins, gpp, 32 ** -0.5, uniform, dpair_dtype=B16)
