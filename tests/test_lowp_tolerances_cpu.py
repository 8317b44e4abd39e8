"""The 8-bit checks in ``kernel_refs`` are tight enough to matter.

The correct result must pass each check and a result built with a plausible kernel mistake must fail it, in bf16 and fp16 inputs where
that applies.  The CPU fallbacks of ``ops/quant.py`` must pass the same checks.
"""
import math

import numpy as np
import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import quant as Q

DTYPES = [torch.bfloat16, torch.float16]


def _gen(seed=0):
    return torch.Generator().manual_seed(seed)


def _x(shape, dtype, seed=0):
    """rows with different magnitudes, so that every row has its own scale"""
    g = _gen(seed)
    x = torch.randn(shape, generator=g, dtype=torch.float64) * torch.exp2(torch.randint(-4, 5, (shape[0], 1), generator=g).double())
    return x.to(dtype)


def _smooth(cols, seed=1):
    return torch.exp(torch.empty(cols, dtype=torch.float64).uniform_(math.log(0.1), math.log(10.0), generator=_gen(seed))).float()


def _quant(x, smooth, fp8, qmax=None, div=True, mode="round"):
    """A float64 per-row quantiser with optional mistakes.  -> (q, scale)"""
    x64 = x.double()
    s = smooth.double() if smooth is not None else torch.ones(x.shape[-1], dtype=torch.float64)
    y = x64 / s if div else x64 * s
    qm = qmax or (448.0 if fp8 else 127.0)
    amax = y.abs().amax(-1)
    scale = torch.where(amax > 0, amax / qm, torch.ones_like(amax)).float()
    t = y / scale.double()[:, None]
    if fp8:
        return R.e4m3_rne(t).to(torch.float8_e4m3fn), scale
    r = torch.trunc(t) if mode == "trunc" else torch.round(t)
    return r.clamp(-128 if mode == "clamp128" else -127, 127).to(torch.int8), scale


def _rejects(x, smooth, q, scale, fp8):
    with pytest.raises(AssertionError):
        R.quantize_rows_check(x, smooth, q, scale, fp8)


# ---------------------------------------------------------------------------------------------------------------- quantize_rows
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("smoothed", [False, True])
def test_quantize_rows_check_accepts_exact_and_reference(dtype, fp8, smoothed):
    x = _x((33, 256), dtype)
    x[3] = 0
    sm = _smooth(256) if smoothed else None
    R.quantize_rows_check(x, sm, *_quant(x, sm, fp8), fp8)
    R.quantize_rows_check(x, sm, *Q.quantize_rows_reference(x, sm, fp8), fp8)


@pytest.mark.parametrize("dtype", DTYPES)
def test_quantize_rows_check_rejects_int8_mistakes(dtype):
    x, sm = _x((33, 256), dtype), _smooth(256)
    _rejects(x, sm, *_quant(x, sm, False, qmax=128.0), False)
    _rejects(x, sm, *_quant(x, sm, False, mode="trunc"), False)
    _rejects(x, sm, *_quant(x, sm, False, div=False), False)
    # amax / qmax taken before the smooth divide
    q, s = _quant(x, sm, False)
    _rejects(x, sm, q, x.double().abs().amax(-1).float() / 127.0, False)
    # the asymmetric int8 range: a row whose amax is negative reaches -128
    xn = x.clone()
    xn[:, 0] = -x.double().abs().amax(-1).to(dtype) * 2
    q, s = _quant(xn, None, False, qmax=127.0)
    s_asym = s * 127.0 / 128.0
    q = torch.round(xn.double() / s_asym.double()[:, None]).clamp(-128, 127).to(torch.int8)
    assert (q == -128).any()
    _rejects(xn, None, q, s_asym, False)


@pytest.mark.parametrize("dtype", DTYPES)
def test_quantize_rows_check_rejects_fp8_mistakes(dtype):
    x, sm = _x((33, 256), dtype), _smooth(256)
    _rejects(x, sm, *_quant(x, sm, True, qmax=127.0), True)
    _rejects(x, sm, *_quant(x, sm, True, div=False), True)
    # e4m3fnuz bytes (exponent bias 8) stored as e4m3fn
    q, s = _quant(x, sm, True)
    t = (x.double() / sm.double() / s.double()[:, None]).clamp(-240, 240).float()
    _rejects(x, sm, t.to(torch.float8_e4m3fnuz).view(torch.uint8).view(torch.float8_e4m3fn), s, True)


# ---------------------------------------------------------------------------------------------------------------- MX
def test_mx_atom_encode_decode_roundtrip():
    R_, K = 300, 256
    e = torch.randint(0, 255, (R_, K // 32), generator=_gen(), dtype=torch.uint8)
    sf = R.mx_encode_sf(e, K)
    assert sf.shape == (3, 2, 512)
    assert torch.equal(R.mx_decode_sf(sf, R_, K), e)
    # rows >= R stay zero
    used = torch.zeros(sf.numel(), dtype=torch.bool)
    r = torch.arange(R_)[:, None].expand(R_, K // 32)
    kb = torch.arange(K // 32)[None, :].expand(R_, K // 32)
    used[R.mx_sf_index(r, kb, K).reshape(-1)] = True
    assert (sf.reshape(-1)[~used] == 0).all()


@pytest.mark.parametrize("dtype", DTYPES)
def test_mx_reference_rejects_floor_and_swapped_atom(dtype):
    x = _x((160, 256), dtype)
    q, sf = R.mx_quantize_ref(x)
    blocks = x.double().reshape(160, 8, 32)
    amax = blocks.abs().amax(-1)
    e_floor = torch.floor(torch.log2(amax / 448.0)).clamp(-127, 127)
    q_floor = R.e4m3_rne(blocks * torch.exp2(-e_floor)[..., None]).reshape(160, 256).to(torch.float8_e4m3fn)
    assert not torch.equal(q_floor.view(torch.uint8), q.view(torch.uint8))
    # (r % 32) and (r % 128) / 32 swapped in the atom
    e_rows = R.mx_decode_sf(sf, 160, 256)
    wrong = torch.zeros_like(sf).reshape(-1)
    for r in range(160):
        for kb in range(8):
            i = ((r // 128) * 2 + kb // 4) * 512 + ((r % 128) // 32) * 16 + (r % 32) * 4 + kb % 4
            wrong[i] = e_rows[r, kb]
    assert not torch.equal(wrong.view_as(sf), sf)


@pytest.mark.parametrize("dtype", DTYPES)
def test_quantize_mx_reference_matches_mx_quantize_ref(dtype):
    x = _x((64, 256), dtype)
    x[1, :32] = 0
    x[2, :32] = 448.0 * 4                      # amax exactly 448 * 2^2: scale 2^2, values 448
    q, sf = R.mx_quantize_ref(x)
    assert torch.equal(Q.quantize_mx_reference(x).double(), R.mx_dequant(q, sf))


# ---------------------------------------------------------------------------------------------------------------- GEMMs
def _int8(shape, seed, lo=-128, hi=128):
    return torch.randint(lo, hi, shape, generator=_gen(seed), dtype=torch.int8)


def _gemm_case(M=129, N=136, K=272):
    a, b = _int8((M, K), 0), _int8((N, K), 1)
    rs = torch.rand(M, generator=_gen(2)) * 1e-3 + 1e-4
    cs = torch.rand(N, generator=_gen(3)) * 1e-2 + 1e-3
    bias = torch.randn(N, generator=_gen(4)).to(torch.bfloat16)
    return a, b, rs, cs, bias


def _int8_check(dtype, got_fn, a, b, rs, cs, bias):
    ref, acc_sc, _ = R.lowp_gemm_ref(a, b, rs, cs, bias)
    R.assert_close(ref.to(dtype), ref, dtype, **R.int8_gemm_bound(acc_sc))
    with pytest.raises(AssertionError):
        R.assert_close(got_fn(ref).to(dtype), ref, dtype, **R.int8_gemm_bound(acc_sc))


@pytest.mark.parametrize("dtype", DTYPES)
def test_int8_gemm_bound_rejects_tiling_mistakes(dtype):
    a, b, rs, cs, bias = _gemm_case()
    bias = bias.to(dtype)
    full = lambda a_, b_, rs_, cs_, bias_: R.lowp_gemm_ref(a_, b_, rs_, cs_, bias_)[0]
    # last k-block dropped (K % 128 != 0)
    _int8_check(dtype, lambda ref: full(a[:, :256], b[:, :256], rs, cs, bias), a, b, rs, cs, bias)
    # row scale of row_lo applied to row_lo + 8
    rs_w = rs.clone().view(-1)
    for r0 in range(0, 128, 16):
        rs_w[r0 + 8:r0 + 16] = rs[r0:r0 + 8]
    _int8_check(dtype, lambda ref: full(a, b, rs_w, cs, bias), a, b, rs, cs, bias)
    # cs.x / cs.y swapped
    cs_w = cs.view(-1, 2).flip(-1).reshape(-1)
    _int8_check(dtype, lambda ref: full(a, b, rs, cs_w, bias), a, b, rs, cs, bias)
    # bias missing on the last 8 columns
    bias_w = bias.clone()
    bias_w[-8:] = 0
    _int8_check(dtype, lambda ref: full(a, b, rs, cs, bias_w), a, b, rs, cs, bias)

    # a 128-row tile written to its neighbour's rows
    def shifted(ref):
        w = ref.clone()
        w[128:129] = ref[0:1]
        return w
    _int8_check(dtype, shifted, a, b, rs, cs, bias)


def _trunc(v, bits=14):
    m, e = np.frexp(v)
    return np.ldexp(np.trunc(m * 2.0 ** bits) / 2.0 ** bits, e)


def _emulate_fp8_mma(a, b, chunk=None, bits=14):
    """An fp8 MMA whose accumulator keeps ``bits`` significand bits, truncating after each K = 32 instruction; with ``chunk`` the chain
    restarts every ``chunk`` K and each partial is added to an fp32 sum."""
    prods = a[:, None, :] * b[None, :, :]
    groups = prods.reshape(a.shape[0], b.shape[0], -1, 32).sum(-1)
    per = (chunk or a.shape[1]) // 32
    out = np.zeros(groups.shape[:2], dtype=np.float32)
    for c0 in range(0, groups.shape[-1], per):
        acc = np.zeros(groups.shape[:2])
        for g in range(c0, c0 + per):
            acc = _trunc(acc + groups[..., g], bits)
        out = (out + acc.astype(np.float32)).astype(np.float32)
    return torch.from_numpy(out.astype(np.float64))


@pytest.mark.parametrize("positive", [True, False])
def test_fp8_bound_rejects_one_long_chain_and_accepts_promoted_chunks(positive):
    K = 16384
    g = _gen(5)
    a = torch.randn(4, K, generator=g, dtype=torch.float64)
    b = torch.randn(8, K, generator=g, dtype=torch.float64)
    if positive:
        a, b = a.abs() + 0.05, b.abs() + 0.05
    a = a.float().to(torch.float8_e4m3fn).double()
    b = b.float().to(torch.float8_e4m3fn).double()
    # cancel the output against a bias, as the GPU test does, so that the check sees the fp32 accumulator and not the bf16 rounding
    acc = a @ b.t()
    bias = (-acc).to(torch.bfloat16).double()
    ref, _, terms = R.lowp_gemm_ref(a, b, None, None, bias[0])
    bound = R.fp8_gemm_bound(terms, K)
    chain = _emulate_fp8_mma(a.numpy(), b.numpy()) + bias[0]
    promoted = _emulate_fp8_mma(a.numpy(), b.numpy(), chunk=128) + bias[0]
    R.assert_close(promoted.to(torch.bfloat16), ref, torch.bfloat16, **bound)
    if positive:
        with pytest.raises(AssertionError):
            R.assert_close(chain.to(torch.bfloat16), ref, torch.bfloat16, **bound)
        # the promoted chunks land far inside the bound; one long chain lies far outside it
        assert R.error_ratio(promoted.to(torch.bfloat16), ref, torch.bfloat16, **bound) < 0.25
        assert R.error_ratio(chain.to(torch.bfloat16), ref, torch.bfloat16, **bound) > 2


# ---------------------------------------------------------------------------------------------------------------- CPU fallbacks
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("K", [48, 2064])
def test_int8_linear_cpu_path_is_within_one_rounding(dtype, K):
    w = torch.randn(24, K, generator=_gen(6)).to(dtype)
    bias = torch.randn(24, generator=_gen(7)).to(dtype)
    lin = Q.Int8Linear.from_float(w, bias)
    assert lin.bias.dtype == dtype
    x = _x((9, K), dtype, seed=8)
    y = lin(x)
    assert y.dtype == dtype
    xq, xs = Q.quantize_rows_reference(x, None)
    ref, acc_sc, _ = R.lowp_gemm_ref(xq, lin.weight_q, xs, lin.weight_scale, lin.bias)
    R.assert_close(y, ref, dtype, **R.int8_gemm_bound(acc_sc), what="Int8Linear cpu")


@pytest.mark.parametrize("recipe", ["rowwise", "mx"])
def test_fp8_linear_cpu_path_is_within_one_rounding(recipe):
    dtype = torch.bfloat16
    K = 2048
    w = torch.randn(16, K, generator=_gen(9)).to(dtype)
    bias = torch.randn(16, generator=_gen(10)).to(dtype)
    x = _x((5, K), dtype, seed=11)
    y = Q.fp8_linear(x, w, bias, recipe=recipe)
    if recipe == "mx":
        a, b = R.mx_dequant(*R.mx_quantize_ref(x)), R.mx_dequant(*R.mx_quantize_ref(w))
        ref, acc_sc, _ = R.lowp_gemm_ref(a, b, None, None, bias)
    else:
        xq, xs = Q.quantize_rows_reference(x, None, True)
        wq, ws = Q.quantize_rows_reference(w, None, True)
        ref, acc_sc, _ = R.lowp_gemm_ref(xq.double(), wq.double(), xs, ws, bias)
    # the reference path sums in float64: one rounding to the output
    R.assert_close(y, ref, dtype, **R.int8_gemm_bound(acc_sc), what=f"fp8_linear {recipe} cpu")
