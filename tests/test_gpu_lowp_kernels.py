"""The 8-bit path against exact and float64 references (needs an H100).

Covers ``quantize_rows`` (int8 / e4m3, with and without a SmoothQuant divisor), ``gemm_lowp`` (int8 and fp8, bf16 and fp16 output),
``quantize_mxfp8`` + ``gemm_mxfp8``, the W8A8 decode GEMV and the ``Int8Linear`` / ``fp8_linear`` layers.  An int8 product is exact in
float64, so the int8 GEMM and GEMV must land within one rounding of the exact result, and bitwise on small integers; the quantisers are
checked element by element (MX bit for bit).  Bounds come from ``kernel_refs`` (see its docstring and the 8-bit section).

Run with ``-s`` to print the largest error/bound ratio seen per kernel and dtype.
"""
from collections import defaultdict

import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import quant as Q

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16
DTYPES = [B16, F16]
RATIOS = defaultdict(float)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for key in sorted(RATIOS, key=str):
        print(f"max error/bound {key[0]:<24} {str(key[1]):<15} {RATIOS[key]:.3f}")


@pytest.fixture(scope="module")
def lib():
    return _native.require()


def _close(kernel, got, ref, dtype, **kw):
    r = R.assert_close(got, ref, dtype, what=kernel, **kw)
    RATIOS[(kernel, dtype)] = max(RATIOS[(kernel, dtype)], r)


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _x(shape, dtype, seed=0):
    g = _gen(seed)
    x = torch.randn(shape, generator=g, device="cuda", dtype=torch.float64)
    return (x * torch.exp2(torch.randint(-6, 7, (shape[0], 1), generator=g, device="cuda").double())).to(dtype)


def _int8(shape, seed, lo=-128, hi=128):
    return torch.randint(lo, hi, shape, generator=_gen(seed), device="cuda", dtype=torch.int8)


def _e4m3(shape, seed, positive=False):
    x = torch.randn(shape, generator=_gen(seed), device="cuda") * 8
    if positive:
        x = x.abs() + 0.05
    return x.clamp(-448, 448).to(torch.float8_e4m3fn)


def _f64(q):
    return q.float().double() if q.dtype == torch.float8_e4m3fn else q.double()


# ---------------------------------------------------------------------------------------------------------------- quantize_rows
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("fp8", [False, True])
@pytest.mark.parametrize("smoothed", [False, True])
@pytest.mark.parametrize("cols", [8, 16, 1032, 4096, 12288, 32768])
def test_quantize_rows(lib, dtype, fp8, smoothed, cols):
    rows = 3 if cols >= 12288 else 4097 if cols <= 1032 else 4
    x = _x((rows, cols), dtype, seed=cols)
    if rows > 2:
        x[0] = 0                                            # zero row: scale 1, q = 0
        x[1] = 0
        x[1, cols // 2] = -3.0                              # one nonzero
        x[2] = 0.75                                         # constant
    if rows > 3:
        x[3, 0], x[3, -1] = 5.0, -5.0                       # both +-amax
    if dtype == B16 and rows > 3 and not smoothed:
        x[-1, :] = torch.finfo(B16).max * (1 - 2.0 ** -7)   # near bf16's largest finite values (finite after / smooth)
        x[-1, ::2] *= -1
    sm = torch.exp(torch.empty(cols, device="cuda").uniform_(-2.302585, 2.302585, generator=_gen(1))) if smoothed else None
    q, s = lib.quantize_rows(x, sm, fp8)
    R.quantize_rows_check(x, sm, q, s, fp8)


def test_quantize_rows_refusals(lib):
    x = torch.randn(4, 64, device="cuda", dtype=B16)
    with pytest.raises(RuntimeError, match="x must be bf16 or fp16"):
        lib.quantize_rows(x.float(), None, False)
    with pytest.raises(RuntimeError, match="smooth"):
        lib.quantize_rows(x, torch.ones(32, device="cuda"), False)
    with pytest.raises(RuntimeError, match="cols"):
        lib.quantize_rows(torch.randn(4, 12, device="cuda", dtype=B16), None, False)
    with pytest.raises(RuntimeError, match="cols"):
        lib.quantize_rows(torch.randn(2, 32776, device="cuda", dtype=B16), None, False)


# ---------------------------------------------------------------------------------------------------------------- int8 GEMM
SHAPES = [(1, 8, 16), (127, 136, 144), (129, 264, 4096), (300, 1032, 16384), (4160, 4104, 1024)]


def _epilogue(M, N, dtype, seed, rs_on, cs_on, bias_on, hi=1e-2):
    g = _gen(seed)
    rs = torch.rand(M, generator=g, device="cuda") * hi + hi / 100 if rs_on else None
    cs = torch.rand(N, generator=g, device="cuda") * hi + hi / 100 if cs_on else None
    bias = (torch.randn(N, generator=g, device="cuda") * 4).to(dtype) if bias_on else None
    return rs, cs, bias


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("dtype", DTYPES)
def test_gemm_int8(lib, shape, dtype):
    M, N, K = shape
    a, b = _int8((M, K), 1), _int8((N, K), 2)
    a[0, :4] = -128                                          # raw int8 operands include -128
    cases = [(True, True, True), (False, True, False), (True, False, True), (False, False, False)]
    for i, (rs_on, cs_on, bias_on) in enumerate(cases if dtype == B16 else cases[:3]):
        # fp16 output: keep |acc| * rs * cs (|acc| <= K * 2^14) inside the fp16 range
        hi = 1e-2 if dtype == B16 else (1e4 / (K * 2.0 ** 14)) ** (0.5 if rs_on and cs_on else 1.0)
        rs, cs, bias = _epilogue(M, N, dtype, 10 + i, rs_on, cs_on, bias_on, hi)
        y = lib.gemm_lowp(a, b, rs, cs, bias, 0, out_dtype=dtype)
        assert y.dtype == dtype
        ref, acc_sc, _ = R.lowp_gemm_ref(a, b, rs, cs, bias)
        _close("gemm_lowp int8", y, ref, dtype, **R.int8_gemm_bound(acc_sc))


def test_gemm_int8_saturated(lib):
    M, N, K = 129, 136, 16384
    a = torch.where(torch.rand(M, K, device="cuda", generator=_gen(3)) < 0.5, 127, -127).to(torch.int8)
    a[:64] = 127
    b = torch.where(torch.rand(N, K, device="cuda", generator=_gen(4)) < 0.5, 127, -127).to(torch.int8)
    b[:64] = -127
    y = lib.gemm_lowp(a, b, None, None, None, 0)
    ref, acc_sc, _ = R.lowp_gemm_ref(a, b)
    _close("gemm_lowp int8", y, ref, B16, **R.int8_gemm_bound(acc_sc))


@pytest.mark.parametrize("shape", SHAPES)
def test_gemm_int8_small_integers_are_bitwise_exact(lib, shape):
    # ternary operands, rs = cs = 1, no bias: every |exact| <= 256 is a bf16 integer, so any tile, raster or tail mapping error shows
    M, N, K = shape
    a, b = _int8((M, K), 5, -1, 2), _int8((N, K), 6, -1, 2)
    y = lib.gemm_lowp(a, b, None, None, None, 0).double()
    exact = a.double() @ b.double().t()
    small = exact.abs() <= 256
    assert small.float().mean() > 0.5
    assert torch.equal(y[small], exact[small])


# ---------------------------------------------------------------------------------------------------------------- fp8 GEMM
@pytest.mark.parametrize("shape", SHAPES + [(256, 264, k) for k in (128, 1024, 8192)])
def test_gemm_fp8(lib, shape):
    M, N, K = shape
    a, b = _e4m3((M, K), 7), _e4m3((N, K), 8)
    rs, cs, bias = _epilogue(M, N, B16, 20, True, True, True)
    y = lib.gemm_lowp(a, b, rs, cs, bias, 0)
    ref, _, terms = R.lowp_gemm_ref(_f64(a), _f64(b), rs, cs, bias)
    _close("gemm_lowp fp8", y, ref, B16, **R.fp8_gemm_bound(terms, K))


@pytest.mark.parametrize("K", [128, 1024, 4096, 8192, 16384])
def test_gemm_fp8_accumulation(lib, K):
    """Positive terms, and a bias that cancels row 0 of the product: row 0 of the output then shows the fp32 accumulator's own error,
    not the bf16 rounding.  One tensor-core chain over all of K lost 2^-6 of the sum at K = 1024 and 2^-2 at K = 16384 on an H100; the
    kernel adds each 128-K chain into fp32 registers, and each chain stays within FP8_MMA of its terms."""
    M, N = 256, 264
    a, b = _e4m3((M, K), 30 + K, positive=True), _e4m3((N, K), 31 + K, positive=True)
    a64, b64 = _f64(a), _f64(b)
    bias = (-(a64[0] @ b64.t())).to(B16)
    y = lib.gemm_lowp(a, b, None, None, bias, 0)
    ref, _, terms = R.lowp_gemm_ref(a64, b64, None, None, bias)
    _close("gemm_lowp fp8 accum", y, ref, B16, **R.fp8_gemm_bound(terms, K))
    chunk_err = float(((y[0].double() - ref[0]).abs() / (a64[0] @ b64.t())).max())
    print(f"fp8 accumulation K={K}: max |err| / sum|terms| = {chunk_err:.3g}")
    assert chunk_err <= R.FP8_MMA


# ---------------------------------------------------------------------------------------------------------------- MX
def _mx_input(R_, K, dtype, seed):
    g = _gen(seed)
    x = torch.randn(R_, K // 32, 32, generator=g, device="cuda", dtype=torch.float64)
    lim = 10 if dtype == F16 else 20                        # |x| < 8 * 2^10 stays finite in fp16
    x = x * torch.exp2(torch.randint(-lim, lim + 1, (R_, K // 32, 1), generator=g, device="cuda").double())
    if R_ > 2:
        x[1, 0] = 0                                          # zero block: byte 0
        x[2, 0] = 1.0
        x[2, 0, 5] = -448.0 * 2.0 ** 3                        # amax exactly 448 * 2^3
        x[2, 1] = 448.0 / 4                                   # amax exactly 448 * 2^-2
    return x.reshape(R_, K).to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", [0, 1, 129, 300])
def test_quantize_mxfp8_bitwise(lib, dtype, rows):
    K = 256
    x = _mx_input(rows, K, dtype, rows)
    q, sf = lib.quantize_mxfp8(x)
    q_ref, sf_ref = R.mx_quantize_ref(x)
    assert q.shape == (rows, K) and sf.shape == sf_ref.shape
    assert torch.equal(q.view(torch.uint8).cpu(), q_ref.view(torch.uint8))
    assert torch.equal(sf.cpu(), sf_ref)


def test_quantize_mxfp8_flushes_fp32_subnormal_blocks(lib):
    """Found but not changed: under --use_fast_math a block whose values are fp32 subnormals (bf16 below 2^-126) flushes to zero; the
    float64 reference keeps it at scale 2^-127.  No real activation or weight is that small.  This fails if the kernel stops flushing."""
    x = torch.zeros(1, 128, device="cuda", dtype=B16)
    x[0, :32] = 2.0 ** -130
    q, sf = lib.quantize_mxfp8(x)
    q_ref, sf_ref = R.mx_quantize_ref(x)
    assert torch.equal(sf.cpu(), sf_ref)                     # byte 0 either way
    assert (q_ref.float()[0, :32] == 2.0 ** -3).all()
    assert (q.float() == 0).all()


@pytest.mark.parametrize("M", [1, 129, 300])
@pytest.mark.parametrize("K", [128, 4096])
def test_gemm_mxfp8(lib, M, K):
    N = 264
    xa, xb = _mx_input(M, K, B16, 40 + M), _mx_input(N, K, B16, 41)
    qa, sa = lib.quantize_mxfp8(xa)
    qb, sb = lib.quantize_mxfp8(xb)
    bias = torch.randn(N, device="cuda", generator=_gen(42)).to(B16)
    y = lib.gemm_mxfp8(qa, sa, qb, sb, bias)
    a64, b64 = R.mx_dequant(qa, sa).cuda(), R.mx_dequant(qb, sb).cuda()
    ref, _, terms = R.lowp_gemm_ref(a64, b64, None, None, bias)
    _close("gemm_mxfp8", y, ref, B16, **R.fp8_gemm_bound(terms, K))


# ---------------------------------------------------------------------------------------------------------------- W8A8 GEMV
@pytest.mark.parametrize("K", [16, 1040, 16384])
@pytest.mark.parametrize("dtype", DTYPES)
def test_gemv_w8a8(lib, K, dtype):
    N = 1001
    w = _int8((N, K), 50)
    ws = torch.rand(N, device="cuda", generator=_gen(51)) * 1e-2 + 1e-4
    bias = torch.randn(N, device="cuda", generator=_gen(52)).to(dtype)
    for M in range(1, 9):
        x = _int8((M, K), 60 + M)
        xs = torch.rand(M, device="cuda", generator=_gen(61)) * 1e-2 + 1e-4
        y = lib.gemv_w8a8(x, w, xs, ws, bias, out_dtype=dtype)
        assert y.dtype == dtype
        ref, acc_sc, _ = R.lowp_gemm_ref(x, w, xs, ws, bias)
        _close("gemv_w8a8", y, ref, dtype, **R.int8_gemm_bound(acc_sc))
        # the GEMM on the same operands agrees to one ulp, plus the two epilogues' fp32 roundings where the bias cancels the product
        y2 = lib.gemm_lowp(x, w[:1000], xs, ws[:1000], bias[:1000], 0, out_dtype=dtype).double()
        y1 = y[:, :1000].double()
        ulp = torch.exp2(torch.floor(torch.log2(torch.maximum(y1.abs(), y2.abs()).clamp(min=1e-30))) - (7 if dtype == B16 else 10))
        assert ((y1 - y2).abs() <= ulp + 2 * R.LOWP_EPILOGUE * acc_sc[:, :1000]).all()
        # ternary operands without scales: small integers are exact
        xt, wt = _int8((M, K), 70 + M, -1, 2), _int8((N, K), 71, -1, 2)
        one_m, one_n = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
        yt = lib.gemv_w8a8(xt, wt, one_m, one_n, None, out_dtype=dtype).double()
        exact = xt.double() @ wt.double().t()
        small = exact.abs() <= 256
        assert torch.equal(yt[small], exact[small])


def test_gemv_w8a8_refusals(lib):
    M, N, K = 2, 64, 64
    x, w = _int8((M, K), 1), _int8((N, K), 2)
    xs, ws = torch.ones(M, device="cuda"), torch.ones(N, device="cuda")
    with pytest.raises(RuntimeError, match="bias"):
        lib.gemv_w8a8(x, w, xs, ws, torch.zeros(N, device="cuda", dtype=F16))           # fp16 bias, bf16 output
    with pytest.raises(RuntimeError, match="bias"):
        lib.gemv_w8a8(x, w, xs, ws, torch.zeros(N - 8, device="cuda", dtype=B16))
    with pytest.raises(RuntimeError, match="xs"):
        lib.gemv_w8a8(x, w, torch.ones(2 * M, device="cuda")[::2], ws)
    with pytest.raises(RuntimeError, match="ws"):
        lib.gemv_w8a8(x, w, xs, torch.ones(N, device="cuda", dtype=torch.float64))
    buf = torch.zeros(M * K + 16, device="cuda", dtype=torch.int8)
    with pytest.raises(RuntimeError, match="xq must be 16-byte aligned"):
        lib.gemv_w8a8(buf[1:1 + M * K].view(M, K), w, xs, ws)


# ---------------------------------------------------------------------------------------------------------------- layers
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", [1, 8, 9, 300])
@pytest.mark.parametrize("smoothed", [False, True])
def test_int8_linear(lib, dtype, M, smoothed):
    N, K = 264, 1040
    w = (torch.randn(N, K, device="cuda", generator=_gen(80)) * 0.05).to(dtype)
    bias = torch.randn(N, device="cuda", generator=_gen(81)).to(dtype)
    sm = torch.exp(torch.empty(K, device="cuda").uniform_(-1.0, 1.0, generator=_gen(82))) if smoothed else None
    lin = Q.Int8Linear.from_float(w, bias, smooth=sm)
    x = _x((M, K), dtype, seed=83)
    y = lin(x)
    assert y.dtype == dtype
    xq, xs = lib.quantize_rows(x, lin.smooth, False)
    R.quantize_rows_check(x, lin.smooth, xq, xs, False)
    ref, acc_sc, _ = R.lowp_gemm_ref(xq, lin.weight_q, xs, lin.weight_scale, lin.bias)
    _close("Int8Linear", y, ref, dtype, **R.int8_gemm_bound(acc_sc))


def test_int8_linear_wide_input(lib):
    K = 32768 + 16
    w = (torch.randn(16, K, device="cuda", generator=_gen(90)) * 0.05).to(B16)
    lin = Q.Int8Linear.from_float(w, None)
    x = _x((3, K), B16, seed=91)
    y = lin(x)
    xq, xs = Q.quantize_rows_reference(x, None)
    ref, acc_sc, _ = R.lowp_gemm_ref(xq, lin.weight_q, xs, lin.weight_scale)
    _close("Int8Linear", y, ref, B16, **R.int8_gemm_bound(acc_sc))


@pytest.mark.parametrize("M", [0, 1, 8, 9, 300])
@pytest.mark.parametrize("recipe", ["rowwise", "mx"])
def test_fp8_linear(lib, M, recipe):
    N, K = 264, 1024
    w = (torch.randn(N, K, device="cuda", generator=_gen(100)) * 0.05).to(B16)
    bias = torch.randn(N, device="cuda", generator=_gen(101)).to(B16)
    x = _x((max(M, 1), K), B16, seed=102)[:M]
    y = Q.fp8_linear(x, w, bias, recipe=recipe)
    assert y.shape == (M, N)
    if M == 0:
        return
    if recipe == "mx":
        a64 = R.mx_dequant(*lib.quantize_mxfp8(x)).cuda()
        b64 = R.mx_dequant(*lib.quantize_mxfp8(w)).cuda()
        ref, _, terms = R.lowp_gemm_ref(a64, b64, None, None, bias)
    else:
        xq, xs = lib.quantize_rows(x, None, True)
        wq, ws = lib.quantize_rows(w, None, True)
        ref, _, terms = R.lowp_gemm_ref(_f64(xq), _f64(wq), xs, ws, bias)
    _close(f"fp8_linear {recipe}", y, ref, B16, **R.fp8_gemm_bound(terms, K))
