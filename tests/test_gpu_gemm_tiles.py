"""The persistent wgmma GEMM at sizes where a CTA runs several tiles (needs an H100).

The other GEMM tests stay under one wave of tiles, so no CTA ever runs a second tile, wraps its shared-memory stage ring from one tile
into the next, or reuses an epilogue staging buffer.  These cases do, in both 16-bit dtypes, against a float64 reference
(``kernel_refs.assert_close``): several waves, partial column tiles, M and K tails, all four operand majors, every epilogue, the 16-bit
and both fp32 output modes, and the two grouped modes with an expert that owns no rows and one with an empty token segment.
"""
import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16
EPI_NONE, EPI_BIAS, EPI_BIAS_GELU, EPI_GELU = 0, 1, 2, 3
# A tile, stage or staging buffer mixed up is wrong by the size of the result, far outside the R.MMA_ACC allowance.
MMA_ACC = R.MMA_ACC


@pytest.fixture(scope="module")
def lib():
    return _native.require()


def _operands(M, N, K, dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    b = torch.randn(N, K, device="cuda", generator=g).to(dtype)
    return a, b


def _product(a, b):
    """float64 a b^T and the sum of |terms| it is formed from."""
    a64, b64 = a.double(), b.double()
    return a64 @ b64.t(), a64.abs() @ b64.abs().t()


def _gemm(lib, a, b, a_k, b_k, bias=None, out=None, epilogue=EPI_NONE, out_mode=0):
    """lib.gemm on a [M, K], b [N, K] handed over in the requested majors (MN-major = the transposed copy)."""
    return lib.gemm(a if a_k else a.t().contiguous(), b if b_k else b.t().contiguous(), bias, out, a_k, b_k, epilogue, out_mode, 0)


MAJORS = [(True, True), (True, False), (False, True), (False, False)]
SHAPES = {
    "waves": (8192, 6144, 2048),       # 3072 tiles of 128 x 128: 23 per CTA on 132 SMs
    "n_half_tile": (1024, 2432, 512),  # N % 256 = 128, as the LM head's 50304
    "n_264": (904, 264, 136),          # N a multiple of 8 but not of 64, M and K tails
}


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("out_mode", [0, 1, 2])
@pytest.mark.parametrize("majors", MAJORS, ids=["nt", "nn", "tn", "tt"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_gemm_tiles(lib, shape, majors, out_mode, dtype):
    M, N, K = SHAPES[shape]
    if shape == "waves" and majors != (True, True) and out_mode != 0:
        pytest.skip("the multi-wave shape runs every major once and every output mode once")
    a, b = _operands(M, N, K, dtype, seed=M + N + K + out_mode)
    ref, terms = _product(a, b)
    out = None
    if out_mode == 2:
        out = torch.randn(M, N, device="cuda")
        ref = ref + out.double()
        terms = terms + out.double().abs()
    elif out_mode == 1:
        out = torch.full((M, N), float("nan"), device="cuda")
    got = _gemm(lib, a, b, *majors, out=out, out_mode=out_mode)
    torch.cuda.synchronize()
    R.assert_close(got, ref, dtype if out_mode == 0 else torch.float32, scale=terms, n=K, approx=MMA_ACC,
                   what=f"gemm {shape} {majors} out {out_mode}")


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("epilogue", ["bias", "bias_gelu", "gelu", "bias_gelu_dual", "dgelu"])
def test_gemm_tiles_epilogues(lib, epilogue, dtype):
    M, N, K = 2304, 2432, 1024     # 18 x 19 tiles of 128 x 128: two or three per CTA
    a, b = _operands(M, N, K, dtype, seed=7)
    g = torch.Generator(device="cuda").manual_seed(8)
    bias = torch.randn(N, device="cuda", generator=g).to(dtype)
    acc, terms = _product(a, b)
    gelu = lambda x: torch.nn.functional.gelu(x, approximate="tanh")
    kw = dict(n=K, approx=MMA_ACC + R.TANH_APPROX)
    if epilogue == "dgelu":
        z = torch.randn(M, N, device="cuda", generator=g).to(dtype)
        z64 = z.double().requires_grad_()
        dg = torch.autograd.grad(gelu(z64).sum(), z64)[0]
        got = lib.gemm_dgelu(a, b.t().contiguous(), z)
        torch.cuda.synchronize()
        scale = terms * dg.abs() + acc.abs() * (1.0 + 2.0 * z.double().abs() ** 3)
        R.assert_close(got, acc * dg, dtype, scale=scale, what="dgelu", **kw)
        return
    pre = acc + bias.double()
    pre_scale = terms + bias.double().abs()
    if epilogue == "bias_gelu_dual":
        z, y = lib.gemm_bias_gelu_dual(a, b, bias)
        torch.cuda.synchronize()
        R.assert_close(z, pre, dtype, scale=pre_scale, what="dual pre-activation", **kw)
        # the GELU is taken of the fp32 pre-activation, before its rounding to the output dtype
        R.assert_close(y, gelu(pre), dtype, scale=1.2 * pre_scale + 0.5 * pre.abs(), what="dual gelu", **kw)
        return
    code = {"bias": EPI_BIAS, "bias_gelu": EPI_BIAS_GELU, "gelu": EPI_GELU}[epilogue]
    if epilogue == "gelu":
        pre, pre_scale, bias = acc, terms, None
    got = _gemm(lib, a, b, True, True, bias=bias, epilogue=code)
    torch.cuda.synchronize()
    if epilogue == "bias":
        R.assert_close(got, pre, dtype, scale=pre_scale, what=epilogue, **kw)
    else:
        R.assert_close(got, gelu(pre), dtype, scale=1.2 * pre_scale + 0.5 * pre.abs(), what=epilogue, **kw)


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
def test_gemm_tiles_grouped_rows(lib, dtype):
    """Grouped mode 1 over many row blocks: expert 1 owns no rows, and blocks marked -1 are left untouched."""
    G, K, N = 4, 512, 2432
    owners = [0, 2, -1, 3, 0, 0, 2, -1, 3, 3, 2, 0] * 4
    M = 128 * len(owners)
    tile_group = torch.tensor(owners, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(11)
    a = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    b = (torch.randn(G, N, K, device="cuda", generator=g) * 0.05).to(dtype)
    bias = torch.randn(G, N, device="cuda", generator=g).to(dtype)
    out = torch.full((M, N), 7.0, device="cuda", dtype=dtype)
    lib.gemm_grouped(a, b, bias.reshape(-1), tile_group, out, True, EPI_BIAS, None, None, 128)
    torch.cuda.synchronize()
    for blk, e in enumerate(owners):
        rows = slice(128 * blk, 128 * (blk + 1))
        if e < 0:
            assert bool((out[rows] == 7.0).all()), f"row block {blk} is owned by no expert but was written"
            continue
        ref, terms = _product(a[rows], b[e])
        R.assert_close(out[rows], ref + bias[e].double(), dtype, scale=terms + bias[e].double().abs(), n=K, approx=MMA_ACC,
                       what=f"grouped rows block {blk}")


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
def test_gemm_tiles_grouped_wgrad(lib, dtype):
    """Grouped mode 2: out[g] = dy[rows of g]^T x[rows of g]; expert 1's segment is empty, so its gradient is zero."""
    Mg, N = 384, 2432
    segs = [(0, 1024), (1024, 0), (1024, 192), (1216, 2048)]
    seg2 = torch.tensor([v for s in segs for v in s], dtype=torch.int32, device="cuda")
    rows = sum(c for _, c in segs)
    g = torch.Generator(device="cuda").manual_seed(12)
    dy = torch.randn(rows, Mg, device="cuda", generator=g).to(dtype)
    x = torch.randn(rows, N, device="cuda", generator=g).to(dtype)
    out = torch.full((len(segs), Mg, N), float("nan"), device="cuda", dtype=dtype)
    lib.gemm_grouped_wgrad(dy, x, seg2, out)
    torch.cuda.synchronize()
    for i, (s, c) in enumerate(segs):
        if c == 0:
            assert bool((out[i] == 0).all()), "the expert without tokens must get a zero gradient"
            continue
        ref, terms = _product(dy[s:s + c].t(), x[s:s + c].t())
        R.assert_close(out[i], ref, dtype, scale=terms, n=c, approx=MMA_ACC, what=f"grouped wgrad expert {i}")
