"""The 128 x 256 tile of the persistent wgmma GEMM (``config = 1``), which the backward pass runs (needs an H100).

Against a float64 reference (``kernel_refs.assert_close``) in both 16-bit dtypes: several waves of tiles per CTA, N a multiple of 256,
N % 256 = 128 (as the LM head's 50304), N = 264 with M and K tails, all four operand majors, and the epilogues the backward uses
(none, bias, GELU derivative).  At GPT-1.3B's backward shapes the wide tile must equal the 128 x 128 tile bit for bit: both accumulate
every output element over K in the same order, 16 at a time.  A request for the wide tile that it does not serve (fp32 output modes,
GELU epilogues) runs 128 x 128 and gives that tile's result exactly.
"""
import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16
EPI_NONE, EPI_BIAS, EPI_BIAS_GELU, EPI_GELU = 0, 1, 2, 3
WIDE = 1
MMA_ACC = R.MMA_ACC


@pytest.fixture(scope="module")
def lib():
    return _native.require()


def _operands(M, N, K, dtype, seed, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    b = (torch.randn(N, K, device="cuda", generator=g) * scale).to(dtype)
    return a, b


def _product(a, b):
    a64, b64 = a.double(), b.double()
    return a64 @ b64.t(), a64.abs() @ b64.abs().t()


def _gemm(lib, a, b, a_k, b_k, config, bias=None, out=None, epilogue=EPI_NONE, out_mode=0):
    return lib.gemm(a if a_k else a.t().contiguous(), b if b_k else b.t().contiguous(), bias, out, a_k, b_k, epilogue, out_mode, config)


MAJORS = [(True, True), (True, False), (False, True), (False, False)]
SHAPES = {
    "waves": (8192, 6144, 2048),       # 1536 tiles of 128 x 256: 11-12 per CTA on 132 SMs; N % 256 = 0
    "n_half_tile": (1024, 2432, 512),  # N % 256 = 128, as the LM head's 50304
    "n_264": (904, 264, 136),          # N a multiple of 8 but not of 64, M and K tails
}


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("majors", MAJORS, ids=["nt", "nn", "tn", "tt"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_gemm_wide_tiles(lib, shape, majors, dtype):
    M, N, K = SHAPES[shape]
    a, b = _operands(M, N, K, dtype, seed=M + N + K)
    ref, terms = _product(a, b)
    got = _gemm(lib, a, b, *majors, WIDE)
    torch.cuda.synchronize()
    R.assert_close(got, ref, dtype, scale=terms, n=K, approx=MMA_ACC, what=f"wide gemm {shape} {majors}")


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("epilogue", ["bias", "dgelu"])
@pytest.mark.parametrize("shape", ["waves", "n_half_tile", "n_264"])
def test_gemm_wide_epilogues(lib, shape, epilogue, dtype):
    M, N, K = SHAPES[shape]
    a, b = _operands(M, N, K, dtype, seed=7 + M)
    g = torch.Generator(device="cuda").manual_seed(8)
    acc, terms = _product(a, b)
    kw = dict(n=K, approx=MMA_ACC + R.TANH_APPROX)
    if epilogue == "dgelu":
        z = torch.randn(M, N, device="cuda", generator=g).to(dtype)
        z64 = z.double().requires_grad_()
        dg = torch.autograd.grad(torch.nn.functional.gelu(z64, approximate="tanh").sum(), z64)[0]
        got = lib.gemm_dgelu(a, b.t().contiguous(), z, WIDE)
        torch.cuda.synchronize()
        scale = terms * dg.abs() + acc.abs() * (1.0 + 2.0 * z.double().abs() ** 3)
        R.assert_close(got, acc * dg, dtype, scale=scale, what=f"wide dgelu {shape}", **kw)
        return
    bias = torch.randn(N, device="cuda", generator=g).to(dtype)
    got = _gemm(lib, a, b, True, True, WIDE, bias=bias, epilogue=EPI_BIAS)
    torch.cuda.synchronize()
    R.assert_close(got, acc + bias.double(), dtype, scale=terms + bias.double().abs(), what=f"wide bias {shape}", **kw)


TOKENS, H, VOCAB = 8 * 1024, 2048, 50304
# GPT-1.3B's backward GEMMs: (form, M, N, K, a_kmajor, b_kmajor).  dgrad dX = dY W (B MN-major); wgrad dW = dY^T X (both MN-major).
BACKWARD = {
    "qkv_dgrad": (TOKENS, H, 3 * H, True, False),
    "qkv_wgrad": (3 * H, H, TOKENS, False, False),
    "attn_out_dgrad": (TOKENS, H, H, True, False),
    "attn_out_wgrad": (H, H, TOKENS, False, False),
    "ffn1_dgrad": (TOKENS, H, 4 * H, True, False),
    "ffn1_wgrad": (4 * H, H, TOKENS, False, False),
    "ffn2_wgrad": (H, 4 * H, TOKENS, False, False),
    "lm_head_dgrad": (TOKENS, H, VOCAB, True, False),
    "lm_head_wgrad": (VOCAB, H, TOKENS, False, False),
}


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("form", list(BACKWARD) + ["ffn2_dgelu"])
def test_gemm_wide_bitwise_at_gpt_shapes(lib, form, dtype):
    g = torch.Generator(device="cuda").manual_seed(len(form))
    if form == "ffn2_dgelu":
        dy = torch.randn(TOKENS, H, device="cuda", generator=g).to(dtype)
        w2 = (torch.randn(H, 4 * H, device="cuda", generator=g) * 0.02).to(dtype)
        z = torch.randn(TOKENS, 4 * H, device="cuda", generator=g).to(dtype)
        narrow, wide = lib.gemm_dgelu(dy, w2, z, 0), lib.gemm_dgelu(dy, w2, z, WIDE)
    else:
        M, N, K, a_k, b_k = BACKWARD[form]
        a = torch.randn(*((M, K) if a_k else (K, M)), device="cuda", generator=g).to(dtype)
        b = (torch.randn(*((N, K) if b_k else (K, N)), device="cuda", generator=g) * 0.02).to(dtype)
        narrow = lib.gemm(a, b, None, None, a_k, b_k, EPI_NONE, 0, 0)
        wide = lib.gemm(a, b, None, None, a_k, b_k, EPI_NONE, 0, WIDE)
    torch.cuda.synchronize()
    assert narrow.isfinite().all()
    assert torch.equal(wide, narrow), f"{form}: the 128 x 256 tile differs from 128 x 128 in {(wide != narrow).sum().item()} elements"


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", ["out_f32", "out_f32_acc", "gelu", "bias_gelu"])
def test_gemm_wide_request_unserved(lib, case, dtype):
    M, N, K = 1024, 2432, 512
    a, b = _operands(M, N, K, dtype, seed=21)
    bias = (torch.randn(N, device="cuda") * 0.1).to(dtype)
    if case in ("out_f32", "out_f32_acc"):
        mode = 1 if case == "out_f32" else 2
        base = torch.randn(M, N, device="cuda")
        outs = [base.clone(), base.clone()]
        for out, config in zip(outs, (0, WIDE)):
            _gemm(lib, a, b, False, False, config, out=out, out_mode=mode)
        narrow, wide = outs
    else:
        epi, bb = (EPI_GELU, None) if case == "gelu" else (EPI_BIAS_GELU, bias)
        narrow = _gemm(lib, a, b, True, True, 0, bias=bb, epilogue=epi)
        wide = _gemm(lib, a, b, True, True, WIDE, bias=bb, epilogue=epi)
    torch.cuda.synchronize()
    assert torch.equal(wide, narrow), f"{case}: a wide request the tile does not serve must give the 128 x 128 result"
