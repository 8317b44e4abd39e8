"""GPU numerics: every native kernel against a plain PyTorch fp32 reference of the same op (needs an H100)."""
import os
import sys

import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

pytestmark = pytest.mark.gpu

import gpu_selftest as st  # noqa: E402

FAST = ["gemm_nt_1cta", "gemm_nt_1cta_n128", "gemm_nt_2cta", "gemm_nt_2cta_n128", "gemm_nn_1cta", "gemm_tn_1cta", "gemm_tk_1cta",
        "gemm_nn_2cta", "gemm_tn_2cta", "gemm_tail", "gemm_tail_2cta", "gemm_bias_gelu", "gemm_f32_acc", "gemm_f32", "layernorm",
        "rmsnorm", "gelu_dropout", "cross_entropy", "adamw", "topp", "rope_softmax", "gemv_skinny", "gemm_smallm", "attention_decode", "gemv_w8a8", "decode_fused", "attention_fwd", "fused_ffn", "gemm_int8", "gemm_int8_pair", "gemm_fp8", "gemm_fp8_pair",
        "gemm_big_sweep", "attention_train", "attention_autograd", "embedding", "norm_residual", "moe_grouped", "evoformer_attention", "gemm_mxfp8"]


@pytest.mark.parametrize("name", FAST)
def test_kernel(name):
    res = st.CHECKS[name]()
    assert res["ok"], res


def test_native_library_is_loaded():
    from paddlefleetx_b200.ops import _native

    lib = _native.require()
    assert "_pfx_native" in lib.__file__


def test_functional_linear_autograd_matches_torch():
    import torch

    from paddlefleetx_b200.ops import functional as OF

    torch.manual_seed(0)
    x = torch.randn(4, 96, 256, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    w = (torch.randn(512, 256, device="cuda") * 0.05).bfloat16().requires_grad_(True)
    b = torch.randn(512, device="cuda", dtype=torch.bfloat16, requires_grad=True)
    g = torch.randn(4, 96, 512, device="cuda", dtype=torch.bfloat16)
    OF.reset_launch_count()
    y = OF.linear(x, w, b)
    y.backward(g)
    assert OF.native_launch_count() >= 3
    xr, wr, br = (t.detach().float().requires_grad_(True) for t in (x, w, b))
    yr = torch.nn.functional.linear(xr, wr, br)
    yr.backward(g.float())
    for got, ref in ((y, yr), (x.grad, xr.grad), (w.grad, wr.grad), (b.grad, br.grad)):
        err = (got.float() - ref).norm() / ref.norm()
        assert err < 2e-2, err


def test_smoke_entry():
    import __graft_entry__ as ge

    ge.smoke()
