"""SwiGLU experts on the grouped sm_90a expert GEMMs (needs an H100): the two SwiGLU epilogues of ``gemm_grouped`` against float64, the whole
``GroupedFFN`` forward and backward against a float64 per-expert loop, the sync-free ``MoELayer`` against its expert loop, and a SwiGLU
GPT-MoE that trains on the grouped path without aten activation kernels.

The epilogues take h and dpre from the fp32 accumulator (``acc + bias`` for the forward, ``dh`` for the dgrad), never rounded to 16 bits,
so they are compared with float64 results of the exact GEMM, not bit for bit with the unfused ``bias_swiglu`` kernels.  The bound is the
``kernel_refs`` GEMM allowance carried through the SwiGLU formulas, plus the SwiGLU kernels' own arithmetic (``swiglu_refs``)."""
import math
import os

import numpy as np
import pytest
import torch

import kernel_refs as R
import swiglu_refs as S
from paddlefleetx_b200.ops import _native

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16
EPI_BIAS_SWIGLU_DUAL, EPI_DSWIGLU = 6, 7
SENTINEL = 7.0


@pytest.fixture(scope="module")
def lib():
    return _native.require()


def _segments(lib, counts, align, cap):
    """Expert-major capacity layout: expert e owns rows [start, start + count) padded to ``align``; the tile table from the native kernel."""
    starts, pos = [], 0
    for c in counts:
        starts.append(pos)
        pos += (c + align - 1) // align * align
    assert pos <= cap
    seg = torch.tensor(starts + list(counts) + [pos, 0], dtype=torch.int32, device="cuda")
    sticky = torch.zeros(1, dtype=torch.int32, device="cuda")
    tile_group, seg2 = lib.moe_tile_table(seg, len(counts), align, cap, sticky)
    torch.cuda.synchronize()
    assert int(sticky) == 0
    return starts, tile_group, seg2


def _rows(cap, width, starts, counts, align, dtype, g, scale=1.0):
    """[cap, width]: NaN in blocks no expert owns (nothing may read them), zero in an expert's padding rows, random on its token rows."""
    t = torch.full((cap, width), float("nan"), device="cuda", dtype=dtype)
    for s0, c in zip(starts, counts):
        t[s0:s0 + (c + align - 1) // align * align] = 0
        t[s0:s0 + c] = (torch.randn(c, width, device="cuda", generator=g) * scale).to(dtype)
    return t


def _e_gemm(K):
    return R.FP32_U * math.sqrt(K) + R.MMA_ACC


CASES = [  # (experts, hidden = K of FFN1, F, token counts, alignment, capacity rows): an expert without tokens in each, unused blocks at the end
    (4, 256, 384, [300, 0, 129, 700], 256, 2048),
    (3, 512, 256, [5, 640, 0], 128, 1024),
]


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_swiglu_dual_epilogue_against_float64(lib, case, dtype):
    E, Hd, F, counts, align, cap = CASES[case]
    g = torch.Generator(device="cuda").manual_seed(100 + case)
    starts, tile_group, _ = _segments(lib, counts, align, cap)
    xs = _rows(cap, Hd, starts, counts, align, dtype, g)
    w1 = (torch.randn(E, 2 * F, Hd, device="cuda", generator=g) * 0.08).to(dtype)
    b1 = torch.randn(E, 2 * F, device="cuda", generator=g) * 0.5
    b1[:, 0:32:4] = -200.0          # saturated gates: __expf overflows, s = 0 and h is exactly 0
    b1[:, 2:32:4] = 200.0
    b1 = b1.to(dtype)
    pre = torch.full((cap, 2 * F), SENTINEL, device="cuda", dtype=dtype)
    h = torch.full((cap, F), SENTINEL, device="cuda", dtype=dtype)
    lib.gemm_grouped(xs, w1, b1.reshape(-1), tile_group, pre, True, EPI_BIAS_SWIGLU_DUAL, h, None, align)
    torch.cuda.synchronize()
    e_g = _e_gemm(Hd)
    owners = tile_group.tolist()
    for blk, e in enumerate(owners):
        rows = slice(128 * blk, 128 * (blk + 1))
        if e < 0:
            assert bool((pre[rows] == SENTINEL).all()) and bool((h[rows] == SENTINEL).all()), f"unused block {blk} was written"
            continue
        x64, w64 = xs[rows].double(), w1[e].double()
        pre_ref = x64 @ w64.t() + b1[e].double()
        terms = x64.abs() @ w64.abs().t() + b1[e].double().abs()
        R.assert_close(pre[rows], pre_ref, dtype, scale=terms, n=Hd, approx=R.MMA_ACC, what=f"pre block {blk}")
        a, b = pre_ref[:, 0::2], pre_ref[:, 1::2]
        sa = torch.sigmoid(a)
        # d(a s b) = s (1 + a (1 - s)) b da + a s db, with |da| <= e_g terms_a, |db| <= e_g terms_b; then the SwiGLU arithmetic itself
        prop = (sa * (1 + a * (1 - sa)) * b).abs() * terms[:, 0::2] + (a * sa).abs() * terms[:, 1::2]
        E_act = S.swiglu_bound(pre_ref)["scale"]
        R.assert_close(h[rows], S.swiglu(pre_ref), dtype, scale=prop + E_act / e_g, n=Hd, approx=R.MMA_ACC, what=f"h block {blk}")
        hb = h[rows].float()
        assert bool(torch.isfinite(hb).all())
        assert bool((hb[:, 0:16:2] == 0).all()), "a gate below -88 must give an exact zero"


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_dswiglu_epilogue_against_float64(lib, case, dtype):
    E, Hd, F, counts, align, cap = CASES[case]
    g = torch.Generator(device="cuda").manual_seed(200 + case)
    starts, tile_group, _ = _segments(lib, counts, align, cap)
    dy = _rows(cap, Hd, starts, counts, align, dtype, g)
    w2 = (torch.randn(E, Hd, F, device="cuda", generator=g) * 0.08).to(dtype)     # [E, H, F]: MN-major B of dh = dY W2[e]
    pre = _rows(cap, 2 * F, starts, counts, align, torch.float32, g, scale=2.0)
    for s0, c in zip(starts, counts):
        pre[s0:s0 + c, 0:32:4] = -200.0
        pre[s0:s0 + c, 2:32:4] = 200.0
    pre = pre.to(dtype)
    dpre = torch.full((cap, 2 * F), SENTINEL, device="cuda", dtype=dtype)
    lib.gemm_grouped(dy, w2, None, tile_group, dpre, False, EPI_DSWIGLU, None, pre, align)
    torch.cuda.synchronize()
    e_g = _e_gemm(Hd)
    for blk, e in enumerate(tile_group.tolist()):
        rows = slice(128 * blk, 128 * (blk + 1))
        if e < 0:
            assert bool((dpre[rows] == SENTINEL).all()), f"unused block {blk} was written"
            continue
        dy64, w64 = dy[rows].double(), w2[e].double()
        dh = dy64 @ w64
        dh_terms = dy64.abs() @ w64.abs()
        z = pre[rows]
        a, b = S.split_pairs(z)
        s = torch.sigmoid(a)
        prop = torch.empty_like(dpre[rows], dtype=torch.float64)
        prop[:, 0::2] = (b * s * (1 + a * (1 - s))).abs() * dh_terms
        prop[:, 1::2] = (a * s).abs() * dh_terms
        E_act = S.swiglu_bound(z, None, dh)["scale"]
        R.assert_close(dpre[rows], S.swiglu_grad(dh, z), dtype, scale=prop + E_act / e_g, n=Hd, approx=R.MMA_ACC, what=f"dpre block {blk}")
        got = dpre[rows].float()
        assert bool(torch.isfinite(got).all())
        assert bool((got[:, 0:32:4] == 0).all()) and bool((got[:, 1:32:4] == 0).all()), "a gate below -88 must give exact zeros"


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("recompute_h", [False, True], ids=["saved_h", "recomputed_h"])
def test_grouped_ffn_forward_backward_against_the_float64_loop(lib, dtype, recompute_h):
    from paddlefleetx_b200.models.language_model.moe.grouped_experts import GroupedExperts, grouped_ffn
    from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer

    E, Hd, F, counts, align, cap = 4, 512, 768, [500, 0, 129, 1100], 256, 3072
    torch.manual_seed(7)
    ex = [ExpertLayer(Hd, F, init_std=0.05, dtype=dtype, device="cuda", activation="swiglu") for _ in range(E)]
    holder = torch.nn.ModuleList(ex)          # noqa: F841 (keeps the expert modules alive beside the stacks)
    ge = GroupedExperts(ex)
    with torch.no_grad():
        ge.b1.normal_(0, 0.3); ge.b2.normal_(0, 0.1)
    g = torch.Generator(device="cuda").manual_seed(8)
    starts, tile_group, seg2 = _segments(lib, counts, align, cap)
    xs = _rows(cap, Hd, starts, counts, align, dtype, g, scale=0.5).requires_grad_(True)
    go = _rows(cap, Hd, starts, counts, align, dtype, g, scale=0.1)
    ys = grouped_ffn(xs, tile_group, seg2, ge, None, align, recompute_h=recompute_h)
    ys.backward(go)
    torch.cuda.synchronize()
    tol = 2e-2 if dtype == B16 else 5e-3
    w1, b1, w2, b2 = (t.detach().double() for t in (ge.w1, ge.b1, ge.w2, ge.b2))
    for e, (s0, c) in enumerate(zip(starts, counts)):
        if not c:       # an expert without tokens: exact zero gradients, written (not left uninitialised)
            for t in (ge.w1.grad[e], ge.b1.grad[e], ge.w2.grad[e], ge.b2.grad[e]):
                assert bool((t == 0).all())
            continue
        xe = xs.detach()[s0:s0 + c].double().requires_grad_(True)
        pw = [t[e].clone().requires_grad_(True) for t in (w1, b1, w2, b2)]
        wg, wu, bg, bu = pw[0][0::2], pw[0][1::2], pw[1][0::2], pw[1][1::2]
        ye = torch.nn.functional.linear(torch.nn.functional.silu(xe @ wg.t() + bg) * (xe @ wu.t() + bu), pw[2], pw[3])
        ye.backward(go[s0:s0 + c].double())
        checks = {"y": (ys.detach()[s0:s0 + c], ye.detach()), "dx": (xs.grad[s0:s0 + c], xe.grad), "dw1": (ge.w1.grad[e], pw[0].grad),
                  "db1": (ge.b1.grad[e], pw[1].grad), "dw2": (ge.w2.grad[e], pw[2].grad), "db2": (ge.b2.grad[e], pw[3].grad)}
        for name, (got, ref) in checks.items():
            assert bool(torch.isfinite(got).all()), f"{name} expert {e}"
            assert _rel(got, ref) < tol, f"{name} expert {e}: {_rel(got, ref)}"


def test_moe_layer_sync_free_swiglu_path_matches_the_expert_loop_on_one_gpu():
    from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer, MoELayer

    def make(fused):
        torch.manual_seed(3)
        ex = [ExpertLayer(256, 512, dtype=torch.bfloat16, device="cuda", activation="swiglu") for _ in range(4)]
        return MoELayer(256, ex, gate={"type": "naive", "top_k": 2}, dtype=torch.bfloat16, device="cuda", fused_p2p=fused)

    ref, fus = make(False), make(True)
    assert fus.grouped is not None and fus.grouped.activation == "swiglu"
    sd = ref.state_dict()
    with torch.no_grad():
        for k in sd:
            if k.endswith("bias") and k.startswith("experts."):
                sd[k].normal_(0, 0.2)
    ref.load_state_dict(sd)
    fus.load_state_dict(sd)
    torch.manual_seed(5)
    x = (torch.randn(1000, 256, device="cuda") * 0.5).bfloat16()
    go = (torch.randn(1000, 256, device="cuda") * 0.1).bfloat16()
    outs = []
    for layer in (ref, fus):
        xi = x.clone().requires_grad_(True)
        y = layer(xi)
        y.backward(go)
        grads = {n: p.grad.float() for n, p in layer.named_parameters() if p.grad is not None}
        outs.append((y.detach().float(), xi.grad.float(), grads))
    assert _rel(outs[1][0], outs[0][0]) < 2e-2 and _rel(outs[1][1], outs[0][1]) < 2e-2
    for stacked, lin, attr in (("w1", "htoh4", "weight"), ("b1", "htoh4", "bias"), ("w2", "h4toh", "weight"), ("b2", "h4toh", "bias")):
        want = torch.stack([outs[0][2][f"experts.{e}.{lin}.{attr}"] for e in range(4)])
        assert _rel(outs[1][2][f"grouped.{stacked}"], want) < 2e-2, stacked


def test_swiglu_gpt_moe_trains_on_the_grouped_path_without_aten_activations():
    from test_gpu_models import CFG, SMALL_GPT, _engine, _gpt_batches
    from paddlefleetx_b200.models.language_model.moe.moe_layer import MoELayer
    from paddlefleetx_b200.utils import config as C

    cfg = C.get_config(os.path.join(CFG, "nlp/moe/pretrain_moe_345M_swiglu_single_card.yaml"), SMALL_GPT + ["Model.ffn_hidden_size=512"], nranks=1)
    eng = _engine(cfg)
    layers = [m for m in eng._module.model.modules() if isinstance(m, MoELayer)]
    assert layers and all(m.grouped is not None and m.grouped.activation == "swiglu" for m in layers), "the grouped SwiGLU path was not built"
    assert layers[0].grouped.w1.shape[1:] == (2 * 512, 256)
    batch = _gpt_batches(cfg, 1)[0]
    losses = [float(eng.train_step(batch)) for _ in range(8)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.train_step(batch)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any("gemm_wgmma_kernel" in n for n in names)
    assert not [n for n in names if "silu" in n.lower() or "sigmoid" in n.lower() or "bias_swiglu" in n], sorted(set(names))
    from paddlefleetx_b200.parallel import tp_layers as _tp
    _tp.configure({})
