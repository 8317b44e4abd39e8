"""float16 on the native wgmma GEMM and flash-attention kernels (needs an H100).

The numerics tests run every case twice, once on fp16 inputs and once on the same inputs rounded to bf16, and compare each result with an
fp32 reference.  fp16 keeps 11 significant bits against bf16's 8, so a genuine fp16 path lands several times closer to its reference; a
kernel that reads, rounds or multiplies fp16 data as bf16 anywhere lands no closer than bf16 itself.  The bound used throughout is
``err(fp16) < 0.5 * err(bf16)``.  Results stored as 16-bit numbers are compared with a reference built from each dtype's own rounded inputs;
fp32 results (fp32 GEMM stores, the log-sum-exp) carry no output rounding, so they are compared with the reference on the fp32 inputs the
two dtypes were rounded from.
"""
import os

import numpy as np
import pytest
import torch

from paddlefleetx_b200.ops import attention as ATT
from paddlefleetx_b200.ops import functional as OF
from paddlefleetx_b200.ops import _native

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16
EPI_NONE, EPI_BIAS, EPI_BIAS_GELU = 0, 1, 2


def _lib():
    return _native.require()


def _rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _gelu(x):
    return torch.nn.functional.gelu(x, approximate="tanh")


def _compare(run, ref, masters, own=None):
    """run(*inputs in dtype) and ref(*fp32 inputs) return tuples of results.  ``own[i]`` says whether result i is a 16-bit output
    (reference from the dtype's own rounded inputs) or an fp32 one (reference from the fp32 masters).  Returns {dtype: [errors]}."""
    errs = {}
    for dt in (F16, B16):
        ins = [m.to(dt) if m.is_floating_point() else m for m in masters]
        got = run(*ins)
        torch.cuda.synchronize()
        want_own = ref(*[i.float() if i.is_floating_point() else i for i in ins])
        want_master = ref(*masters)
        errs[dt] = [_rel(g, wo if (own is None or own[i]) else wm) for i, (g, wo, wm) in enumerate(zip(got, want_own, want_master))]
    return errs


def _assert_fp16_closer(errs, bf16_bound=3e-2):
    for i, (e16, eb) in enumerate(zip(errs[F16], errs[B16])):
        assert eb < bf16_bound, ("bf16 result is off", i, errs)
        assert e16 < 0.5 * eb, ("fp16 result is not closer to fp32 than bf16's", i, errs)


# ---------------------------------------------------------------------------------------------------------------- GEMM
def _gemm_case(a_k, b_k, M, N, K, epilogue=EPI_NONE, out_mode=0):
    torch.manual_seed(0)
    A, B = torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda")
    bias = torch.randn(N, device="cuda") if epilogue in (EPI_BIAS, EPI_BIAS_GELU) else None
    acc0 = torch.randn(M, N, device="cuda") if out_mode == 2 else None

    def run(a, b, *rest):
        bb = rest[0] if bias is not None else None
        out = acc0.clone() if acc0 is not None else None
        return (_lib().gemm(a if a_k else a.t().contiguous(), b if b_k else b.t().contiguous(), bb, out, a_k, b_k, epilogue, out_mode, 0),)

    def ref(a, b, *rest):
        y = a @ b.t()
        if bias is not None:
            y = y + rest[0]
        if epilogue == EPI_BIAS_GELU:
            y = _gelu(y)
        return (y + acc0 if acc0 is not None else y,)

    masters = [A, B] + ([bias] if bias is not None else [])
    return _compare(run, ref, masters, own=[out_mode == 0])


GEMM_CASES = {
    "nt": dict(a_k=True, b_k=True, M=512, N=512, K=256),
    "nn": dict(a_k=True, b_k=False, M=512, N=512, K=256),
    "tn": dict(a_k=False, b_k=True, M=512, N=512, K=256),
    "tt": dict(a_k=False, b_k=False, M=512, N=512, K=256),
    "tail": dict(a_k=True, b_k=True, M=300, N=264, K=136),
    "bias": dict(a_k=True, b_k=True, M=384, N=256, K=256, epilogue=EPI_BIAS),
    "bias_gelu": dict(a_k=True, b_k=True, M=384, N=256, K=256, epilogue=EPI_BIAS_GELU),
    # the wgrad form (both operands MN-major) storing into / accumulating onto an fp32 main_grad
    "wgrad_f32_store": dict(a_k=False, b_k=False, M=256, N=384, K=512, out_mode=1),
    "wgrad_f32_accumulate": dict(a_k=False, b_k=False, M=256, N=384, K=512, out_mode=2),
}


@pytest.mark.parametrize("name", list(GEMM_CASES))
def test_gemm_fp16(name):
    _assert_fp16_closer(_gemm_case(**GEMM_CASES[name]))


def test_gemm_fp16_bias_must_match_operands():
    a = torch.randn(128, 64, device="cuda", dtype=F16)
    with pytest.raises(RuntimeError, match="bias"):
        _lib().gemm(a, a, torch.zeros(128, device="cuda", dtype=B16), None, True, True, EPI_BIAS, 0, 0)


def test_ffn1_dual_output_fp16():
    torch.manual_seed(1)
    M, H, Fh = 300, 256, 1032
    masters = [torch.randn(M, H, device="cuda"), torch.randn(Fh, H, device="cuda") * 0.05, torch.randn(Fh, device="cuda") * 0.1]

    def ref(x, w, b):
        z = x @ w.t() + b
        return z, _gelu(z)

    errs = _compare(lambda x, w, b: tuple(_lib().gemm_bias_gelu_dual(x, w, b)), ref, masters)
    _assert_fp16_closer(errs)


def test_dgelu_fp16():
    torch.manual_seed(2)
    M, K, N = 300, 256, 1032
    masters = [torch.randn(M, K, device="cuda"), torch.randn(K, N, device="cuda") * 0.05, torch.randn(M, N, device="cuda")]

    def ref(dy, w, z):
        zz = z.clone().requires_grad_(True)
        with torch.enable_grad():
            (_gelu(zz) * (dy @ w)).sum().backward()
        return (zz.grad,)

    _assert_fp16_closer(_compare(lambda dy, w, z: (_lib().gemm_dgelu(dy, w, z),), ref, masters))


@pytest.mark.parametrize("M,N,K,split", [(4, 512, 512, 1), (16, 512, 1024, 2), (33, 4096, 4096, 0), (100, 2048, 4096, 0), (128, 4096, 4096, 4)])
def test_smallm_fp16(M, N, K, split):
    """The swap-AB small-M GEMM, including the split-K reduction through distributed shared memory and the bias."""
    torch.manual_seed(3)
    masters = [torch.randn(M, K, device="cuda"), torch.randn(N, K, device="cuda") * 0.05, torch.randn(N, device="cuda")]
    errs = _compare(lambda x, w, b: (_lib().gemm_smallm(x, w, b, split),), lambda x, w, b: (x @ w.t() + b,), masters)
    _assert_fp16_closer(errs)


def test_grouped_rows_fp16():
    """Grouped mode 1: each 128-row block multiplies the weight slice of the expert that owns it, plus that expert's bias."""
    torch.manual_seed(4)
    G, K, N = 3, 256, 384
    tile_group = torch.tensor([2, 0, 0, 1], dtype=torch.int32, device="cuda")
    owner = tile_group.long().repeat_interleave(128)
    masters = [torch.randn(4 * 128, K, device="cuda"), torch.randn(G, N, K, device="cuda") * 0.05, torch.randn(G, N, device="cuda")]

    def run(a, b, bias):
        out = torch.empty(a.shape[0], N, device="cuda", dtype=a.dtype)
        return (_lib().gemm_grouped(a, b, bias.reshape(-1), tile_group, out, True, EPI_BIAS, None, None, 128),)

    def ref(a, b, bias):
        return (torch.einsum("mk,mnk->mn", a, b[owner]) + bias[owner],)

    _assert_fp16_closer(_compare(run, ref, masters))


def test_grouped_wgrad_fp16():
    """Grouped mode 2: out[g] = dy[rows of g]^T x[rows of g] over each expert's (start, padded count) token range."""
    torch.manual_seed(5)
    G, Mg, N = 2, 128, 256
    segs = [(0, 192), (192, 128)]
    seg2 = torch.tensor([v for s in segs for v in s], dtype=torch.int32, device="cuda")
    R = sum(c for _, c in segs)
    masters = [torch.randn(R, Mg, device="cuda"), torch.randn(R, N, device="cuda")]

    def run(dy, x):
        out = torch.empty(G, Mg, N, device="cuda", dtype=dy.dtype)
        return (_lib().gemm_grouped_wgrad(dy, x, seg2, out),)

    def ref(dy, x):
        return (torch.stack([dy[s:s + c].t() @ x[s:s + c] for s, c in segs]),)

    _assert_fp16_closer(_compare(run, ref, masters))


def test_fp16_overflow_is_inf():
    """A product beyond 65504 comes out as +-inf (what the dynamic loss scaler detects), as torch.matmul in fp16 does, never as NaN or a
    saturated finite value."""
    a = torch.full((256, 64), 64.0, device="cuda", dtype=F16)
    b = torch.full((128, 64), 64.0, device="cuda", dtype=F16)
    b[64:] = -64.0                                   # every dot product is +-64^3 = +-262144
    d = _lib().gemm(a, b, None, None, True, True, EPI_NONE, 0, 0)
    ref = torch.matmul(a, b.t())
    torch.cuda.synchronize()
    assert torch.isinf(ref).all()
    assert torch.isinf(d).all() and not torch.isnan(d).any()
    assert torch.equal(torch.sign(d), torch.sign(ref))


# ---------------------------------------------------------------------------------------------------------------- flash attention
ATTN_CASES = [  # B, Sq, Sk, H, causal, p, layout, D
    (2, 256, 256, 2, True, 0.0, "plain", 128), (2, 200, 200, 3, False, 0.0, "plain", 128), (1, 128, 256, 2, True, 0.0, "plain", 128),
    (1, 192, 320, 2, False, 0.0, "plain", 64), (2, 577, 577, 4, False, 0.1, "plain", 64), (2, 512, 512, 4, True, 0.1, "packed", 128),
    (1, 300, 300, 2, True, 0.0, "packed", 64), (2, 384, 384, 2, True, 0.1, "seq_major", 128), (2, 197, 197, 3, False, 0.0, "seq_major", 64)]


def _views(masters, layout, dt):
    """q, k, v in the requested storage (read in place by the kernels) and matching gradient views."""
    q, k, v = (m.to(dt) for m in masters)
    if layout == "plain":
        return (q, k, v), tuple(torch.empty_like(t) for t in (q, k, v))
    mix = torch.stack([q, k, v], dim=3)                      # [B, S, H, 3, D]
    if layout == "seq_major":
        mix = mix.transpose(0, 1).contiguous().transpose(0, 1)
        dmix = torch.empty_like(mix.transpose(0, 1)).transpose(0, 1)
    else:
        dmix = torch.empty_like(mix)
    return mix.unbind(3), dmix.unbind(3)


@pytest.mark.parametrize("case", ATTN_CASES, ids=lambda c: "B{}_Sq{}_Sk{}_H{}_{}_p{}_{}_D{}".format(*c[:4], "causal" if c[4] else "full", *c[5:]))
def test_flash_attention_fp16(case):
    B, Sq, Sk, H, causal, p, layout, D = case
    torch.manual_seed(6)
    scale = D ** -0.5
    seed = 0x1234567 + 977 * Sq
    keep = ATT.attn_keep_mask(seed, B, H, Sq, Sk, p, "cuda") if p > 0 else None
    masters = [torch.randn(B, Sq, H, D, device="cuda"), torch.randn(B, Sk, H, D, device="cuda"), torch.randn(B, Sk, H, D, device="cuda"),
               torch.randn(B, Sq, H, D, device="cuda") * 0.5]
    errs = {}
    for dt in (F16, B16):
        (q, k, v), (dq, dk, dv) = _views(masters[:3], layout, dt)
        go = masters[3].to(dt)
        out, lse = _lib().attention_fwd_v2(q, k, v, causal, scale, p, seed)
        _lib().attention_bwd(q, k, v, out, go, lse, dq, dk, dv, causal, scale, p, seed)
        torch.cuda.synchronize()
        assert out.dtype == dt and dq.dtype == dt

        def ref(qr, kr, vr):
            qr, kr, vr = (t.detach().clone().requires_grad_(True) for t in (qr, kr, vr))
            with torch.enable_grad():
                s = torch.einsum("bqhd,bkhd->bhqk", qr, kr) * scale
                if causal:
                    s = s.masked_fill(~torch.ones(Sq, Sk, dtype=torch.bool, device="cuda").tril(Sk - Sq), float("-inf"))
                pr = torch.softmax(s, -1)
                if keep is not None:
                    pr = pr * keep.float() / (1.0 - p)
                o = torch.einsum("bhqk,bkhd->bqhd", pr, vr)
                o.backward(go.float())
            return o.detach(), torch.logsumexp(s.detach(), -1), qr.grad, kr.grad, vr.grad

        own = ref(*(t.float() for t in (q, k, v)))
        master_lse = ref(*masters[:3])[1]
        errs[dt] = [_rel(out, own[0]), _rel(lse, master_lse), _rel(dq, own[2]), _rel(dk, own[3]), _rel(dv, own[4])]
    _assert_fp16_closer(errs)


def test_dropout_keeps_the_same_pairs_in_fp16_and_bf16():
    """With q = k = 0 every probability is 1 / Sk, and with V = identity each output channel is one key's (kept, rescaled) probability:
    the output's non-zeros are the keep mask.  Both dtypes must drop exactly the pairs attn_keep_mask names for the seed."""
    B, Sq, Sk, H, D, p, seed = 2, 100, 128, 3, 128, 0.25, 987654321
    masks = []
    for dt in (F16, B16):
        q = torch.zeros(B, Sq, H, D, device="cuda", dtype=dt)
        k = torch.zeros(B, Sk, H, D, device="cuda", dtype=dt)
        v = torch.eye(Sk, D, device="cuda", dtype=dt).view(1, Sk, 1, D).expand(B, Sk, H, D).contiguous()
        out, _ = _lib().attention_fwd_v2(q, k, v, False, D ** -0.5, p, seed)
        masks.append((out.float() > 0).permute(0, 2, 1, 3))          # [B, H, Sq, Sk]
    want = ATT.attn_keep_mask(seed, B, H, Sq, Sk, p, "cuda")
    assert torch.equal(masks[0], want) and torch.equal(masks[1], want)
    assert 0.6 < float(want.float().mean()) < 0.9


def test_flash_attention_packed_fp16_returns_one_packed_gradient():
    torch.manual_seed(7)
    B, S, H, D = 2, 256, 4, 128
    mix = torch.randn(B, S, H, 3, D, device="cuda", dtype=F16).requires_grad_(True)
    go = torch.randn(B, S, H, D, device="cuda", dtype=F16)
    out = ATT.flash_attention_packed(mix, causal=True)
    assert out is not None and out.dtype == F16
    out.backward(go)
    assert mix.grad is not None and mix.grad.dtype == F16 and mix.grad.shape == mix.shape
    q, k, v = (t.detach().float().requires_grad_(True) for t in mix.detach().unbind(3))
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * D ** -0.5
    s = s.masked_fill(~torch.ones(S, S, dtype=torch.bool, device="cuda").tril(), float("-inf"))
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v)
    ref.backward(go.float())
    assert _rel(out, ref) < 2e-3
    assert _rel(mix.grad, torch.stack([q.grad, k.grad, v.grad], dim=3)) < 5e-3


@pytest.mark.parametrize("c,s,d", [(2, 1024, 128), (4, 2048, 64)])
def test_ring_block_schedule_fp16(c, s, d):
    """The single-GPU replay of the ring-attention block schedule (tests/test_ring_attention_blocks.py) with fp16 blocks."""
    from paddlefleetx_b200.parallel import ring_attention as R
    from test_ring_attention_blocks import _reference, _replay

    torch.manual_seed(2)
    b, h = 2, 4
    masters = [torch.randn(b, s, h, d, device="cuda") for _ in range(3)] + [torch.randn(b, s, h, d, device="cuda") * 0.5]
    errs = {}
    for dt in (F16, B16):
        q, k, v, do = (m.to(dt) for m in masters)
        loc = R.zigzag_slice(q, c, 1)
        assert R.ATT._native_ok(loc, loc, loc, None, True, True) and R.ATT._native_ok(loc[:, loc.shape[1] // 2:], loc, loc, None, False, True)
        got = _replay(q, k, v, do, c, True, d ** -0.5)
        ref = _reference(q, k, v, do, True, d ** -0.5)
        errs[dt] = [_rel(a, r_) for a, r_ in zip(got, ref)]
    _assert_fp16_closer(errs)


# ---------------------------------------------------------------------------------------------------------------- models
def _gpt_cfg(dtype, extra=()):
    from test_gpu_models import CFG, SMALL_GPT
    from paddlefleetx_b200.utils import config as C

    return C.get_config(os.path.join(CFG, "nlp/gpt/pretrain_gpt_345M_single_card.yaml"),
                        SMALL_GPT + [f"Engine.mix_precision.dtype={dtype}"] + list(extra), nranks=1)


@pytest.fixture
def no_library_kernels(monkeypatch):
    """torch.nn.functional.linear / scaled_dot_product_attention raise: a step that still reaches cuBLAS or SDPA fails."""
    def refuse(name):
        def f(*a, **k):
            raise AssertionError(f"torch.nn.functional.{name} was called")
        return f
    monkeypatch.setattr(torch.nn.functional, "linear", refuse("linear"))
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", refuse("scaled_dot_product_attention"))


def _one_step_launches(dtype):
    from test_gpu_models import _engine, _gpt_batches

    cfg = _gpt_cfg(dtype)
    eng = _engine(cfg)
    assert next(eng._module.model.parameters()).dtype == getattr(torch, dtype)
    batch = _gpt_batches(cfg, 1)[0]
    eng.train_step(batch)                                   # first step: lazily built state (optimizer buckets, tensor-map cache)
    OF.reset_launch_count()
    loss = float(eng.train_step(batch))
    assert np.isfinite(loss)
    from paddlefleetx_b200.parallel import tp_layers as _tp
    _tp.configure({})
    return OF.native_launch_count()


def test_gpt_step_uses_no_library_gemm_or_attention(no_library_kernels):
    counts = {dt: _one_step_launches(dt) for dt in ("bfloat16", "float16")}
    assert counts["float16"] == counts["bfloat16"] > 100, counts


def test_gpt_trains_in_fp16_with_the_dynamic_scaler():
    from test_gpu_models import _engine, _gpt_batches

    cfg = _gpt_cfg("float16", ["Engine.mix_precision.scale_loss=32768.0"])
    eng = _engine(cfg)
    assert next(eng._module.model.parameters()).dtype == F16 and eng._scaler is not None
    batch = _gpt_batches(cfg, 1)[0]
    losses = [float(eng.train_step(batch)) for _ in range(12)]          # same batch: the loss must go down
    assert np.isfinite(losses).all() and losses[-1] < losses[0] - 0.3, losses
    from paddlefleetx_b200.parallel import tp_layers as _tp
    _tp.configure({})


def test_gpt_first_step_fp16_is_at_least_as_close_to_fp32_as_bf16():
    """Loss and gradient norm of one forward + backward, for fp16 and bf16 copies of the same weights, against the fp32 model."""
    from paddlefleetx_b200.models.language_model.gpt import model as gpt

    def build(dtype):
        torch.manual_seed(0)
        core = gpt.GPTModel(vocab_size=1024, hidden_size=256, num_layers=2, num_attention_heads=4, ffn_hidden_size=1024, max_position_embeddings=128,
                            hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, dtype=torch.float32, device="cuda")
        return gpt.GPTForPretraining(core).to(dtype)

    torch.manual_seed(1)
    tokens = torch.randint(0, 1024, (4, 129), device="cuda")
    x, y = tokens[:, :-1].contiguous(), tokens[:, 1:].contiguous()
    mask = torch.ones(4, 128, device="cuda")
    crit = gpt.GPTPretrainingCriterion()
    res = {}
    for dt, scale in ((torch.float32, 1.0), (F16, 1024.0), (B16, 1.0)):        # fp16: a static loss scale keeps small gradients normal
        model = build(dt)
        loss = crit(model(x), y, mask)
        (loss * scale).backward()
        gn = torch.sqrt(sum((p.grad.double() / scale).pow(2).sum() for p in model.parameters() if p.grad is not None))
        res[dt] = (float(loss), float(gn))
    l32, g32 = res[torch.float32]
    d16 = (abs(res[F16][0] - l32), abs(res[F16][1] - g32) / g32)
    db = (abs(res[B16][0] - l32), abs(res[B16][1] - g32) / g32)
    assert np.isfinite(res[F16]).all() and d16[0] <= db[0] and d16[1] <= db[1], res


def test_moe_trains_in_fp16_on_the_grouped_gemms(monkeypatch):
    from test_gpu_models import CFG, SMALL_GPT, _engine, _gpt_batches
    from paddlefleetx_b200.models.language_model.moe import grouped_experts as GE
    from paddlefleetx_b200.models.language_model.moe.moe_layer import MoELayer
    from paddlefleetx_b200.utils import config as C

    calls = []
    real = GE.grouped_ffn
    monkeypatch.setattr(GE, "grouped_ffn", lambda *a, **k: calls.append(1) or real(*a, **k))
    cfg = C.get_config(os.path.join(CFG, "nlp/moe/pretrain_moe_345M_single_card.yaml"),
                       SMALL_GPT + ["Model.moe_configs.fused_p2p=True", "Engine.mix_precision.dtype=float16"], nranks=1)
    eng = _engine(cfg)
    layers = [m for m in eng._module.model.modules() if isinstance(m, MoELayer)]
    assert layers and all(m.grouped is not None and m.grouped.w1.dtype == F16 for m in layers)
    batch = _gpt_batches(cfg, 1)[0]
    losses = [float(eng.train_step(batch)) for _ in range(6)]
    assert calls, "the grouped expert GEMMs were not used"
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses
