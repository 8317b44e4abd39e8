"""SwiGLU on the sm_90a kernels (needs an H100): ``bias_swiglu`` forward / backward and the SwiGLU decode GEMV against float64 within the
bounds of ``swiglu_refs`` and ``decode_refs``, a SwiGLU GPT that trains with no library GEMM or activation kernel, and CUDA-graph decoding."""
import os

import numpy as np
import pytest
import torch

import decode_refs as D
import kernel_refs as R
import swiglu_refs as S
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import functional as OF

pytestmark = pytest.mark.gpu

B16, F16 = torch.bfloat16, torch.float16
DTYPES = [B16, F16]
_worst = {}


def _record(name, dtype, r):
    key = f"{name} {str(dtype).split('.')[-1]}"
    _worst[key] = max(_worst.get(key, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(_worst.items()):
        print(f"largest error / bound: {k}: {v:.3g}")


def _inputs(rows, f, dtype, bias, seed=0, gates=()):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(rows, 2 * f, generator=g) * 2.0
    for i, a in enumerate(gates):                 # saturated gates on the first row (gate columns 0, 2, 4, ..); their up values stay
        z[0, 2 * i] = a                           # within +-3, so that a = 1e4 gives h within fp16's range
        z[0, 2 * i + 1] = z[0, 2 * i + 1].clamp(-3.0, 3.0)
    b = torch.randn(2 * f, generator=g) * 0.5 if bias else None
    dh = torch.randn(rows, f, generator=g)
    dev = lambda t, dt: None if t is None else t.to(dt).cuda()
    return dev(z, dtype), (None if b is None else b.cuda()), dev(dh, dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("f", [8, 72, 5632])
@pytest.mark.parametrize("rows", [1, 3, 129, 16384])
@pytest.mark.parametrize("bias", ["none", "same", "fp32"])
def test_bias_swiglu_against_float64(dtype, f, rows, bias):
    z, b32, dh = _inputs(rows, f, dtype, bias != "none", seed=rows + f)
    b = None if b32 is None else (b32 if bias == "fp32" else b32.to(dtype))
    zr = z.clone().requires_grad_(True)
    br = None if b is None else b.clone().requires_grad_(True)
    h = OF.bias_swiglu(zr, br)
    assert h.shape == (rows, f) and h.dtype == dtype
    h.backward(dh)
    torch.cuda.synchronize()
    kb = None if b is None else b.to(dtype)       # the kernel reads the bias in the activation dtype
    _record("bias_swiglu fwd", dtype, R.assert_close(h, S.swiglu(z, kb), dtype, **S.swiglu_bound(z, kb), what="bias_swiglu fwd"))
    gref = S.swiglu_grad(dh, z, kb)
    _record("bias_swiglu bwd", dtype, R.assert_close(zr.grad, gref, dtype, **S.swiglu_bound(z, kb, dh), what="bias_swiglu bwd"))
    if b is not None:
        assert br.grad.dtype == b.dtype and br.grad.shape == b.shape
        want = R.colsum(zr.grad)                   # the bias gradient is the column sum of the 16-bit dz (kernel_refs' colsum)
        R.assert_close(br.grad, want, dtype, scale=R.colsum(zr.grad.abs()), n=rows, what="bias grad")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("gate", [30.0, -30.0, 90.0, -90.0, 1e4, -1e4])
def test_bias_swiglu_saturated_gates(dtype, gate):
    z, _, dh = _inputs(64, 72, dtype, False, seed=7, gates=[gate] * 8)
    b = (torch.randn(144, generator=torch.Generator().manual_seed(1)) * 0.5).to(dtype).cuda()
    b[0:16:2] = 0                                  # the gate bias of the saturated channels is 0, so a = gate exactly
    zr = z.clone().requires_grad_(True)
    h = OF.bias_swiglu(zr, b)
    h.backward(dh)
    torch.cuda.synchronize()
    assert torch.isfinite(h).all() and torch.isfinite(zr.grad).all()
    _record("bias_swiglu saturated fwd", dtype, R.assert_close(h, S.swiglu(z, b), dtype, **S.swiglu_bound(z, b)))
    _record("bias_swiglu saturated bwd", dtype, R.assert_close(zr.grad, S.swiglu_grad(dh, z, b), dtype, **S.swiglu_bound(z, b, dh)))
    if gate < -88:                                 # __expf overflows: the kernel returns the limit 0 for h and both gradients
        assert (h[0, :8] == 0).all() and (zr.grad[0, :16] == 0).all()


def test_bias_swiglu_rejects_bad_shapes():
    lib = _native.require()
    z = torch.randn(4, 24, device="cuda", dtype=B16)                # F = 12 is not a multiple of 8
    with pytest.raises(RuntimeError, match="F % 8"):
        lib.bias_swiglu_fwd(z, None)
    z = torch.randn(4, 32, device="cuda", dtype=B16)
    with pytest.raises(RuntimeError, match="dh"):
        lib.bias_swiglu_bwd(torch.randn(4, 8, device="cuda", dtype=B16), z, None)
    with pytest.raises(RuntimeError, match="bias"):
        lib.bias_swiglu_fwd(z, torch.randn(16, device="cuda", dtype=B16))


# ---------------------------------------------------------------------------------------------------------------- decode GEMV
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("ln,res", [(False, False), (True, False), (True, True), (False, True)])
def test_gemv_swiglu_against_float64(dtype, rows, ln, res):
    K, N = 512, 2 * 1376                               # 1376 pairs: not a multiple of the 8 column groups per CTA
    g = torch.Generator().manual_seed(rows)
    x = (torch.randn(rows, K, generator=g)).to(dtype).cuda()
    w = (torch.randn(N, K, generator=g) * K ** -0.5 * 2).to(dtype).cuda()
    b = (torch.randn(N, generator=g) * 0.5).to(dtype).cuda()
    lnp = ((torch.rand(K, generator=g) + 0.5).to(dtype).cuda(), (torch.randn(K, generator=g) * 0.1).to(dtype).cuda(), 1e-5) if ln else None
    r = (torch.randn(rows, N // 2, generator=g)).to(dtype).cuda() if res else None
    for cols, split in ((0, 0), (2, 1), (4, 2), (2, 8)):   # the heuristic choice, then both column-group widths and several K splits
        _native.require().gemv_set_tuning(cols, split)
        try:
            y = OF.gemv_fused(x, w, b, ln=lnp, residual=r, act="swiglu")
        finally:
            _native.require().gemv_set_tuning(0, 0)
        torch.cuda.synchronize()
        assert y.shape == (rows, N // 2) and y.dtype == dtype
        want, kw = D.gemv_ref(x, w, b, lnp, r, act="swiglu")
        _record("gemv swiglu", dtype, R.assert_close(y, want, dtype, **kw, what=f"gemv swiglu cols {cols} split {split}"))


# ---------------------------------------------------------------------------------------------------------------- GPT
def _gpt_cfg(extra=()):
    from test_gpu_models import CFG, SMALL_GPT
    from paddlefleetx_b200.utils import config as C

    return C.get_config(os.path.join(CFG, "nlp/gpt/pretrain_gpt_345M_single_card.yaml"), SMALL_GPT + ["Model.ffn_activation=swiglu"] + list(extra),
                        nranks=1)


def _reset_tp():
    from paddlefleetx_b200.parallel import tp_layers as _tp
    _tp.configure({})


def test_swiglu_gpt_trains_without_library_kernels(monkeypatch):
    from test_gpu_models import _engine, _gpt_batches

    def refuse(name):
        def f(*a, **k):
            raise AssertionError(f"torch.nn.functional.{name} was called")
        return f
    monkeypatch.setattr(torch.nn.functional, "linear", refuse("linear"))
    monkeypatch.setattr(torch.nn.functional, "scaled_dot_product_attention", refuse("scaled_dot_product_attention"))
    cfg = _gpt_cfg()
    eng = _engine(cfg)
    layer = eng._module.model.gpt.decoder.layers[0]
    assert layer.linear1.weight.shape == (2 * 1024, 256) and layer.linear2.weight.shape == (256, 1024)
    batch = _gpt_batches(cfg, 1)[0]
    OF.reset_launch_count()
    losses = [float(eng.train_step(batch)) for _ in range(12)]
    assert OF.native_launch_count() > 100
    assert np.isfinite(losses).all() and losses[-1] < losses[0] - 0.3, losses
    _reset_tp()


def _step_kernels(extra):
    from test_gpu_models import _engine, _gpt_batches
    from test_gpu_models import CFG, SMALL_GPT
    from paddlefleetx_b200.utils import config as C

    cfg = C.get_config(os.path.join(CFG, "nlp/gpt/pretrain_gpt_345M_single_card.yaml"), SMALL_GPT + list(extra), nranks=1)
    eng = _engine(cfg)
    batch = _gpt_batches(cfg, 1)[0]
    eng.train_step(batch)
    eng.train_step(batch)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        eng.train_step(batch)
        torch.cuda.synchronize()
    _reset_tp()
    return [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_swiglu_step_runs_no_aten_activation_kernels():
    swiglu, gelu = _step_kernels(["Model.ffn_activation=swiglu"]), _step_kernels([])
    # forward + backward in each of the 2 layers, for each of the 2 micro-batches of a step (local batch 4, micro-batch 2)
    assert sum("bias_swiglu_kernel" in n for n in swiglu) == 2 * 2 * 2, sorted(set(swiglu))
    assert not [n for n in swiglu if "silu" in n.lower()]
    mul = lambda names: sorted(n for n in names if "MulFunctor" in n)
    assert len(mul(swiglu)) <= len(mul(gelu)), (mul(swiglu), mul(gelu))                       # the loss mask multiply is in both


def test_swiglu_gpt_fp16_o2_stays_finite():
    from test_gpu_models import _engine, _gpt_batches

    cfg = _gpt_cfg(["Engine.mix_precision.dtype=float16"])
    eng = _engine(cfg)
    assert next(eng._module.model.parameters()).dtype == torch.float16
    batch = _gpt_batches(cfg, 1)[0]
    losses = [float(eng.train_step(batch)) for _ in range(12)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0] - 0.3, losses
    assert all(torch.isfinite(p).all() for p in eng._module.model.parameters())
    _reset_tp()


def test_swiglu_generation_graph_eager_and_recompute_agree():
    from paddlefleetx_b200.models.language_model.gpt import model as gpt
    from paddlefleetx_b200.models.language_model.gpt.generation import GPTForGeneration

    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=1024, hidden_size=256, num_layers=2, num_attention_heads=4, ffn_hidden_size=704, max_position_embeddings=128,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, ffn_activation="swiglu", dtype=B16, device="cuda")
    cfg = dict(max_dec_len=10, decode_strategy="greedy_search", eos_token_id=None, pad_token_id=0)
    eager = GPTForGeneration(core, dict(cfg, use_cuda_graph=False))
    graph = GPTForGeneration(core, dict(cfg, use_cuda_graph=True))
    for bs in (1, 3, 12):
        ids = torch.randint(1, 1000, (bs, 9), device="cuda")
        a, _ = eager.generate(ids)
        b, _ = graph.generate(ids)
        c, _ = graph.generate(ids)
        assert torch.equal(b, c)
        assert (a == b).float().mean() > 0.9, (a, b)       # bf16 ties may flip an argmax; sequences must essentially agree
        seq = ids
        with torch.no_grad():
            for _ in range(a.shape[1]):
                h = core(seq)[:, -1]
                seq = torch.cat([seq, (h @ core.embeddings.word_embeddings.weight.t()).argmax(-1, keepdim=True)], 1)
        assert (seq[:, ids.shape[1]:] == a).float().mean() > 0.9, (seq, a)
