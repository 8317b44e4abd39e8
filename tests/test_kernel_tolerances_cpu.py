"""The error bounds in ``kernel_refs`` are tight enough to matter.

For every operation the GPU tests check, the correct float64 result rounded to the output dtype must pass ``assert_close`` and a result
built with a plausible kernel mistake (rounded the same way) must fail it, in bf16 and in fp16.  A bound that lets one of these mistakes
through would let the kernel make it too.
"""
import math

import pytest
import torch

import kernel_refs as R

DTYPES = [torch.bfloat16, torch.float16]


def _check(dtype, ref, wrong, **kw):
    """``ref`` rounded to ``dtype`` passes; ``wrong`` rounded to ``dtype`` is rejected."""
    R.assert_close(ref.to(dtype), ref, dtype, **kw)
    with pytest.raises(AssertionError):
        R.assert_close(wrong.to(dtype), ref, dtype, **kw)


def _gen(seed=0):
    return torch.Generator().manual_seed(seed)


def _in(shape, dtype, seed=0, scale=1.0, offset=0.0):
    """16-bit test inputs: the exact values a kernel would be given."""
    return (torch.randn(shape, generator=_gen(seed), dtype=torch.float64) * scale + offset).to(dtype)


# ---------------------------------------------------------------------------------------------------------------- norms
@pytest.mark.parametrize("dtype", DTYPES)
def test_layer_norm_eps_is_seen_on_near_constant_rows(dtype):
    x = _in((16, 256), dtype, scale=2e-3, offset=1.0)
    w, b = _in((256,), dtype, 1), _in((256,), dtype, 2)
    ref = R.layer_norm(x, w, b, 1e-5)[0]
    _check(dtype, ref, R.layer_norm(x, w, b, 1e-6)[0])


@pytest.mark.parametrize("dtype", DTYPES)
def test_layer_norm_rejects_unbiased_variance(dtype):
    x, w, b = _in((16, 64), dtype), _in((64,), dtype, 1), _in((64,), dtype, 2)
    ref = R.layer_norm(x, w, b, 1e-5)[0]
    xd = x.double()
    mean = xd.mean(-1, keepdim=True)
    wrong = (xd - mean) / torch.sqrt(xd.var(-1, unbiased=True, keepdim=True) + 1e-5) * w.double() + b.double()
    _check(dtype, ref, wrong)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rms_norm_rejects_mean_subtraction(dtype):
    x, w = _in((16, 256), dtype, offset=0.3), _in((256,), dtype, 1)
    ref = R.rms_norm(x, w, 1e-6)[0]
    _check(dtype, ref, R.layer_norm(x, w, None, 1e-6)[0])


@pytest.mark.parametrize("dtype", DTYPES)
def test_norm_weight_grad_rejects_dropped_rows(dtype):
    # dw is a reduction over rows: a CTA whose partial never reaches the sum must be caught despite the sum-of-|terms| allowance
    x, w, b, dy = _in((300, 64), dtype), _in((64,), dtype, 1), _in((64,), dtype, 2), _in((300, 64), dtype, 3)
    _, dw, _ = R.norm_bwd(dy, x, w, b, 1e-5, False)
    _, dw_short, _ = R.norm_bwd(dy[:-1], x[:-1], w, b, 1e-5, False)
    y, mean, rstd = R.layer_norm(x, w, b, 1e-5)
    terms = (dy.double() * (x.double() - mean[:, None]) * rstd[:, None]).abs().sum(0)
    _check(dtype, dw, dw_short, scale=terms, n=300)


# ---------------------------------------------------------------------------------------------------------------- GELU
@pytest.mark.parametrize("dtype", DTYPES)
def test_gelu_erf_rejects_the_tanh_form(dtype):
    # the two forms agree to 5e-4 for |x| < 3; they separate, relative to the result, in the negative tail
    x = torch.linspace(-6.0, 3.0, 901, dtype=torch.float64).to(dtype)
    ref, dref = R.gelu(x, True), R.gelu_grad(x, True)
    _check(dtype, ref, R.gelu(x, False), **R.gelu_bound(x, ref, True))
    _check(dtype, dref, R.gelu_grad(x, False), **R.gelu_bound(x, dref, True, grad=True))


@pytest.mark.parametrize("dtype", DTYPES)
def test_gelu_tanh_bound_is_wider_than_the_erf_difference(dtype):
    """The tanh-GELU kernels evaluate tanh with tanh.approx.f32, whose documented error (2^-10.987) is larger than the whole difference
    between the tanh and erf forms (at most 3.6e-4 in units of t).  So a bound every correct tanh kernel meets cannot reject an erf
    kernel in its place; that mistake is caught by the erf kernels' own bound instead.  If the kernels ever evaluate tanh accurately,
    this test fails and the tanh bound can be tightened."""
    x = torch.linspace(-6.0, 3.0, 901, dtype=torch.float64).to(dtype)
    ref = R.gelu(x, False)
    R.assert_close(ref.to(dtype), ref, dtype, **R.gelu_bound(x, ref, False))
    R.assert_close(R.gelu(x, True).to(dtype), ref, dtype, **R.gelu_bound(x, ref, False))


# ---------------------------------------------------------------------------------------------------------------- dropout
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p", [0.1, 0.3])
def test_dropout_rejects_scale_of_one_over_p(dtype, p):
    x = _in((64, 64), dtype)
    keep = torch.rand((64, 64), generator=_gen(5)) >= p
    ref = x.double() * keep * R.dropout_scale(p)
    _check(dtype, ref, x.double() * keep / p)


# ---------------------------------------------------------------------------------------------------------------- column sums
@pytest.mark.parametrize("dtype", DTYPES)
def test_colsum_rejects_a_missing_part(dtype):
    x = _in((4096, 64), dtype)
    ref = R.colsum(x)
    terms = x.double().abs().sum(0)
    _check(dtype, ref, R.colsum(x[32:]), scale=terms, n=4096)


# ---------------------------------------------------------------------------------------------------------------- cross-entropy
def _ce_inputs(dtype, rows=32, V=1000):
    logits = _in((rows, V), dtype, scale=3.0)
    labels = torch.randint(0, V - 1, (rows,), generator=_gen(7))
    return logits, labels


@pytest.mark.parametrize("dtype", DTYPES)
def test_ce_rejects_target_off_by_one(dtype):
    logits, labels = _ce_inputs(dtype)
    ref = R.ce_loss(logits, labels)
    _check(torch.float32, ref, R.ce_loss(logits, labels + 1), scale=ref.abs() + 1)
    lse = R.ce_stats(logits, labels)[0] + torch.log(R.ce_stats(logits, labels)[1])
    g = torch.ones(32, dtype=torch.float64)
    _check(dtype, R.ce_grad(logits, labels, lse, g), R.ce_grad(logits, labels + 1, lse, g), scale=1.0)


@pytest.mark.parametrize("dtype", DTYPES)
def test_ce_rejects_ignoring_vocab_start(dtype):
    logits, labels = _ce_inputs(dtype)
    start = 500
    labels = labels % 500 + torch.where(torch.arange(32) % 2 == 0, 0, start)   # half the labels fall in the shard
    mx, sm, tg = R.ce_stats(logits[:, start:], labels, start)
    _, _, tg_wrong = R.ce_stats(logits[:, start:], labels.clamp(max=499), 0)
    _check(torch.float32, tg, tg_wrong, scale=tg.abs() + 1)
    lse = mx + torch.log(sm)
    g = torch.ones(32, dtype=torch.float64)
    _check(dtype, R.ce_grad(logits[:, start:], labels, lse, g, start), R.ce_grad(logits[:, start:], labels.clamp(max=499), lse, g, 0),
           scale=1.0)


# ---------------------------------------------------------------------------------------------------------------- AdamW
def _adam_state(n=4096):
    master = torch.randn(n, generator=_gen(1), dtype=torch.float64)
    grad = torch.randn(n, generator=_gen(2), dtype=torch.float64)
    m = torch.randn(n, generator=_gen(3), dtype=torch.float64) * 0.1
    v = torch.rand(n, generator=_gen(4), dtype=torch.float64) * 0.01
    return master, grad, m, v


@pytest.mark.parametrize("step", [1, 3])
def test_adamw_rejects_missing_bias_correction(step):
    master, grad, m, v = _adam_state()
    args = (1e-3, 0.9, 0.95, 1e-8, 0.1)
    ref = R.adamw_step(master, grad, m, v, *args, step)[0]
    g = grad
    m2 = 0.9 * m + 0.1 * g
    v2 = 0.95 * v + 0.05 * g * g
    wrong = master * (1 - 1e-3 * 0.1) - 1e-3 * m2 / (v2.sqrt() + 1e-8)
    _check(torch.float32, ref, wrong, scale=master.abs())


def test_adamw_rejects_coupled_weight_decay():
    master, grad, m, v = _adam_state()
    lr, wd = 1e-3, 0.1
    ref = R.adamw_step(master, grad, m, v, lr, 0.9, 0.95, 1e-8, wd, 2)[0]
    wrong = R.adamw_step(master, grad + wd * master, m, v, lr, 0.9, 0.95, 1e-8, 0.0, 2)[0]   # L2 folded into the gradient
    _check(torch.float32, ref, wrong, scale=master.abs())


# ---------------------------------------------------------------------------------------------------------------- rotary
def _interleaved_rope(x, pos, base=10000.0):
    x = x.double()
    d = x.shape[-1]
    inv = base ** (-torch.arange(0, d // 2, dtype=torch.float64) * 2.0 / d)
    ang = pos.double()[:, None] * inv
    cs, sn = torch.cos(ang)[:, None, :], torch.sin(ang)[:, None, :]
    x1, x2 = x[..., 0::2], x[..., 1::2]
    return torch.stack([x1 * cs - x2 * sn, x2 * cs + x1 * sn], -1).flatten(-2)


@pytest.mark.parametrize("dtype", DTYPES)
def test_rope_rejects_interleaved_pairs_and_inverse_rotation(dtype):
    x = _in((64, 4, 64), dtype)
    pos = torch.randint(0, 4096, (64,), generator=_gen(3))
    ref = R.rope(x, pos)
    _check(dtype, ref, _interleaved_rope(x, pos), scale=x.double().abs().amax(-1, keepdim=True))
    _check(dtype, ref, R.rope(x, pos, inverse=True), scale=x.double().abs().amax(-1, keepdim=True))


# ---------------------------------------------------------------------------------------------------------------- causal softmax
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shift", [1, -1])
def test_causal_softmax_rejects_shifted_diagonal(dtype, shift):
    sq, sk = 24, 40
    x = _in((2, sq, sk), dtype)
    ref = R.causal_softmax(x, 0.5)
    keep = torch.arange(sk)[None, :] <= torch.arange(sq)[:, None] + (sk - sq) + shift
    wrong = torch.softmax((x.double() * 0.5).masked_fill(~keep, -math.inf), -1)
    _check(dtype, ref, wrong)


def test_bounds_accept_only_roundoff_sized_errors():
    """Sanity of the bound itself: a relative perturbation of 1.5 u fails (normwise), one of 0.5 u passes."""
    ref = torch.linspace(0.5, 2.0, 1000, dtype=torch.float64)
    for dt in DTYPES:
        u = R.UNIT_ROUNDOFF[dt]
        R.assert_close(ref * (1 + 0.5 * u), ref, dt)
        with pytest.raises(AssertionError):
            R.assert_close(ref * (1 + 1.5 * u), ref, dt)
