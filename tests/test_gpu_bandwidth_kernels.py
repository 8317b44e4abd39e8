"""The bandwidth-bound kernels against float64 references, in bf16 and fp16 (needs an H100).

Covers LayerNorm / RMSNorm forward and backward, bias + GELU, bias + dropout + residual, column sums, softmax cross-entropy, the
squared-norm / clip / AdamW optimizer kernels, rotary embedding and the causal softmax.  Every case runs through the bindings directly
and, where one exists, through the autograd router in ``ops.functional``.  Bounds come from ``kernel_refs.assert_close`` (see its
docstring).  Each 16-bit case runs in both dtypes on the same inputs and the fp16 error must be well under the bf16 one: fp16 keeps three
more significant bits, so a kernel that computes or rounds in the wrong 16-bit type anywhere cannot meet that.

Run with ``-s`` to print the largest error/bound ratio seen per kernel and dtype.
"""
import math
from collections import defaultdict

import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import functional as OF

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


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _close(kernel, got, ref, dtype, **kw):
    r = R.assert_close(got, ref, dtype, what=kernel, **kw)
    RATIOS[(kernel, dtype)] = max(RATIOS[(kernel, dtype)], r)
    return R.rel_err(got, ref)


def _fp16_closer(errs, what):
    """errs: {dtype: relative error of the same computation on the same inputs}."""
    assert errs[F16] < 0.5 * errs[B16], (what, "fp16 is not closer to the reference than bf16", errs)


def _randn(*shape, seed=0, scale=1.0, offset=0.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale + offset


# ================================================================================================================ norms
NORM_COLS = [8, 64, 264, 768, 1024, 1032, 2048, 2056, 4096, 4104, 8192, 8200, 16384, 16392, 32768]
NORM_KINDS = ["ln_bias_res", "ln_nobias", "rms", "rms_res"]


def _norm_case(kind, rows, cols, offset=0.0, const_rows=False, eps=1e-5):
    rms, has_bias, has_res = kind.startswith("rms"), kind == "ln_bias_res", kind.endswith("_res")
    xm = _randn(rows, cols, seed=1, offset=offset)
    if const_rows:
        xm[::2] = xm[::2, :1]                          # every other row constant: (x - mean) = 0, only eps keeps rstd finite
    wm, bm = _randn(cols, seed=2, scale=0.5, offset=1.0), _randn(cols, seed=3)
    dym, dresm = _randn(rows, cols, seed=4), _randn(rows, cols, seed=5)
    errs = {}
    for dt in DTYPES:
        x, w, b, dy, dres = (t.to(dt) for t in (xm, wm, bm, dym, dresm))
        y, mean, rstd = _lib().norm_fwd(x, w, b if has_bias else None, eps, rms)
        dx, dw, db = _lib().norm_bwd(dy, x, w, mean, rstd, rms, has_bias, dres if has_res else None)
        torch.cuda.synchronize()
        xd, wd, dyd = x.double(), w.double(), dy.double()
        if rms:
            yr, rstd_r = R.rms_norm(x, w, eps)
            mean_r = torch.zeros_like(rstd_r)
        else:
            yr, mean_r, rstd_r = R.layer_norm(x, w, b if has_bias else None, eps)
        dxr, dwr, dbr = R.norm_bwd(dy, x, w, b if has_bias else None, eps, rms, dres if has_res else None)
        rs, mu = rstd_r[:, None], mean_r[:, None]
        xhat = (xd - mu) * rs
        # fp32 error of the statistics: the row mean is formed from |x| ~ |mean|, and that error moves every xhat by |mean| * rstd
        shift = mu.abs() * rs
        e = [_close("norm_fwd.y", y, yr, dt, scale=yr.abs() + (shift + xhat.abs()) * wd.abs(), n=cols)]
        if not rms:
            _close("norm_fwd.mean", mean, mean_r, F32, scale=xd.abs().mean(-1), n=cols)
        _close("norm_fwd.rstd", rstd, rstd_r, F32, scale=rstd_r * (1 + shift.squeeze(-1)), n=cols, approx=2.0 ** -22)
        gw = dyd * wd
        c2 = (gw * xhat).mean(-1, keepdim=True)
        sdx = rs * (gw.abs() + gw.abs().mean(-1, keepdim=True) + (xhat.abs() + shift) * c2.abs()) + (dres.double().abs() if has_res else 0)
        e.append(_close("norm_bwd.dx", dx, dxr, dt, scale=sdx, n=cols))
        e.append(_close("norm_bwd.dw", dw, dwr, dt, scale=(dyd.abs() * (xhat.abs() + shift)).sum(0), n=rows))
        if has_bias:
            e.append(_close("norm_bwd.db", db, dbr, dt, scale=dyd.abs().sum(0), n=rows))
        else:
            assert db.numel() == 0
        errs[dt] = e
    return errs


@pytest.mark.parametrize("cols", NORM_COLS)
@pytest.mark.parametrize("kind", NORM_KINDS)
def test_norm_columns(kind, cols):
    """Every backward (VPT, threads) instantiation, on both sides of each switch."""
    rows = 2 * _sms() + 1
    errs = _norm_case(kind, rows, cols)
    for i in range(len(errs[B16])):
        if i < 2 or cols >= 64:                        # dw / db of 8 columns are too few numbers to compare two dtypes' errors
            _fp16_closer({dt: errs[dt][i] for dt in DTYPES}, (kind, cols, i))


@pytest.mark.parametrize("cols", [768, 4104])
@pytest.mark.parametrize("rows_kind", ["1", "3", "2sm-1", "2sm+1", "16k"])
@pytest.mark.parametrize("kind", ["ln_bias_res", "rms_res"])
def test_norm_rows_offset_inputs(kind, rows_kind, cols):
    """Row counts around the persistent backward's grid (2 CTAs per SM), on inputs offset by +100 (one-pass variance cancels there)."""
    rows = {"1": 1, "3": 3, "2sm-1": 2 * _sms() - 1, "2sm+1": 2 * _sms() + 1, "16k": 16384 + 7}[rows_kind]
    if cols == 4104 and rows > 1000:
        rows = 4099
    _norm_case(kind, rows, cols, offset=100.0)


@pytest.mark.parametrize("kind", NORM_KINDS)
def test_norm_constant_rows(kind):
    _norm_case(kind, 2 * _sms() + 1, 1032, const_rows=True)


@pytest.mark.parametrize("dtype", DTYPES)
def test_norm_routers_autograd(dtype):
    torch.manual_seed(0)
    x0 = _randn(4, 33, 768, seed=6).to(dtype)
    w, b = _randn(768, seed=7, offset=1.0).to(dtype), _randn(768, seed=8).to(dtype)
    g, g2 = _randn(4, 33, 768, seed=9).to(dtype), _randn(4, 33, 768, seed=10).to(dtype)
    for name, rms in (("layer_norm", False), ("rms_norm", True), ("norm_with_residual", False), ("norm_with_residual_rms", True)):
        x, wl, bl = (t.clone().requires_grad_(True) for t in (x0, w, b))
        eps = 1e-6 if rms else 1e-5
        OF.reset_launch_count()
        if name.startswith("norm_with_residual"):
            y, res = OF.norm_with_residual(x, wl, None if rms else bl, eps, rms=rms)
            torch.autograd.backward([y, res], [g, g2])
            dres = g2
        else:
            y = OF.rms_norm(x, wl, eps) if rms else OF.layer_norm(x, wl, bl, eps)
            y.backward(g)
            dres = None
        assert OF.native_launch_count() >= 2, name
        yr = (R.rms_norm(x0, w, eps)[0] if rms else R.layer_norm(x0, w, b, eps)[0]).view_as(y)
        dxr, dwr, dbr = R.norm_bwd(g.view(-1, 768), x0.view(-1, 768), w, None if rms else b, eps, rms, None if dres is None else dres.view(-1, 768))
        R.assert_close(y, yr, dtype, scale=yr.abs() + 1, n=768, what=name)
        R.assert_close(x.grad.view(-1, 768), dxr, dtype, scale=dxr.abs() + g.double().abs().view(-1, 768) * 4, n=768, what=name)
        R.assert_close(wl.grad, dwr, dtype, scale=(g.double().abs() * 4).sum((0, 1)), n=132, what=name)
        if not rms:
            R.assert_close(bl.grad, dbr, dtype, scale=g.double().abs().sum((0, 1)), n=132, what=name)
        else:
            assert bl.grad is None


# ================================================================================================================ bias + GELU
@pytest.mark.parametrize("rows,cols", [(1000, 8), (4099, 1160), (7, 64)])
@pytest.mark.parametrize("with_bias", [True, False])
@pytest.mark.parametrize("exact", [True, False])
def test_bias_gelu(exact, with_bias, rows, cols):
    xm = (_randn(rows, cols, seed=1) * 3).clamp(-10, 10)
    k = min(2001, xm.numel())
    xm.view(-1)[:k] = torch.linspace(-10, 10, k, device="cuda")
    bm, dym = _randn(cols, seed=2, scale=0.5), _randn(rows, cols, seed=3)
    errs = {}
    for dt in DTYPES:
        x, b, dy = xm.to(dt), bm.to(dt), dym.to(dt)
        bb = b if with_bias else None
        y = _lib().bias_gelu_fwd(x, bb, exact)
        dx = _lib().bias_gelu_bwd(dy, x, bb, exact)
        torch.cuda.synchronize()
        xb = x.double() + (b.double() if with_bias else 0)
        yr, gr = R.gelu(xb, exact), R.gelu_grad(xb, exact)
        e = [_close("bias_gelu_fwd" + ("_erf" if exact else "_tanh"), y, yr, dt, **R.gelu_bound(xb, yr, exact))]
        kw = R.gelu_bound(xb, gr, exact, grad=True)
        kw["scale"] = kw["scale"] * dy.double().abs()
        e.append(_close("bias_gelu_bwd" + ("_erf" if exact else "_tanh"), dx, dy.double() * gr, dt, **kw))
        errs[dt] = e
    for i in range(2):
        _fp16_closer({dt: errs[dt][i] for dt in DTYPES}, ("gelu", exact, i))


@pytest.mark.parametrize("dtype", DTYPES)
def test_bias_gelu_router(dtype):
    x0 = _randn(3, 40, 256, seed=4).to(dtype)
    b0 = _randn(256, seed=5).to(dtype)
    g = _randn(3, 40, 256, seed=6).to(dtype)
    for exact in (False, True):
        x, b = x0.clone().requires_grad_(True), b0.clone().requires_grad_(True)
        y = OF.bias_gelu(x, b, exact=exact)
        y.backward(g)
        xb = x0.double() + b0.double()
        yr, dxr = R.gelu(xb, exact), g.double() * R.gelu_grad(xb, exact)
        R.assert_close(y, yr, dtype, **R.gelu_bound(xb, yr, exact))
        kw = R.gelu_bound(xb, dxr, exact, grad=True)
        kw["scale"] = kw["scale"] * g.double().abs()
        R.assert_close(x.grad, dxr, dtype, **kw)
        gx = x.grad.double().reshape(-1, 256)                   # the bias gradient is the column sum of the 16-bit input gradient
        R.assert_close(b.grad, gx.sum(0), dtype, scale=gx.abs().sum(0), n=120)


# ================================================================================================================ dropout
def _dropout(dt, x, b, r, p, seed=1234, offset=77):
    return _lib().bias_dropout_add_fwd(x.to(dt), None if b is None else b.to(dt), None if r is None else r.to(dt), p, seed, offset)


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_dropout_exact(p):
    rows, cols = 1031, 520
    xm, bm, rm = _randn(rows, cols, seed=1), _randn(cols, seed=2), _randn(rows, cols, seed=3)
    scale = R.dropout_scale(p)
    masks = {}
    for dt in DTYPES:
        x, b, r = xm.to(dt), bm.to(dt), rm.to(dt)
        y = _dropout(dt, x, b, r, p)
        ones = torch.ones(rows, cols, device="cuda", dtype=dt)
        kept = _lib().dropout_bwd(ones, p, 1234, 77) != 0
        dyy = _randn(rows, cols, seed=4).to(dt)
        dx = _lib().dropout_bwd(dyy, p, 1234, 77)
        torch.cuda.synchronize()
        masks[dt] = kept
        # the backward zeroes exactly what the forward dropped, and scales the rest by the quantised 1 / (1 - p)
        assert torch.equal(dx == 0, ~kept | (dyy == 0))
        assert torch.equal(dx[kept], (dyy.float()[kept] * scale).to(dt))
        # dropped elements are the residual; kept ones are (x + b) * scale + res with one or two fp32 roundings (fused or not)
        assert torch.equal(y[~kept], r[~kept])
        xb = x.float() + b.float()
        two = ((xb * scale) + r.float()).to(dt)
        fused = (xb.double() * scale + r.double()).float().to(dt)
        assert bool(((y == two) | (y == fused))[kept].all())
        frac = kept.double().mean().item()
        n = kept.numel()
        sd = math.sqrt(p * (1 - p) / n)
        assert abs(frac - (1 - p)) < 6 * sd, (frac, p)
    assert torch.equal(masks[B16], masks[F16]), "the mask depends on the dtype"


def test_dropout_mask_does_not_depend_on_the_grid():
    rows, cols = 2 * 4099, 1160                     # the [2R, C] call runs with the grid capped, the [R, C] call with fewer CTAs
    ones = torch.ones(rows, cols, device="cuda", dtype=B16)
    big = _lib().dropout_bwd(ones, 0.3, 99, 5) != 0
    small = _lib().dropout_bwd(ones[: rows // 2].contiguous(), 0.3, 99, 5) != 0
    tiny = _lib().dropout_bwd(ones[:3].contiguous(), 0.3, 99, 5) != 0
    assert torch.equal(big[: rows // 2], small)
    assert torch.equal(big[:3], tiny)


@pytest.mark.parametrize("dtype", DTYPES)
def test_dropout_p0_is_the_plain_sum(dtype):
    x, b, r = _randn(33, 64, seed=1).to(dtype), _randn(64, seed=2).to(dtype), _randn(33, 64, seed=3).to(dtype)
    y = _lib().bias_dropout_add_fwd(x, b, r, 0.0, 1, 0)
    assert torch.equal(y, ((x.float() + b.float()) + r.float()).to(dtype))
    assert torch.equal(_lib().bias_dropout_add_fwd(x, None, None, 0.0, 1, 0), x)


@pytest.mark.parametrize("dtype", DTYPES)
def test_dropout_router(dtype):
    x = _randn(4, 32, 128, seed=1).to(dtype).requires_grad_(True)
    b = _randn(128, seed=2).to(dtype).requires_grad_(True)
    r = _randn(4, 32, 128, seed=3).to(dtype).requires_grad_(True)
    y = OF.bias_dropout_add(x, b, r, 0.25, True)
    g = _randn(4, 32, 128, seed=4).to(dtype)
    y.backward(g)
    kept = x.grad != 0
    scale = R.dropout_scale(0.25)
    assert torch.equal(y[~kept & (g != 0)], r.detach()[~kept & (g != 0)])
    assert torch.equal(x.grad[kept], (g.float()[kept] * scale).to(dtype))
    assert torch.equal(r.grad, g)
    R.assert_close(b.grad, x.grad.double().reshape(-1, 128).sum(0), dtype, scale=x.grad.double().abs().reshape(-1, 128).sum(0), n=128)


# ================================================================================================================ colsum
@pytest.mark.parametrize("rows", [1, 7, 33, 8191, 100000])
@pytest.mark.parametrize("cols", [8, 264, 1000])
def test_colsum(rows, cols):
    xm = _randn(rows, cols, seed=rows + cols, offset=0.5)
    errs = {}
    for dt in DTYPES:
        x = xm.to(dt)
        ref = R.colsum(x)
        sc = x.double().abs().sum(0)
        e = []
        for out_fp32 in (True, False):
            got = _lib().colsum(x, out_fp32)
            assert got.dtype == (F32 if out_fp32 else dt)
            e.append(_close("colsum" + ("_f32out" if out_fp32 else ""), got, ref, F32 if out_fp32 else dt, scale=sc, n=rows))
        errs[dt] = e
    if rows > 1:
        _fp16_closer({dt: errs[dt][1] for dt in DTYPES}, ("colsum", rows, cols))


# ================================================================================================================ cross-entropy
CE_V = [8, 1000, 50304, 7, 129, 30522]


def _ce_logits(rows, V, scale, seed, neg_inf=False):
    lm = _randn(rows, V, seed=seed, scale=scale)
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    labels = torch.randint(0, V, (rows,), device="cuda", generator=g)
    labels[0] = 0
    labels[-1] = V - 1
    if neg_inf:
        lm[:, : min(V - 1, 40)] = -math.inf                       # leading run: every thread's first vectors / elements are -inf
        lm[:, V // 2: V // 2 + V // 4] = -math.inf
        labels = torch.where((labels < 40) | ((labels >= V // 2) & (labels < V // 2 + V // 4)), torch.full_like(labels, V - 1), labels)
    return lm, labels


def _ce_check(logits, labels, dt, vocab_start=0, what="ce"):
    lib = _lib()
    mx, sm, tg = lib.ce_stats(logits, labels, vocab_start)
    torch.cuda.synchronize()
    mxr, smr, tgr = R.ce_stats(logits, labels, vocab_start)
    assert torch.equal(mx.double(), mxr), what
    assert torch.equal(tg.double(), tgr), what
    xd = logits.double()
    dev = (xd - mxr[:, None]).abs().nan_to_num(0, 0, 0)
    _close(what + ".row_sum", sm, smr, F32, scale=(torch.exp(xd - mxr[:, None]) * (1 + dev)).sum(-1), n=logits.shape[-1], approx=2.0 ** -21)
    lse = mx + torch.log(sm)
    gs = _randn(logits.shape[0], seed=11).abs() + 0.1
    work = logits.clone()
    lib.ce_bwd_(work, labels, lse, gs, vocab_start)
    torch.cuda.synchronize()
    gr = R.ce_grad(logits, labels, lse, gs, vocab_start)
    p = torch.exp(xd - lse.double()[:, None])
    onehot = (torch.arange(logits.shape[-1], device="cuda")[None, :] == (labels - vocab_start)[:, None]).double()
    sc = gs.double()[:, None] * (p * (1 + (xd - lse.double()[:, None]).abs().nan_to_num(0, 0, 0)) + onehot)
    return _close(what + ".grad", work, gr, dt, scale=sc, approx=2.0 ** -21)


@pytest.mark.parametrize("rows", [1, 3, 2048])
@pytest.mark.parametrize("V", CE_V)
def test_ce(V, rows):
    for scale in (1.0, 30.0):
        lm, labels = _ce_logits(rows, V, scale, seed=V + rows)
        errs = {dt: _ce_check(lm.to(dt), labels, dt, what="ce") for dt in DTYPES}
        if rows == 2048 and scale == 1.0:              # with fewer rows, or at scale 30, a handful of entries carry the whole gradient
            _fp16_closer(errs, ("ce", V, rows, scale))


@pytest.mark.parametrize("V", [129, 1000, 30522])
def test_ce_neg_inf_runs(V):
    lm, labels = _ce_logits(5, V, 3.0, seed=V, neg_inf=True)
    for dt in DTYPES:
        _ce_check(lm.to(dt), labels, dt, what="ce_neginf")
        loss = OF.softmax_cross_entropy(lm.to(dt).clone(), labels)
        assert torch.isfinite(loss).all()
        ref = torch.nn.functional.cross_entropy(lm.to(dt).double(), labels, reduction="none")
        R.assert_close(loss, ref, F32, scale=ref.abs() + 10, n=V, approx=2.0 ** -21)


@pytest.mark.parametrize("V", [1000, 30522, 50304])
def test_ce_vocab_shard(V):
    """A shard [vocab_start, vocab_start + Vs) of a larger vocabulary, with labels inside and outside it."""
    rows, start = 64, 3 * V
    lm, labels = _ce_logits(rows, V, 3.0, seed=V)
    labels = labels + torch.where(torch.arange(rows, device="cuda") % 3 == 0, 0, start)   # a third of the rows point at other shards
    labels[1] = start
    labels[2] = start + V - 1
    labels[3] = start + V                                                                 # one past the shard
    for dt in DTYPES:
        _ce_check(lm.to(dt), labels, dt, vocab_start=start, what="ce_shard")


@pytest.mark.parametrize("V", [8, 7, 129, 30522, 50304])
@pytest.mark.parametrize("dtype", DTYPES)
def test_ce_router(V, dtype):
    rows = 3 * 37
    lm, labels = _ce_logits(rows, V, 4.0, seed=V)
    logits = lm.to(dtype).view(3, 37, V)
    lab = labels.view(3, 37)
    x = logits.clone().requires_grad_(True)
    OF.reset_launch_count()
    loss = OF.softmax_cross_entropy(x.clone(), lab)
    gl = _randn(3, 37, seed=3)
    loss.backward(gl)
    assert OF.native_launch_count() >= 2
    xd = logits.double().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(xd.view(-1, V), labels, reduction="none")
    ref.backward(gl.double().view(-1))
    R.assert_close(loss.view(-1), ref, F32, scale=ref.abs() + 4, n=V, approx=2.0 ** -21)
    gmag = gl.double().abs().view(3, 37, 1)
    p = torch.softmax(logits.double(), -1)
    R.assert_close(x.grad, xd.grad, dtype, scale=gmag * (p * (1 + (logits.double() - logits.double().logsumexp(-1, keepdim=True)).abs()) + 1e-3),
                   approx=2.0 ** -20)


def test_ce_unaligned_base():
    """A view whose first row is not 16-byte aligned takes the scalar kernels."""
    buf = _randn(2 * 1000 + 8, seed=5, scale=2.0)
    labels = torch.tensor([3, 999], device="cuda")
    for dt in DTYPES:
        flat = buf.to(dt)
        logits = flat[1: 1 + 2000].view(2, 1000)
        assert logits.data_ptr() % 16 != 0
        _ce_check(logits, labels, dt, what="ce_unaligned")


# ================================================================================================================ optimizer
OPT_N = [1, 3, 7, 8, 4097, 2 ** 20 + 5]
PAIRS = [(F32, None), (F32, F32), (F32, B16), (F32, F16), (B16, None), (B16, B16), (B16, F32), (F16, None), (F16, F16), (F16, F32)]


@pytest.mark.parametrize("n", OPT_N)
@pytest.mark.parametrize("dtype", [F32, B16, F16])
def test_sumsq(dtype, n):
    x = _randn(n + 1, seed=n).to(dtype)
    out = torch.zeros(1, device="cuda")
    for view in (x[:n], x[1:]):                     # x[1:] is 2 bytes off 16-byte alignment: the scalar path
        _lib().sumsq_(view, out, False)
        ref = R.sumsq(view)
        _close("sumsq", out[0], ref, F32, scale=ref, n=n)
        before = out.clone()
        _lib().sumsq_(view, out, True)
        _close("sumsq_acc", out[0], before.double()[0] + ref, F32, scale=2 * ref + before.double()[0], n=n)


@pytest.mark.parametrize("clip", [0.0, 1.0])
@pytest.mark.parametrize("pair", PAIRS, ids=lambda p: f"{p[0]}-{p[1]}".replace("torch.", ""))
@pytest.mark.parametrize("n", OPT_N)
def test_adamw_three_steps(n, pair, clip):
    gdt, lpdt = pair
    lib = _lib()
    # the kernel takes its hyperparameters as fp32; the reference gets the same values
    lr, b1, b2, eps, wd = (float(torch.tensor(h, dtype=F32)) for h in (2e-3, 0.9, 0.95, 1e-8, 0.1))
    inv_scale = 1.0 / 1024
    master = _randn(n, seed=1)
    m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    lp = None if lpdt is None else master.to(lpdt, copy=True)
    rm, rmm, rv = master.double(), m.double(), v.double()
    sq, gscale, found, gnorm = (torch.zeros(1, device="cuda") for _ in range(4))
    mterms = vterms = torch.zeros(n, device="cuda", dtype=torch.float64)   # decayed sums of |terms| that formed m and v
    for step in (1, 2, 3):
        grad = (_randn(n, seed=10 + step) * 1024 * 3).to(gdt)           # scaled by the loss scale, as the optimizer sees it
        lib.sumsq_(grad, sq, False)
        lib.clip_coef_(sq, inv_scale, clip, gscale, found, gnorm)
        lib.adamw_flat_(lp, master, grad, m, v, lr, b1, b2, eps, wd, step, gscale, found, 0)
        torch.cuda.synchronize()
        gs_r, fi_r, gn_r = R.clip_coef(R.sumsq(grad), inv_scale, clip)
        assert found.item() == fi_r == 0.0
        _close("clip_coef.gnorm", gnorm[0], torch.tensor(gn_r, dtype=torch.float64), F32, n=n, approx=2.0 ** -21)
        _close("clip_coef.gscale", gscale[0], torch.tensor(gs_r, dtype=torch.float64), F32, n=n, approx=2.0 ** -21)
        # the reference takes the kernel's fp32 gscale, so the update itself is what is compared
        rm, rmm, rv = R.adamw_step(rm, grad, rmm, rv, lr, b1, b2, eps, wd, step, gscale.double().item())
        gmag = grad.double().abs() * gscale.double().item()
        mterms, vterms = b1 * mterms + gmag, b2 * vterms + gmag * gmag
        _close("adamw.m", m, rmm, F32, scale=mterms, n=2 * step)
        _close("adamw.v", v, rv, F32, scale=vterms, n=2 * step)
        _close("adamw.master", master, rm, F32, scale=rm.abs() + lr * 3, n=2 * step, approx=2.0 ** -22)
        if lp is not None:
            assert torch.equal(lp, master.to(lpdt)), "the low-precision copy is not the rounded master"


@pytest.mark.parametrize("gdt", [F32, B16, F16])
def test_adamw_skips_a_step_with_inf_grads(gdt):
    lib = _lib()
    n = 4097
    lpdt = B16 if gdt == F32 else gdt
    master, m, v = _randn(n, seed=1), _randn(n, seed=2) * 0.1, _randn(n, seed=3).abs() * 0.01
    lp = master.to(lpdt)
    grad = _randn(n, seed=4).to(gdt)
    grad[1234] = math.inf
    sq, gscale, found, gnorm = (torch.zeros(1, device="cuda") for _ in range(4))
    lib.sumsq_(grad, sq, False)
    lib.clip_coef_(sq, 0.5, 1.0, gscale, found, gnorm)
    before = [t.clone() for t in (master, m, v, lp)]
    lib.adamw_flat_(lp, master, grad, m, v, 1e-3, 0.9, 0.95, 1e-8, 0.1, 5, gscale, found, 0)
    torch.cuda.synchronize()
    assert found.item() == 1.0 and gscale.item() == 0.0
    for a, b in zip(before, (master, m, v, lp)):
        assert torch.equal(a.view(torch.int32) if a.dtype == F32 else a.view(torch.int16), b.view(torch.int32) if b.dtype == F32 else b.view(torch.int16))


def test_adamw_cta_budget_is_bitwise_identical():
    lib = _lib()
    n = 2 ** 20 + 5
    grad = _randn(n, seed=1).to(B16)
    outs = []
    for budget in (0, 8, 100):
        master, m, v = _randn(n, seed=2), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        lp = master.to(B16)
        lib.adamw_flat_(lp, master, grad, m, v, 1e-3, 0.9, 0.95, 1e-8, 0.1, 1, None, None, budget)
        outs.append((master, m, v, lp))
    for o in outs[1:]:
        for a, b in zip(outs[0], o):
            assert torch.equal(a, b)


@pytest.mark.parametrize("n", OPT_N)
@pytest.mark.parametrize("dtype", [F32, B16, F16])
def test_accumulate_f32(dtype, n):
    dst0 = _randn(n, seed=1)
    src = _randn(n, seed=2).to(dtype)
    for scale in (1.0, 0.37):
        dst = dst0.clone()
        _lib().accumulate_f32_(dst, src, scale)
        ref = dst0.double() + src.double() * scale
        _close("accumulate_f32", dst, ref, F32, scale=dst0.double().abs() + src.double().abs())


# ================================================================================================================ rope
def _torch_rope_fp32(x, pos, base=10000.0):
    """The fp32 expression ``functional.rope`` falls back to, on [tokens, heads, d]."""
    d = x.shape[-1]
    inv = base ** (-torch.arange(0, d, 2, device=x.device, dtype=torch.float32) / d)
    ang = pos.float()[:, None] * inv
    cs, sn = ang.cos()[:, None, :], ang.sin()[:, None, :]
    xf = x.float()
    x1, x2 = xf[..., : d // 2], xf[..., d // 2:]
    return torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], -1).to(x.dtype)


@pytest.mark.parametrize("d", [32, 64, 80, 128])
def test_rope(d):
    tokens, heads = 1024, 4
    g = torch.Generator(device="cuda").manual_seed(d)
    pos = torch.randint(0, 32768, (tokens,), device="cuda", generator=g)
    pos[:4] = torch.tensor([32767, 0, 1, 32766])
    xm = _randn(tokens, heads, d, seed=d)
    errs = {}
    for dt in (B16, F16, F32):
        x = xm.to(dt)
        y = _lib().rope(x, pos, 0, 10000.0, False)
        back = _lib().rope(x, pos, 0, 10000.0, True)
        torch.cuda.synchronize()
        ref, refb = R.rope(x, pos), R.rope(x, pos, inverse=True)
        # any fp32 evaluation rounds the angle pos * inv_freq, an absolute error of up to |angle| * 2^-24
        sc = x.double().abs().amax(-1, keepdim=True) * (1 + pos.double()[:, None, None])
        errs[dt] = _close("rope", y, ref, dt, scale=sc)
        _close("rope_bwd", back, refb, dt, scale=sc)
        e_torch = R.rel_err(_torch_rope_fp32(x, pos), ref)
        assert errs[dt] <= 1.25 * e_torch + 1e-7, ("rope is less accurate than the fp32 torch expression", dt, errs[dt], e_torch)
    _fp16_closer(errs, ("rope", d))


@pytest.mark.parametrize("dtype", [B16, F16, F32])
def test_rope_router_autograd(dtype):
    b, s, h, d = 2, 96, 4, 64
    x = _randn(b, s, h, d, seed=1).to(dtype).requires_grad_(True)
    pos = torch.randperm(s * 4, device="cuda")[: b * s].view(b, s)
    g = _randn(b, s, h, d, seed=2).to(dtype)
    for positions in (None, pos):
        x.grad = None
        y = OF.rope(x, positions)
        y.backward(g)
        p = (torch.arange(s, device="cuda").repeat(b) if positions is None else positions.reshape(-1))
        ref = R.rope(x.detach().view(b * s, h, d), p).view_as(y)
        dref = R.rope(g.view(b * s, h, d), p, inverse=True).view_as(y)
        sc = x.detach().double().abs().amax(-1, keepdim=True) * (1 + p.double().view(b, s, 1, 1))
        R.assert_close(y, ref, dtype, scale=sc)
        R.assert_close(x.grad, dref, dtype, scale=g.double().abs().amax(-1, keepdim=True) * (1 + p.double().view(b, s, 1, 1)))


# ================================================================================================================ causal softmax
@pytest.mark.parametrize("batch,sq,sk", [(3, 64, 64), (2, 48, 100), (4, 1, 1), (2, 7, 33), (1, 128, 4096)])
def test_causal_softmax(batch, sq, sk):
    xm = _randn(batch, sq, sk, seed=sk, scale=3.0)
    dym = _randn(batch, sq, sk, seed=sk + 1)
    scale = 0.37
    errs = {}
    for dt in (B16, F16, F32):
        x, dy = xm.to(dt), dym.to(dt)
        y = _lib().causal_softmax_fwd(x, scale)
        dx = _lib().causal_softmax_bwd(dy, y, scale)
        torch.cuda.synchronize()
        yr = R.causal_softmax(x, scale)
        dev = (x.double() * scale - (x.double() * scale).masked_fill(~R.causal_mask(sq, sk, x.device), -math.inf).amax(-1, keepdim=True)).abs()
        errs[dt] = _close("causal_softmax_fwd", y, yr, dt, scale=yr * (1 + dev), n=sk, approx=2.0 ** -21)
        dxr = R.causal_softmax_bwd(dy, y, scale)                 # against the kernel's own y: the backward is checked on its own
        ydd = y.double()
        sc = scale * ydd * (dy.double().abs() + (dy.double() * ydd).abs().sum(-1, keepdim=True))
        _close("causal_softmax_bwd", dx, dxr, dt, scale=sc, n=sk)
        assert torch.equal(y.masked_fill(R.causal_mask(sq, sk, x.device), 0), torch.zeros_like(y))
    if sk > 1:
        _fp16_closer(errs, ("causal_softmax", sq, sk))


# ================================================================================================================ refusals
def test_refusals():
    lib = _lib()
    x32 = torch.randn(4, 64, device="cuda")
    w32 = torch.randn(64, device="cuda")
    f = torch.zeros(4, device="cuda")
    lab = torch.zeros(4, dtype=torch.long, device="cuda")
    calls = {
        "norm_fwd": lambda: lib.norm_fwd(x32, w32, None, 1e-5, False),
        "norm_bwd": lambda: lib.norm_bwd(x32, x32, w32, f, f, False, False, None),
        "bias_gelu_fwd": lambda: lib.bias_gelu_fwd(x32, None, False),
        "bias_gelu_bwd": lambda: lib.bias_gelu_bwd(x32, x32, None, False),
        "bias_dropout_add_fwd": lambda: lib.bias_dropout_add_fwd(x32, None, None, 0.1, 1, 0),
        "dropout_bwd": lambda: lib.dropout_bwd(x32, 0.1, 1, 0),
        "colsum": lambda: lib.colsum(x32, True),
        "ce_stats": lambda: lib.ce_stats(x32, lab, 0),
        "ce_bwd_": lambda: lib.ce_bwd_(x32, lab, f, f, 0),
    }
    for name, call in calls.items():
        with pytest.raises(RuntimeError, match="bf16 or fp16"):
            call()
    n = 64
    master, m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    for gdt, lpdt in ((B16, F16), (F16, B16)):
        lp = torch.zeros(n, device="cuda", dtype=lpdt)
        with pytest.raises(RuntimeError, match="p_lp"):
            lib.adamw_flat_(lp, master, torch.zeros(n, device="cuda", dtype=gdt), m, v, 1e-3, 0.9, 0.95, 1e-8, 0.0, 1, None, None, 0)
        assert torch.equal(lp, torch.zeros_like(lp))
    for size in (n - 8, n + 8):
        with pytest.raises(RuntimeError, match="p_lp"):
            lib.adamw_flat_(torch.zeros(size, device="cuda", dtype=B16), master, torch.zeros(n, device="cuda", dtype=B16), m, v, 1e-3, 0.9,
                            0.95, 1e-8, 0.0, 1, None, None, 0)
    for cols in (12, 32776):
        xb = torch.zeros(2, cols, device="cuda", dtype=B16)
        wb = torch.ones(cols, device="cuda", dtype=B16)
        with pytest.raises(RuntimeError):
            lib.norm_fwd(xb, wb, None, 1e-5, True)
        with pytest.raises(RuntimeError):
            lib.norm_bwd(xb, xb, wb, torch.zeros(2, device="cuda"), torch.ones(2, device="cuda"), True, False, None)
    torch.cuda.synchronize()
