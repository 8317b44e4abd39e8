"""float64 references and error bounds for the bandwidth-bound kernels (norms, GELU, dropout, column sums, cross-entropy, AdamW,
rotary embedding, causal softmax) and for the 8-bit path (per-row and MX quantisers, int8 / fp8 / MX GEMMs, the W8A8 GEMV).  Nothing
here needs CUDA: the references run on whatever device their inputs live on.

Every reference takes the exact values a kernel was given (16-bit inputs upcast, never re-rounded) and computes in float64, so the only
differences left are the kernel's own: fp32 arithmetic, approximate intrinsics and the final rounding to the output dtype.

``assert_close`` bounds that difference with the output dtype's unit roundoff ``u`` (2^-8 bf16, 2^-11 fp16, 2^-24 fp32):

    |got - ref| <= c * (u * (|ref| + tiny) + e * scale + 2^-122)   for every element        (c = 4)
    ||got - ref|| <= cn * (u * ||ref|| + e * ||scale||)  over the whole tensor    (cn = 1)

with ``e = 2^-24 * sqrt(n) + approx`` and ``tiny`` the dtype's smallest normal number (for results that underflow).  ``scale`` is the magnitude of the terms a result is formed from (the sum of |terms| for a
reduction of ``n`` terms); it covers fp32 cancellation, which a bound relative to |ref| alone cannot.  ``approx`` is the relative error of
an approximate intrinsic the kernel is built on.  A pure rounding to the output dtype has ||err|| <= u * ||ref||, so the normwise bound
is tight; the elementwise bound catches a few badly wrong elements that a norm would average away.
"""
from __future__ import annotations

import math

import numpy as np
import torch

UNIT_ROUNDOFF = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 2.0 ** -24}
FP32_U = 2.0 ** -24
FTZ_FLOOR = 2.0 ** -122
# tanh.approx.f32 (the tanh-GELU kernels): the PTX ISA gives a maximum relative error of 2^-10.987
TANH_APPROX = 2.0 ** -10.987


def _d(t):
    """float64 view of t; float64 tensors pass through so that float64 autograd sees the references' operations."""
    return t if t.dtype == torch.float64 else t.detach().to(torch.float64)


def error_ratio(got, ref, dtype, scale=None, n=1, approx=0.0, c=4.0, cn=1.0):
    """max over (elementwise, normwise) of error / bound; <= 1 passes."""
    got, ref = _d(got).detach(), _d(ref).detach()
    u = UNIT_ROUNDOFF[dtype]
    e = FP32_U * math.sqrt(max(n, 1)) + approx
    sc = ref.abs() if scale is None else _d(torch.as_tensor(scale, device=ref.device)).abs().expand_as(ref)
    err = (got - ref).abs()
    if not torch.isfinite(got).all():
        return math.inf
    # gradual underflow: below the smallest normal number a rounding error is at most u * smallest_normal, not u * |ref|; and the
    # kernels' fp32 arithmetic flushes results under 2^-126 to zero (--use_fast_math), which bf16 outputs can represent
    elem = c * (u * (ref.abs() + torch.finfo(dtype).smallest_normal) + e * sc + FTZ_FLOOR) + 1e-300
    norm = cn * (u * ref.norm() + e * sc.norm()) + 1e-300
    return max(float((err / elem).max()) if err.numel() else 0.0, float(err.norm() / norm))


def assert_close(got, ref, dtype, scale=None, n=1, approx=0.0, c=4.0, cn=1.0, what=""):
    """Raise AssertionError unless ``got`` is within the bound described in the module docstring.  Returns the error ratio."""
    r = error_ratio(got, ref, dtype, scale=scale, n=n, approx=approx, c=c, cn=cn)
    if not r <= 1.0:
        got64, ref64 = _d(got), _d(ref)
        i = int((got64 - ref64).abs().reshape(-1).nan_to_num(math.inf).argmax())
        raise AssertionError(f"{what} {dtype}: error/bound = {r:.3g}; worst element {i}: got {got64.reshape(-1)[i].item()!r}, "
                             f"ref {ref64.reshape(-1)[i].item()!r}")
    return r


def rel_err(got, ref):
    got, ref = _d(got), _d(ref)
    return float((got - ref).norm() / (ref.norm() + 1e-300))


# ---------------------------------------------------------------------------------------------------------------- norms
def layer_norm(x, w, b, eps):
    """-> (y, mean, rstd) over the last dim; biased variance."""
    x = _d(x)
    mean = x.mean(-1, keepdim=True)
    var = ((x - mean) ** 2).mean(-1, keepdim=True)
    rstd = (var + eps).rsqrt()
    y = (x - mean) * rstd * _d(w)
    if b is not None:
        y = y + _d(b)
    return y, mean.squeeze(-1), rstd.squeeze(-1)


def rms_norm(x, w, eps):
    """-> (y, rstd); no mean subtraction."""
    x = _d(x)
    rstd = ((x * x).mean(-1, keepdim=True) + eps).rsqrt()
    return x * rstd * _d(w), rstd.squeeze(-1)


def norm_bwd(dy, x, w, b, eps, rms, dres=None):
    """-> (dx, dw, db) of layer_norm / rms_norm by float64 autograd; ``dres`` is added to dx (pre-norm residual branch)."""
    xd = _d(x).requires_grad_(True)
    wd = _d(w).requires_grad_(True)
    bd = None if (rms or b is None) else _d(b).requires_grad_(True)
    y = rms_norm(xd, wd, eps)[0] if rms else layer_norm(xd, wd, bd, eps)[0]
    ins = [xd, wd] + ([bd] if bd is not None else [])
    grads = torch.autograd.grad(y, ins, _d(dy))
    dx = grads[0] + (_d(dres) if dres is not None else 0.0)
    return dx, grads[1], (grads[2] if bd is not None else None)


# ---------------------------------------------------------------------------------------------------------------- GELU
def gelu(x, exact):
    x = _d(x)
    if exact:
        return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))
    return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + 0.044715 * x ** 3)))


def gelu_grad(x, exact):
    x = _d(x)
    if exact:
        return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)
    k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
    t = torch.tanh(k0 * (x + k1 * x ** 3))
    return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * k0 * (1.0 + 3.0 * k1 * x * x)


def gelu_bound(x, ref, exact, grad=False):
    """``assert_close`` arguments for GELU (``grad``: its derivative) of x.  fp32 evaluation of 1 + erf / 1 + tanh cancels in the negative
    tail, which costs up to 2^-24 |x| absolutely.  The tanh form runs on tanh.approx.f32: an error dt in t = tanh(k0 (x + k1 x^3)) moves
    the GELU by 0.5 |x| dt and its derivative by (0.5 + |x| |t| k0 (1 + 3 k1 x^2)) dt."""
    ax = _d(x).abs()
    if exact:
        return dict(scale=ax)
    if not grad:
        return dict(scale=0.5 * ax, approx=TANH_APPROX)
    k0, k1 = math.sqrt(2.0 / math.pi), 0.044715
    t = torch.tanh(k0 * (_d(x) + k1 * _d(x) ** 3)).abs()
    return dict(scale=0.5 + ax * t * k0 * (1.0 + 3.0 * k1 * ax * ax), approx=TANH_APPROX)


# ---------------------------------------------------------------------------------------------------------------- dropout
def dropout_scale(p):
    """The scale the dropout kernels apply to kept elements: p is quantised to a 16-bit threshold first."""
    thresh = min(int(p * 65536.0 + 0.5), 65535)
    # 1 - thresh / 65536 is exact in fp32; the kernels' scale is its fp32 reciprocal, rounded once
    return float(np.float32(1.0) / np.float32(1.0 - thresh / 65536.0)) if thresh else 1.0


# ---------------------------------------------------------------------------------------------------------------- reductions
def colsum(x):
    return _d(x).sum(0)


def sumsq(x):
    x = _d(x)
    return (x * x).sum()


# ---------------------------------------------------------------------------------------------------------------- cross-entropy
def ce_stats(logits, labels, vocab_start=0):
    """-> (row_max, row_sum, tgt) of one vocab shard: sum_j exp(x_j - max), tgt = x[label - vocab_start] or 0 off the shard."""
    x = _d(logits)
    mx = x.max(-1).values
    sm = torch.exp(x - mx[:, None]).sum(-1)
    local = labels.to(x.device) - vocab_start
    inside = (local >= 0) & (local < x.shape[-1])
    tg = torch.where(inside, x.gather(-1, local.clamp(0, x.shape[-1] - 1)[:, None]).squeeze(-1), torch.zeros_like(mx))
    return mx, sm, tg


def ce_loss(logits, labels, vocab_start=0):
    mx, sm, tg = ce_stats(logits, labels, vocab_start)
    return mx + torch.log(sm) - tg


def ce_grad(logits, labels, lse, gscale, vocab_start=0):
    """(softmax(x) against the given lse - onehot(label - vocab_start)) * gscale[row]."""
    x = _d(logits)
    p = torch.exp(x - _d(lse)[:, None])
    local = labels.to(x.device) - vocab_start
    inside = (local >= 0) & (local < x.shape[-1])
    onehot = torch.zeros_like(p)
    onehot.scatter_(-1, local.clamp(0, x.shape[-1] - 1)[:, None], inside.to(p.dtype)[:, None])
    return (p - onehot) * _d(gscale)[:, None]


# ---------------------------------------------------------------------------------------------------------------- AdamW
def clip_coef(sq, inv_loss_scale, clip_norm):
    """-> (gscale, found_inf, gnorm) as the optimizer defines them."""
    s = float(sq)
    if not math.isfinite(s):
        return 0.0, 1.0, math.sqrt(s) * inv_loss_scale if s == s else s
    norm = math.sqrt(s) * inv_loss_scale
    coef = min(1.0, clip_norm / (norm + 1e-6)) if clip_norm > 0 else 1.0
    return inv_loss_scale * coef, 0.0, norm


def adamw_step(master, grad, m, v, lr, beta1, beta2, eps, wd, step, gscale=1.0):
    """One decoupled-weight-decay AdamW step with bias correction -> (master, m, v)."""
    g = _d(grad) * gscale
    m = beta1 * _d(m) + (1.0 - beta1) * g
    v = beta2 * _d(v) + (1.0 - beta2) * g * g
    bc1, bc2 = 1.0 - beta1 ** step, 1.0 - beta2 ** step
    master = _d(master) * (1.0 - lr * wd) - lr * (m / bc1) / (torch.sqrt(v / bc2) + eps)
    return master, m, v


# ---------------------------------------------------------------------------------------------------------------- rotary
def rope(x, positions, base=10000.0, inverse=False):
    """NeoX rotary embedding of x [tokens, heads, d] (first half / second half pairs) at integer ``positions`` [tokens]."""
    x = _d(x)
    d = x.shape[-1]
    inv = base ** (-torch.arange(0, d // 2, dtype=torch.float64, device=x.device) * 2.0 / d)
    ang = _d(positions)[:, None] * inv
    cs, sn = torch.cos(ang)[:, None, :], torch.sin(ang)[:, None, :]
    if inverse:
        sn = -sn
    x1, x2 = x[..., : d // 2], x[..., d // 2:]
    return torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], -1)


# ---------------------------------------------------------------------------------------------------------------- causal softmax
def causal_mask(sq, sk, device=None):
    """True where row r may attend to column c: c <= r + (sk - sq), i.e. the last query sees every key."""
    r = torch.arange(sq, device=device)[:, None]
    c = torch.arange(sk, device=device)[None, :]
    return c <= r + (sk - sq)


def causal_softmax(x, scale):
    x = _d(x) * scale
    keep = causal_mask(x.shape[-2], x.shape[-1], x.device)
    return torch.softmax(x.masked_fill(~keep, -math.inf), -1)


def causal_softmax_bwd(dy, y, scale):
    """dx of causal_softmax given its output y (masked entries of y are 0, so they get 0)."""
    dy, y = _d(dy), _d(y)
    keep = causal_mask(y.shape[-2], y.shape[-1], y.device)
    dy = dy * keep
    return scale * y * (dy - (dy * y).sum(-1, keepdim=True))


# ---------------------------------------------------------------------------------------------------------------- 8-bit
# The 8-bit references are exact or nearly so: an int8 x int8 sum over K is an integer below K * 2^14 << 2^53, products of e4m3 values
# (and of MX block scales) are exact in float64, and the quantisers are deterministic functions of their input.
E4M3_MAX = 448.0
INT8_MAX = 127.0
# quantize_rows computes scale = amax(x / smooth) / qmax with --use_fast_math division (x / smooth and amax / qmax, 2 ulp each) and
# quantises with x * rcp(scale); the scale therefore lies within 4 fp32 ulp of the float64 value, and x / (smooth * scale) within 2^-20
# relative of what the kernel rounds.
QUANT_SCALE_ULPS = 4
QUANT_REL = 2.0 ** -20
# Epilogue of the 8-bit GEMMs and the W8A8 GEMV: I2F of the int32 sum, * row scale, * column scale, + bias, each an fp32 rounding.
LOWP_EPILOGUE = 4 * FP32_U
# In-chain error of one fp8 wgmma chain (128 K: four m64n128k32 instructions accumulating in the tensor core), relative to the sum of
# |terms| in that chunk.  The PTX ISA does not document the accumulator's width.  Measured on an H100 80GB HBM3 (700 W), 2026-10-17:
# 2^-10.1 at K = 128 for positive terms (test_gpu_lowp_kernels.py::test_fp8_gemm_accumulation).  A single chain over K = 16384 lost 2^-2.
FP8_MMA = 2.0 ** -9


def _e4m3_grid(a):
    """quantum of e4m3fn around |a| (float64 array/tensor): 2^(floor(log2 a) - 3), subnormal quantum 2^-9 below 2^-6."""
    ex = torch.floor(torch.log2(a.clamp(min=2.0 ** -6)))
    return torch.exp2(ex - 3)


def e4m3_rne(t):
    """float64 values of the round-to-nearest-even, saturating (satfinite) e4m3fn conversion of the float64 tensor t."""
    t = _d(t)
    a = t.abs()
    q = _e4m3_grid(a)
    r = torch.round(a / q) * q            # torch.round rounds half to even
    return torch.sign(t) * r.clamp(max=E4M3_MAX)


def _near_e4m3_tie(t, rel=QUANT_REL):
    a = _d(t).abs()
    q = _e4m3_grid(a)
    mid = (torch.floor(a / q) + 0.5) * q
    return ((a - mid).abs() <= rel * a) & (a < E4M3_MAX + 16)


def quantize_rows_check(x, smooth, q, scale, fp8):
    """Check a per-row quantisation (``quantize_rows``) of x [rows, cols] element by element against float64.  Takes the kernel's own
    ``scale`` for the element check, so ties and fast-math rounding of the scale cannot make it flaky.  Raises AssertionError."""
    cols = x.shape[-1]
    x64 = _d(x).reshape(-1, cols)
    s64 = _d(smooth).reshape(1, cols) if smooth is not None else torch.ones((1, cols), dtype=torch.float64, device=x64.device)
    sc = _d(scale).reshape(-1)
    qv = _d(q.view(torch.float8_e4m3fn) if fp8 else q).reshape(-1, cols)
    amax = (x64 / s64).abs().amax(-1) if cols else torch.zeros(x64.shape[0], dtype=torch.float64)
    qmax = E4M3_MAX if fp8 else INT8_MAX
    want = torch.where(amax > 0, amax / qmax, torch.ones_like(amax))
    ulp = torch.exp2(torch.floor(torch.log2(want)) - 23)
    bad = (sc - want).abs() > QUANT_SCALE_ULPS * ulp
    if bad.any():
        i = int(bad.nonzero()[0])
        raise AssertionError(f"quantize_rows scale row {i}: got {sc[i].item()!r}, want {want[i].item()!r} (amax {amax[i].item()!r} / {qmax})")
    zero = amax == 0
    if (qv[zero] != 0).any():
        raise AssertionError("quantize_rows: an all-zero row quantised to nonzero values")
    t = x64 / (s64 * sc[:, None])
    if fp8:
        want_q = e4m3_rne(t)
        bad = (qv != want_q) & ~_near_e4m3_tie(t)
    else:
        bad = ((qv - t).abs() > 0.5 + QUANT_REL * t.abs()) | (qv.abs() > INT8_MAX)
    if bad.any():
        r, c = (int(v) for v in bad.nonzero()[0])
        raise AssertionError(f"quantize_rows q[{r}, {c}]: got {qv[r, c].item()!r} for x / (smooth * scale) = {t[r, c].item()!r}")


def mx_sf_index(r, kb, K):
    """Byte offset of the E8M0 scale of row r, 32-element K block kb in the [ceil(R / 128), K / 128, 512] atom layout."""
    return ((r // 128) * (K // 128) + kb // 4) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + kb % 4


def mx_encode_sf(e_biased, K):
    """e_biased uint8 [R, K / 32] (row-major scale bytes) -> the atom layout, zeros for rows >= R."""
    R = e_biased.shape[0]
    out = torch.zeros(((R + 127) // 128) * (K // 128) * 512, dtype=torch.uint8)
    r = torch.arange(R)[:, None].expand(R, K // 32)
    kb = torch.arange(K // 32)[None, :].expand(R, K // 32)
    out[mx_sf_index(r, kb, K).reshape(-1)] = e_biased.reshape(-1).cpu()
    return out.view((R + 127) // 128, K // 128, 512)


def mx_decode_sf(sf, R, K):
    """Atom layout -> uint8 [R, K / 32] scale bytes."""
    r = torch.arange(R)[:, None].expand(R, K // 32)
    kb = torch.arange(K // 32)[None, :].expand(R, K // 32)
    return sf.reshape(-1).cpu()[mx_sf_index(r, kb, K)]


def mx_quantize_ref(x):
    """OCP MX fp8 of x [R, K] (K % 128 == 0) -> (q e4m3fn [R, K], sf uint8 atoms) as ``quantize_mxfp8`` must produce them bit for bit:
    per 32-element block the scale exponent e = ceil(log2(amax / 448)) clamped to [-127, 127] (-127 for a zero block), stored as e + 127,
    and q = RNE-saturating e4m3 of x * 2^-e."""
    R, K = x.shape
    blocks = _d(x).cpu().reshape(R, K // 32, 32)
    amax = blocks.abs().amax(-1)
    e = torch.where(amax > 0, torch.ceil(torch.log2(amax / E4M3_MAX)), torch.full_like(amax, -127.0)).clamp(-127, 127)
    q = e4m3_rne(blocks * torch.exp2(-e)[..., None]).reshape(R, K)
    return q.to(torch.float8_e4m3fn), mx_encode_sf((e + 127).to(torch.uint8), K)


def mx_dequant(q, sf):
    """float64 values of MX operands: e4m3 values times 2^(byte - 127) per (row, 32-element block); byte 0 is 2^-127."""
    R, K = q.shape
    e = mx_decode_sf(sf, R, K).to(torch.float64) - 127
    return (_d(q.view(torch.float8_e4m3fn)).cpu().reshape(R, K // 32, 32) * torch.exp2(e)[..., None]).reshape(R, K)


def lowp_gemm_ref(a, b, row_scale=None, col_scale=None, bias=None):
    """D = (a @ b^T) * row_scale[:, None] * col_scale[None, :] + bias in float64, for float64 operand values a [M, K], b [N, K] (int8
    values, decoded e4m3 or MX-dequantised).  -> (ref, acc_scale, terms_scale): |acc| |rs| |cs| + |bias| bounds the epilogue's rounding,
    sum|terms| |rs| |cs| + |bias| the in-chain error of a floating-point accumulation."""
    a64, b64 = _d(a), _d(b)
    acc = a64 @ b64.t()
    terms = a64.abs() @ b64.abs().t()
    mul = torch.ones((), dtype=torch.float64, device=acc.device)
    if row_scale is not None:
        mul = mul * _d(row_scale).reshape(-1, 1).to(acc.device)
    if col_scale is not None:
        mul = mul * _d(col_scale).reshape(1, -1).to(acc.device)
    bb = _d(bias).reshape(1, -1).to(acc.device) if bias is not None else torch.zeros((), dtype=torch.float64, device=acc.device)
    return acc * mul + bb, acc.abs() * mul.abs() + bb.abs(), terms * mul.abs() + bb.abs()


def int8_gemm_bound(acc_scale):
    """``assert_close`` arguments for the int8 GEMM and GEMV: the int32 sum is exact, so one rounding to the output (c = 1) plus the
    epilogue's fp32 roundings."""
    return dict(scale=acc_scale, approx=LOWP_EPILOGUE, c=1.0)


def fp8_gemm_bound(terms_scale, K):
    """``assert_close`` arguments for the fp8 and MX GEMMs: the usual c = 4 bound with an fp32 sum over K / 128 chunks and the in-chain
    error ``FP8_MMA`` of each chunk, both relative to the sum of |terms|."""
    return dict(scale=terms_scale, n=max(K // 128, 1), approx=FP8_MMA + LOWP_EPILOGUE)
