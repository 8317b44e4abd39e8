"""float64 references and error bounds for the bandwidth-bound kernels (norms, GELU, dropout, column sums, cross-entropy, AdamW,
rotary embedding, causal softmax), for the 8-bit path (per-row and MX quantisers, int8 / fp8 / MX GEMMs, the W8A8 GEMV) and for the
attention kernels (flash forward / backward, single-query decode, Evoformer gated attention).  Nothing here needs CUDA: the references
run on whatever device their inputs live on.

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
# ex2.approx.f32 (exp2f under --use_fast_math, the flash and Evoformer softmax): the PTX ISA gives a maximum relative error of 2 ulp (2^-22)
EX2_APPROX = 2.0 ** -22
# lg2.approx.f32 (log2f under --use_fast_math, the log-sum-exp): maximum absolute error 2^-22 on the result (PTX ISA: 2^-22.6 for the mantissa)
LG2_APPROX = 2.0 ** -22
# __expf(x) (the decode softmax, the Evoformer gate's sigmoid) is ex2.approx of x * log2(e): the CUDA C++ Programming Guide gives a maximum
# error of 2 + floor(1.173 |x|) ulp, so the error grows with |x|
EXPF_ULP = 2.0 ** -23
# In-chain error of the fp32 tensor-core accumulation (wgmma), relative to the sum of |terms|.  An allowance, not a measurement: the PTX ISA
# does not document the accumulator's width, so the bound leaves room for a truncating one.
MMA_ACC = 2.0 ** -16


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


# ---------------------------------------------------------------------------------------------------------------- attention
# The attention bounds are first-order error budgets.  Every bound below returns ``assert_close`` arguments ``dict(scale=E, approx=1.0)``,
# where E is the absolute error the kernel may make before its final rounding to the output dtype, so the elementwise test reads
# |got - ref| <= 4 (u (|ref| + tiny) + E).  E is built from these terms (u: the 16-bit unit roundoff, pi: the exact probabilities, a = pi
# times the dropout keep factor keep / (1 - p), tiny: the dtype's smallest normal number, which bounds the error of rounding a subnormal P):
#
#   logits   ds   = MMA_ACC scale max_k sum_d |q_d| |k_d| + 4 * 2^-24 (max |logit| + |lse|): the fp32 tensor-core sum of q.k, and the fp32
#                   roundings of the exp2 argument (logit * scale * log2e - row max), per query row and in natural-log units.  An absolute
#                   error ds of a logit is a relative error ds of its probability.
#   exp2          EX2_APPROX, relative, on every probability.
#   P             rounded to 16 bits before P V while the row sum l adds the unrounded fp32 p: u sum_k (pi_k + tiny) keep_k |v_k|.  This is the
#                 dominant term and the reason the bound is stated against sum pi |v| rather than |O|.
#   P V           MMA_ACC sum_k a_k |v_k| (the accumulator is carried across all key tiles), plus one fp32 rescale per 128-key tile.
#   output        the final rounding u |O| (the u |ref| term of assert_close).
#   lse           fp32 and natural log, absolute: ds + EX2_APPROX + LG2_APPROX + 2^-24 (sqrt(Sk) + |lse|).
#   backward      p is recomputed from the stored lse (relative error ds + E_lse + EX2_APPROX); delta = rowsum(dO o O) is formed from the
#                 16-bit-rounded O, so it carries the forward's error E_O + u |O| weighted by |dO|; P and dS are rounded to 16 bits before
#                 the dV, dK and dQ products (u (|.| + tiny), tiny / scale for dS, which is rounded as dS scale); dP = dO V^T is a tensor-core sum (MMA_ACC); dQ is one fp32 reduce-add per
#                 64-key tile and one rounding.  Then E_dS = rel_p |dS| + pi keep MMA_ACC (|dO| |V|^T) + pi |d delta|, and
#                 E_dQ = scale ((u (|dS| + tiny) + E_dS) |K| + (MMA_ACC + 2^-24 Sk / 64) |dS| |K|), likewise for dK and dV.
#   Evoformer     the same, plus the gate's sigmoid 1 / (1 + __expf(-g)) (relative error EXPF_ULP (4 + 1.2 |g|)), dO' = dOut sig rounded to
#                 bf16 before dV and dP, and dgate / delta formed from the bf16-rounded gated output.
# A mistake that moves O by a fraction of |O| is caught only where sum pi |v| is close to |O|, i.e. where attention is peaked: the tests feed
# logits with a spread of a few units (``attention_inputs``), so that a handful of keys carry each row.

def attention_inputs(B, Sq, Sk, H, D, Hkv=None, seed=0, rising=False, device="cpu"):
    """float32 masters (q [B,Sq,H,D], k / v [B,Sk,Hkv,D], dout [B,Sq,H,D]) for the attention tests: q and k at 1.6 sigma, so that the logits
    scale q.k spread over about 2.5 units and each row is carried by a few keys.  ``rising`` adds a component along one channel that grows by
    one logit unit per 128 keys, so that every row's maximum moves into every later key tile."""
    Hkv = Hkv or H
    g = torch.Generator(device=device).manual_seed(seed)
    q = torch.randn(B, Sq, H, D, generator=g, device=device) * 1.6
    k = torch.randn(B, Sk, Hkv, D, generator=g, device=device) * 1.6
    v = torch.randn(B, Sk, Hkv, D, generator=g, device=device)
    do = torch.randn(B, Sq, H, D, generator=g, device=device)
    if rising:
        q[..., 0] = 4.0
        k[..., 0] = torch.arange(Sk, device=device, dtype=torch.float32).view(1, Sk, 1) * (D ** 0.5 / (4.0 * 128))
    return q, k, v, do


def decode_new_kv(q, Hkv, seed=0):
    """This step's key / value [B, Hkv, D] for the decode tests: the key is 3 x the mean of its group's queries, so it carries most of the
    group's attention and a cache append that goes missing or to the wrong row moves the output by about |O|."""
    B, _, H, D = q.shape
    k_new = 3.0 * q.float().reshape(B, Hkv, H // Hkv, D).mean(2)
    v_new = torch.randn(B, Hkv, D, generator=torch.Generator(device=q.device).manual_seed(seed), device=q.device)
    return k_new, v_new


def evoformer_inputs(G, Sq, Sk, H, gpp, mask=True, pair=True, gate=True, seed=0, device="cpu"):
    """float32 masters (q, k, v, mask_bias, pair_bias, gate, dout) for the Evoformer tests: q / k at 1.6 sigma (peaked rows, as
    ``attention_inputs``), a unit-variance pair bias, about 10 % of the keys of every group masked with the model's -1e9 (key 0 never), and
    the absent operands None."""
    g = torch.Generator(device=device).manual_seed(seed)
    q = torch.randn(G, Sq, H, 32, generator=g, device=device) * 1.6
    k = torch.randn(G, Sk, H, 32, generator=g, device=device) * 1.6
    v = torch.randn(G, Sk, H, 32, generator=g, device=device)
    do = torch.randn(G, Sq, H, 32, generator=g, device=device)
    keep = torch.rand(G, Sk, generator=g, device=device) >= 0.1
    keep[:, 0] = True
    mb = 1e9 * (keep.float() - 1.0) if mask else None
    pb = torch.randn(G // gpp, H, Sq, Sk, generator=g, device=device) if pair else None
    gt = torch.randn(G, Sq, H, 32, generator=g, device=device) if gate else None
    return q, k, v, mb, pb, gt, do


def _bhsd(t, H=None):
    """[B, S, Hkv, D] -> float64 [B, H, S, D], K/V head h // G serving query head h (``repeat_interleave``)."""
    t = _d(t)
    if H is not None and H != t.shape[2]:
        t = t.repeat_interleave(H // t.shape[2], dim=2)
    return t.transpose(1, 2)


def _softmax_rows(s):
    """-> (pi, lse) of logits s (-inf = masked); a row with no finite logit gets pi = 0 and lse = -inf (the kernels' l = 0 convention)."""
    m = s.amax(-1, keepdim=True)
    m0 = torch.where(torch.isfinite(m), m, torch.zeros_like(m))
    e = torch.exp(s - m0)
    l = e.sum(-1, keepdim=True)
    pi = e / torch.where(l > 0, l, torch.ones_like(l))
    return pi, (m0 + torch.log(l)).squeeze(-1)


def _keep_factor(keep, p, like):
    return torch.ones_like(like) if keep is None else _d(keep.to(like.device)) / (1.0 - p)


def attention(q, k, v, scale, causal, keep=None, p=0.0):
    """Flash attention forward -> (out [B,Sq,H,D], lse [B,H,Sq]).  q [B,Sq,H,D], k / v [B,Sk,Hkv,D] (head h uses K/V head h // (H / Hkv)),
    the causal mask bottom-right aligned (``causal_mask``), ``keep`` [B,H,Sq,Sk] the dropout keep mask (kept probabilities scaled by
    1 / (1 - p)).  The log-sum-exp does not see dropout."""
    qh = _bhsd(q)
    H = qh.shape[1]
    kh, vh = _bhsd(k, H), _bhsd(v, H)
    s = qh @ kh.transpose(-1, -2) * scale
    if causal:
        s = s.masked_fill(~causal_mask(s.shape[-2], s.shape[-1], s.device), -math.inf)
    pi, lse = _softmax_rows(s)
    out = (pi * _keep_factor(keep, p, pi)) @ vh
    return out.transpose(1, 2), lse


def attention_bwd(q, k, v, dout, scale, causal, keep=None, p=0.0):
    """-> (dq, dk, dv) of ``attention`` by float64 autograd, with the same keep mask (dk / dv summed over the heads of a group)."""
    qd, kd, vd = (_d(t).clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        out, _ = attention(qd, kd, vd, scale, causal, keep, p)
        return torch.autograd.grad(out, (qd, kd, vd), _d(dout))


def _logit_err(qh, kh, s, pi, lse, scale):
    """Absolute error (natural-log units) of a kernel logit as seen by exp2, per query row [.., Sq, 1]: the tensor-core sum of q.k and the
    fp32 roundings of the exp2 argument, over the keys that carry any probability (a masked key's error does not matter)."""
    terms = (qh.abs() @ kh.abs().transpose(-1, -2)).amax(-1, keepdim=True) * scale
    mag = torch.where(pi > 0, s.abs(), torch.zeros_like(s)).amax(-1, keepdim=True)
    lse_abs = torch.where(torch.isfinite(lse), lse.abs(), torch.zeros_like(lse)).unsqueeze(-1)
    return MMA_ACC * terms + 4 * FP32_U * (mag + lse_abs)


def _abs_bound(E):
    """``assert_close`` arguments for an absolute error budget E (module docstring): e = 2^-24 + 1 >= 1, so e * E >= E."""
    return dict(scale=E, approx=1.0)


def _fwd_budget(pi, kw, vh, out_h, ds, dtype, n_tiles):
    """-> E_O [.., Sq, D] (before the output rounding) for P = pi * kw against V vh; out_h the float64 output [.., Sq, D]."""
    u, tiny = UNIT_ROUNDOFF[dtype], torch.finfo(dtype).smallest_normal
    live = (pi > 0).to(pi.dtype)
    vabs = vh.abs()
    a = pi * kw
    p_round = u * (((pi + tiny * live) * kw) @ vabs)
    rel = MMA_ACC + EX2_APPROX + FP32_U * n_tiles + ds
    return p_round + rel * (a @ vabs + out_h.abs())


def attention_bounds(q, k, v, scale, causal, dtype, keep=None, p=0.0):
    """``assert_close`` arguments for (out, lse) of the flash forward on these inputs; lse is checked as float32."""
    qh = _bhsd(q)
    H = qh.shape[1]
    kh, vh = _bhsd(k, H), _bhsd(v, H)
    s = qh @ kh.transpose(-1, -2) * scale
    if causal:
        s = s.masked_fill(~causal_mask(s.shape[-2], s.shape[-1], s.device), -math.inf)
    pi, lse = _softmax_rows(s)
    kw = _keep_factor(keep, p, pi)
    out_h = (pi * kw) @ vh
    ds = _logit_err(qh, kh, s, pi, lse, scale)
    Sk = s.shape[-1]
    E_o = _fwd_budget(pi, kw, vh, out_h, ds, dtype, -(-Sk // 128))
    E_lse = ds.squeeze(-1) + EX2_APPROX + LG2_APPROX + FP32_U * math.sqrt(Sk)
    return _abs_bound(E_o.transpose(1, 2)), _abs_bound(E_lse)


def _group_sum(t, Hkv):
    """[B, H, S, D] per query head -> [B, Hkv, S, D] summed over each group."""
    B, H, S, D = t.shape
    return t.reshape(B, Hkv, H // Hkv, S, D).sum(2)


def _bwd_budget(qh, kh, vh, doh, pi, kw, s_lse_err, E_o, out_h, dtype, scale, q_tiles, k_tiles, do_round=0.0):
    """-> (E_dq, E_dk, E_dv) per query head, [B, H, S, D].  ``s_lse_err`` is the relative error of the recomputed probabilities per row;
    ``do_round`` the relative rounding of dO before the products (the Evoformer's dO' = dOut sig)."""
    u, tiny = UNIT_ROUNDOFF[dtype], torch.finfo(dtype).smallest_normal
    live = (pi > 0).to(pi.dtype)
    a = pi * kw
    dP = doh @ vh.transpose(-1, -2)
    delta = (doh * out_h).sum(-1, keepdim=True)
    dS = pi * (kw * dP - delta)
    dS_abs = dS.abs()
    d_delta = (doh.abs() * (E_o + u * out_h.abs())).sum(-1, keepdim=True) + FP32_U * qh.shape[-1] * (doh.abs() * out_h.abs()).sum(-1, keepdim=True)
    dP_err = (MMA_ACC + do_round) * (doh.abs() @ vh.abs().transpose(-1, -2))
    E_ds = s_lse_err * dS_abs + a * dP_err + pi * d_delta
    # the kernels round dS * scale, so a subnormal costs u tiny / scale in dS units
    ds_op = u * (dS_abs + tiny / scale * live) + E_ds + (MMA_ACC + FP32_U * k_tiles) * dS_abs
    E_dq = scale * (ds_op @ kh.abs())
    E_dk = scale * ((u * (dS_abs + tiny / scale * live) + E_ds + (MMA_ACC + FP32_U * q_tiles) * dS_abs).transpose(-1, -2) @ qh.abs())
    E_dv = ((u * (a + tiny * live * kw) + (s_lse_err + MMA_ACC + do_round + FP32_U * q_tiles) * a).transpose(-1, -2)) @ doh.abs()
    return E_dq, E_dk, E_dv


def attention_bwd_bounds(q, k, v, dout, scale, causal, dtype, keep=None, p=0.0):
    """``assert_close`` arguments for (dq, dk, dv) of the flash backward (layouts as ``attention_bwd`` returns them)."""
    qh = _bhsd(q)
    H, Hkv = qh.shape[1], k.shape[2]
    kh, vh, doh = _bhsd(k, H), _bhsd(v, H), _bhsd(dout)
    s = qh @ kh.transpose(-1, -2) * scale
    if causal:
        s = s.masked_fill(~causal_mask(s.shape[-2], s.shape[-1], s.device), -math.inf)
    pi, lse = _softmax_rows(s)
    kw = _keep_factor(keep, p, pi)
    out_h = (pi * kw) @ vh
    Sq, Sk = s.shape[-2], s.shape[-1]
    ds = _logit_err(qh, kh, s, pi, lse, scale)
    E_o = _fwd_budget(pi, kw, vh, out_h, ds, dtype, -(-Sk // 128))
    rel_p = 2 * ds + EX2_APPROX + LG2_APPROX + FP32_U * math.sqrt(Sk) + EX2_APPROX
    E_dq, E_dk, E_dv = _bwd_budget(qh, kh, vh, doh, pi, kw, rel_p, E_o, out_h, dtype, scale, -(-Sq // 64), -(-Sk // 64))
    return (_abs_bound(E_dq.transpose(1, 2)), _abs_bound(_group_sum(E_dk, Hkv).transpose(1, 2)),
            _abs_bound(_group_sum(E_dv, Hkv).transpose(1, 2)))


# ---------------------------------------------------------------------------------------------------------------- decode
def attention_decode(q, k, v, mask, L, scale):
    """Single-query attention over a cache: q [B,1,H,D], k / v [B,Lmax,Hkv,D], mask additive [B,Lmax] (the values the kernel adds, i.e.
    already in the activation dtype) or None.  Keys at L and beyond are ignored whatever the mask says; a row whose L keys are all -inf
    returns 0.  -> out [B,1,H,D]."""
    qh = _bhsd(q)
    H = qh.shape[1]
    kh, vh = _bhsd(k, H)[:, :, :L], _bhsd(v, H)[:, :, :L]
    s = qh @ kh.transpose(-1, -2) * scale
    if mask is not None:
        s = s + _d(mask).reshape(s.shape[0], 1, 1, -1)[..., :L]
    pi, _ = _softmax_rows(s)
    return (pi @ vh).transpose(1, 2)


def attention_decode_bound(q, k, v, mask, L, scale):
    """``assert_close`` arguments for ``attention_decode``.  The decode kernel keeps P in fp32 (no 16-bit P), so only fp32 terms are left:
    the scalar fp32 dot product (within MMA_ACC of the sum of |terms|), and __expf along each key's chain of online-softmax rescales, whose
    arguments add up to the key's distance x below the row maximum: at most EXPF_ULP (2 (T + 2) + 1.2 |x|) with T = ceil(L / 16) rescales
    per softmax state.  Keys more than 104 below the maximum underflow to 0 in fp32 and weigh less than 2^-150."""
    qh = _bhsd(q)
    H = qh.shape[1]
    kh, vh = _bhsd(k, H)[:, :, :L], _bhsd(v, H)[:, :, :L]
    s = qh @ kh.transpose(-1, -2) * scale
    if mask is not None:
        s = s + _d(mask).reshape(s.shape[0], 1, 1, -1)[..., :L]
    pi, lse = _softmax_rows(s)
    out_h = pi @ vh
    m = s.amax(-1, keepdim=True)
    x = torch.where(torch.isfinite(s) & torch.isfinite(m), (m - s).clamp(max=104.0), torch.zeros_like(s))
    rel = EXPF_ULP * (2 * (-(-L // 16) + 2) + 1.2 * x) + _logit_err(qh, kh, s, pi, lse, scale) + FP32_U * L
    E = (pi * rel) @ vh.abs() + (pi * rel).sum(-1, keepdim=True) * out_h.abs()
    return _abs_bound(E.transpose(1, 2))


# ---------------------------------------------------------------------------------------------------------------- Evoformer
def _evo_logits(q, k, mask_bias, pair_bias, gpp, scale, uniform=None):
    """float64 logits [G, H, Sq, Sk] of the Evoformer attention; ``uniform`` [G] bool marks groups held at equal logits (see ``evoformer``)."""
    qh, kh = _bhsd(q), _bhsd(k)
    s = qh @ kh.transpose(-1, -2) * scale
    if mask_bias is not None:
        s = s + _d(mask_bias)[:, None, None, :]
    if pair_bias is not None:
        s = s + _d(pair_bias).repeat_interleave(gpp, dim=0)
    if uniform is not None:
        s = torch.where(uniform.to(s.device).view(-1, 1, 1, 1), s - s.detach(), s)
    return s


def evoformer(q, k, v, mask_bias, pair_bias, gate, gpp, scale, uniform=None):
    """Evoformer gated attention [G, Sq, H, D]: softmax_k(scale q.k + mask_bias[g, k] + pair_bias[g // gpp, h, q, k]) v * sigmoid(gate).

    ``uniform`` [G] bool: groups whose every key carries the model's -1e9 padding bias.  In fp32 their logits all round to the same number
    (the spacing at 1.44e9 is 128), so the kernels and ``EA.reference`` return the gated mean of V, while float64 keeps the scores.  For those
    groups the logits are replaced by ``s - s.detach()``: value 0 (uniform probabilities), derivative that of s, which is what fp32 autograd
    of the expression gives."""
    s = _evo_logits(q, k, mask_bias, pair_bias, gpp, scale, uniform)
    pi, _ = _softmax_rows(s)
    o = (pi @ _bhsd(v)).transpose(1, 2)
    return o * torch.sigmoid(_d(gate)) if gate is not None else o


def evoformer_bwd(q, k, v, mask_bias, pair_bias, gate, gpp, scale, dout, uniform=None):
    """-> (dq, dk, dv, dgate or None, dpair [G / gpp, H, Sq, Sk] or None) of ``evoformer`` by float64 autograd; dpair is summed over the
    groups that share a pair bias."""
    ins = [_d(t).clone().requires_grad_(True) if t is not None else None for t in (q, k, v, gate, pair_bias)]
    qd, kd, vd, gd, pd = ins
    with torch.enable_grad():
        out = evoformer(qd, kd, vd, mask_bias, pd, gd, gpp, scale, uniform)
        want = [t for t in ins if t is not None]
        grads = iter(torch.autograd.grad(out, want, _d(dout)))
    return tuple(next(grads) if t is not None else None for t in ins)


def sigmoid_err(gate):
    """Relative error of the kernels' sigmoid 1 / (1 + __expf(-g)): __expf's EXPF_ULP (2 + 1.173 |g|), plus the fast division and add."""
    return EXPF_ULP * (4 + 1.2 * _d(gate).abs())


def evoformer_bounds(q, k, v, mask_bias, pair_bias, gate, gpp, scale, dout=None, uniform=None):
    """``assert_close`` arguments for the bf16 Evoformer kernels on these inputs: out, and with ``dout`` also dq, dk, dv, dgate (or None)
    and dpair (fp32, summed over the groups sharing a pair bias; or None)."""
    dtype = torch.bfloat16
    u = UNIT_ROUNDOFF[dtype]
    qh, kh, vh = _bhsd(q), _bhsd(k), _bhsd(v)
    G, H, Sq, Sk = qh.shape[0], qh.shape[1], qh.shape[2], kh.shape[2]
    s = _evo_logits(q, k, mask_bias, pair_bias, gpp, scale, uniform)
    pi, lse = _softmax_rows(s)
    ones = torch.ones_like(pi)
    o_h = pi @ vh
    ds = _logit_err(qh, kh, s, pi, lse, scale)
    E_o = _fwd_budget(pi, ones, vh, o_h, ds, dtype, -(-Sk // 128))                      # ungated, [G, H, Sq, D]
    if gate is not None:
        sig = torch.sigmoid(_bhsd(gate))
        se = sigmoid_err(_bhsd(gate))
        E_out = sig * E_o + (se + FP32_U) * sig * o_h.abs()
    else:
        sig, se, E_out = torch.ones_like(o_h), torch.zeros_like(o_h), E_o
    out_kw = _abs_bound(E_out.transpose(1, 2))
    if dout is None:
        return out_kw
    d = _bhsd(dout)
    out_h = o_h * sig
    dop = d * sig                                                                           # dO' = dOut sig, rounded to bf16 by the kernel
    rel_p = 2 * ds + 2 * EX2_APPROX + LG2_APPROX + FP32_U * math.sqrt(Sk)
    # delta = rowsum(dOut o out16) = rowsum(dO' o O): hand _bwd_budget the error of out16 expressed against dO' (E_out / sig)
    E_dq, E_dk, E_dv = _bwd_budget(qh, kh, vh, dop, pi, ones, rel_p, E_out / sig, o_h, dtype, scale,
                                   -(-Sq // 64), -(-Sk // 64), do_round=u + se.amax().item())
    res = [out_kw, _abs_bound(E_dq.transpose(1, 2)), _abs_bound(E_dk.transpose(1, 2)), _abs_bound(E_dv.transpose(1, 2))]
    if gate is not None:
        # dgate = dOut out16 (1 - sig): the error of out16 (E_out + u |out|) and of 1 - sig (sig * se absolutely)
        E_dg = d.abs() * ((E_out + u * out_h.abs()) * (1 - sig) + out_h.abs() * sig * se + FP32_U * 4 * out_h.abs())
        res.append(_abs_bound(E_dg.transpose(1, 2)))
    else:
        res.append(None)
    if pair_bias is not None:
        # dpair[q, k] = sum over the gpp groups of dS (fp32 red.add, no 16-bit rounding): the dS budget without the u terms
        dP = dop @ vh.transpose(-1, -2)
        delta = (dop * o_h).sum(-1, keepdim=True)
        dS = pi * (dP - delta)
        d_delta = (dop.abs() * (E_out / sig + u * o_h.abs())).sum(-1, keepdim=True)
        E_ds = rel_p * dS.abs() + pi * ((MMA_ACC + u + se.amax().item()) * (dop.abs() @ vh.abs().transpose(-1, -2)) + d_delta) \
            + FP32_U * gpp * dS.abs()
        res.append(dict(scale=E_ds.reshape(G // gpp, gpp, H, Sq, Sk).sum(1), approx=1.0))
    else:
        res.append(None)
    return tuple(res)
