"""float64 references and error bounds for the bandwidth-bound kernels (norms, GELU, dropout, column sums, cross-entropy, AdamW,
rotary embedding, causal softmax).  Nothing here needs CUDA: the references run on whatever device their inputs live on.

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
