"""float64 references and error bounds for flash attention under a boolean mask on top of the causal one (the document mask of
``DocumentMask``).  The same computations and budgets as the flash section of ``kernel_refs``, with the masked logits set to -inf
before the softmax: a masked key carries no probability, so it adds neither to the result nor to its bound."""
import math

import torch

import kernel_refs as R


def _logits(q, k, scale, mask):
    """-> (qh, kh, s): float64 [B, H, S, D] views of q / k and the logits with the causal mask and ``mask`` (bool [B, Sq, Sk], True =
    attend) set to -inf."""
    qh = R._bhsd(q)
    kh = R._bhsd(k, qh.shape[1])
    s = qh @ kh.transpose(-1, -2) * scale
    s = s.masked_fill(~R.causal_mask(s.shape[-2], s.shape[-1], s.device), -math.inf)
    return qh, kh, s.masked_fill(~mask.to(s.device).unsqueeze(1), -math.inf)


def attention(q, k, v, scale, mask, keep=None, p=0.0):
    """``kernel_refs.attention`` (causal) restricted to ``mask`` -> (out [B, Sq, H, D], lse [B, H, Sq])."""
    qh, kh, s = _logits(q, k, scale, mask)
    vh = R._bhsd(v, qh.shape[1])
    pi, lse = R._softmax_rows(s)
    out = (pi * R._keep_factor(keep, p, pi)) @ vh
    return out.transpose(1, 2), lse


def attention_bwd(q, k, v, dout, scale, mask, keep=None, p=0.0):
    """-> (dq, dk, dv) of ``attention`` by float64 autograd (dk / dv summed over the heads of a group)."""
    qd, kd, vd = (R._d(t).clone().requires_grad_(True) for t in (q, k, v))
    with torch.enable_grad():
        out, _ = attention(qd, kd, vd, scale, mask, keep, p)
        return torch.autograd.grad(out, (qd, kd, vd), R._d(dout))


def attention_bounds(q, k, v, scale, mask, dtype, keep=None, p=0.0):
    """``assert_close`` arguments for (out, lse), as ``kernel_refs.attention_bounds``; lse is checked as float32."""
    qh, kh, s = _logits(q, k, scale, mask)
    vh = R._bhsd(v, qh.shape[1])
    pi, lse = R._softmax_rows(s)
    kw = R._keep_factor(keep, p, pi)
    out_h = (pi * kw) @ vh
    ds = R._logit_err(qh, kh, s, pi, lse, scale)
    Sk = s.shape[-1]
    E_o = R._fwd_budget(pi, kw, vh, out_h, ds, dtype, -(-Sk // 128))
    E_lse = ds.squeeze(-1) + R.EX2_APPROX + R.LG2_APPROX + R.FP32_U * math.sqrt(Sk)
    return R._abs_bound(E_o.transpose(1, 2)), R._abs_bound(E_lse)


def attention_bwd_bounds(q, k, v, dout, scale, mask, dtype, keep=None, p=0.0):
    """``assert_close`` arguments for (dq, dk, dv), as ``kernel_refs.attention_bwd_bounds``."""
    qh, kh, s = _logits(q, k, scale, mask)
    H, Hkv = qh.shape[1], k.shape[2]
    vh, doh = R._bhsd(v, H), R._bhsd(dout)
    pi, lse = R._softmax_rows(s)
    kw = R._keep_factor(keep, p, pi)
    out_h = (pi * kw) @ vh
    Sq, Sk = s.shape[-2], s.shape[-1]
    ds = R._logit_err(qh, kh, s, pi, lse, scale)
    E_o = R._fwd_budget(pi, kw, vh, out_h, ds, dtype, -(-Sk // 128))
    rel_p = 2 * ds + R.EX2_APPROX + R.LG2_APPROX + R.FP32_U * math.sqrt(Sk) + R.EX2_APPROX
    E_dq, E_dk, E_dv = R._bwd_budget(qh, kh, vh, doh, pi, kw, rel_p, E_o, out_h, dtype, scale, -(-Sq // 64), -(-Sk // 64))
    return (R._abs_bound(E_dq.transpose(1, 2)), R._abs_bound(R._group_sum(E_dk, Hkv).transpose(1, 2)),
            R._abs_bound(R._group_sum(E_dv, Hkv).transpose(1, 2)))
