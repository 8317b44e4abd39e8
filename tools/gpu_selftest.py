"""Stand-alone numerics + timing sweep of the native kernels on one H100.

Each check runs in its own subprocess under a timeout so that a hung or trapping kernel cannot take the whole
sweep (or the GPU box) down.  Results are appended to ``gpurun_out/selftest.log`` as JSON lines.

    python tools/gpu_selftest.py            # all checks
    python tools/gpu_selftest.py gemm_nt    # one check (runs in-process)
"""
from __future__ import annotations

import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
OUT = os.path.join(ROOT, "gpurun_out")


def _lib():
    from paddlefleetx_b200.ops import _native
    return _native.require()


def _time(fn, iters=20, warmup=5, flush_mb=256):
    import torch
    flush = torch.empty(flush_mb * 1024 * 1024, dtype=torch.uint8, device="cuda")
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        flush.zero_()  # > L2 (126 MB): cold-L2 timing
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def _relerr(a, b):
    import torch
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


# ------------------------------------------------------------------------------------ checks
def check_gemm(a_k=True, b_k=True, cfg=1, M=512, N=512, K=256, out_mode=0, epilogue=0, time_it=False):
    import torch
    lib = _lib()
    torch.manual_seed(0)
    A = torch.randn(M, K, device="cuda", dtype=torch.bfloat16)
    B = torch.randn(N, K, device="cuda", dtype=torch.bfloat16)
    bias = torch.randn(N, device="cuda", dtype=torch.bfloat16) if epilogue in (1, 2) else None
    a = A if a_k else A.t().contiguous()
    b = B if b_k else B.t().contiguous()
    ref = A.float() @ B.float().t()
    if bias is not None:
        ref = ref + bias.float()
    if epilogue in (2, 3):
        ref = torch.nn.functional.gelu(ref, approximate="tanh")
    out = None
    if out_mode == 2:
        out = torch.randn(M, N, device="cuda", dtype=torch.float32)
        ref = ref + out
    d = lib.gemm(a, b, bias, out, a_k, b_k, epilogue, out_mode, cfg)
    torch.cuda.synchronize()
    err = _relerr(d, ref)
    res = dict(err=err, ok=bool(err < 2e-2 if out_mode == 0 else err < 1e-2))
    if time_it:
        med, best = _time(lambda: lib.gemm(a, b, bias, None if out_mode != 2 else out, a_k, b_k, epilogue, out_mode, cfg))
        res.update(ms=med, ms_best=best, tflops=2.0 * M * N * K / med / 1e9, tflops_best=2.0 * M * N * K / best / 1e9)
        med2, best2 = _time(lambda: torch.matmul(A, B.t()))
        res.update(cublas_ms=med2, cublas_tflops=2.0 * M * N * K / med2 / 1e9)
    return res


def check_norm(rms=False, rows=4096, cols=4096):
    import torch
    lib = _lib()
    torch.manual_seed(0)
    x = torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16)
    w = (torch.randn(cols, device="cuda") * 0.1 + 1).bfloat16()
    b = (torch.randn(cols, device="cuda") * 0.1).bfloat16()
    dy = torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16)
    xf = x.float().requires_grad_(True); wf = w.float().requires_grad_(True); bf = b.float().requires_grad_(True)
    if rms:
        ref = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
    else:
        ref = torch.nn.functional.layer_norm(xf, (cols,), wf, bf, 1e-5)
    ref.backward(dy.float())
    y, mean, rstd = lib.norm_fwd(x, w, None if rms else b, 1e-5, rms)
    dx, dw, db = lib.norm_bwd(dy, x, w, mean, rstd, rms, not rms)
    torch.cuda.synchronize()
    errs = dict(y=_relerr(y, ref), dx=_relerr(dx, xf.grad), dw=_relerr(dw, wf.grad))
    if not rms:
        errs["db"] = _relerr(db, bf.grad)
    med, _ = _time(lambda: lib.norm_fwd(x, w, None if rms else b, 1e-5, rms))
    medb, _ = _time(lambda: lib.norm_bwd(dy, x, w, mean, rstd, rms, not rms))
    nbytes = rows * cols * 2
    return dict(errs=errs, ok=all(v < 1.5e-2 for v in errs.values()), fwd_ms=med, fwd_gbs=2 * nbytes / med / 1e6,
                bwd_ms=medb, bwd_gbs=3 * nbytes / medb / 1e6)


def check_gelu_dropout():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    rows, cols = 4096, 4096
    x = torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16)
    bias = torch.randn(cols, device="cuda", dtype=torch.bfloat16)
    res = torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16)
    dy = torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16)
    xf = (x.float() + bias.float()).requires_grad_(True)
    ref = torch.nn.functional.gelu(xf, approximate="tanh")
    ref.backward(dy.float())
    y = lib.bias_gelu_fwd(x, bias, False)
    dx = lib.bias_gelu_bwd(dy, x, bias, False)
    errs = dict(gelu=_relerr(y, ref), dgelu=_relerr(dx, xf.grad))
    xe = (x.float() + bias.float()).requires_grad_(True)
    refe = torch.nn.functional.gelu(xe)                     # exact (erf) form used by the vision models
    refe.backward(dy.float())
    errs.update(gelu_erf=_relerr(lib.bias_gelu_fwd(x, bias, True), refe), dgelu_erf=_relerr(lib.bias_gelu_bwd(dy, x, bias, True), xe.grad))
    p = 0.1
    yd = lib.bias_dropout_add_fwd(x, bias, res, p, 1234, 77)
    dxd = lib.dropout_bwd(dy, p, 1234, 77)
    pre = (x.float() + bias.float())
    kept = (yd.float() - res.float()).abs() > 1e-6 * 0  # placeholder
    diff = yd.float() - res.float()
    keep_mask = dxd.float() != 0
    frac = float(keep_mask.float().mean())
    # where kept, diff ~= pre / (1-p); where dropped, diff ~= 0 (bf16 rounding of res + val)
    exp = torch.where(keep_mask, pre / (1 - p), torch.zeros_like(pre)) + res.float()
    errs["dropout_fwd"] = _relerr(yd, exp)
    errs["dropout_bwd"] = _relerr(dxd, torch.where(keep_mask, dy.float() / (1 - p), torch.zeros_like(pre)))
    y0 = lib.bias_dropout_add_fwd(x, bias, res, 0.0, 1, 0)
    errs["p0"] = _relerr(y0, pre + res.float())
    cs = lib.colsum(dy, True)
    errs["colsum"] = _relerr(cs, dy.float().sum(0))
    med, _ = _time(lambda: lib.bias_dropout_add_fwd(x, bias, res, p, 1234, 77))
    return dict(errs=errs, keep_frac=frac, ok=all(v < 1.5e-2 for v in errs.values()) and abs(frac - 0.9) < 5e-3,
                bda_ms=med, bda_gbs=3 * rows * cols * 2 / med / 1e6)


def check_ce():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    rows, V = 2048, 50304
    logits = (torch.randn(rows, V, device="cuda") * 2).bfloat16()
    labels = torch.randint(0, V, (rows,), device="cuda")
    lf = logits.float().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(lf, labels, reduction="none")
    g = torch.rand(rows, device="cuda")
    (ref * g).sum().backward()
    mx, sm, tg = lib.ce_stats(logits, labels, 0)
    lse = mx + sm.log()
    loss = lse - tg
    work = logits.clone()
    lib.ce_bwd_(work, labels, lse, g, 0)
    errs = dict(loss=_relerr(loss, ref), dlogits=_relerr(work, lf.grad))
    med, _ = _time(lambda: lib.ce_stats(logits, labels, 0))
    return dict(errs=errs, ok=all(v < 1.5e-2 for v in errs.values()), stats_ms=med, stats_gbs=rows * V * 2 / med / 1e6)


def check_adam():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    n = 1 << 24
    master = torch.randn(n, device="cuda")
    grad = (torch.randn(n, device="cuda") * 0.01).bfloat16()
    m = torch.zeros(n, device="cuda"); v = torch.zeros(n, device="cuda")
    p_lp = master.bfloat16()
    ref_p = torch.nn.Parameter(master.clone())
    opt = torch.optim.AdamW([ref_p], lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.01)
    sq = torch.zeros(1, device="cuda"); gscale = torch.zeros(1, device="cuda"); finf = torch.zeros(1, device="cuda"); gn = torch.zeros(1, device="cuda")
    lib.sumsq_(grad, sq, False)
    norm_ref = grad.float().norm()
    lib.clip_coef_(sq, 1.0, 1.0, gscale, finf, gn)
    coef = min(1.0, 1.0 / (float(norm_ref) + 1e-6))
    for step in (1, 2, 3):
        ref_p.grad = grad.float() * coef
        opt.step()
        lib.adamw_flat_(p_lp, master, grad, m, v, 1e-3, 0.9, 0.95, 1e-8, 0.01, step, gscale, finf)
    errs = dict(norm=abs(float(gn) - float(norm_ref)) / float(norm_ref), master=_relerr(master, ref_p.data), lp=_relerr(p_lp, ref_p.data))
    med, _ = _time(lambda: lib.adamw_flat_(p_lp, master, grad, m, v, 1e-3, 0.9, 0.95, 1e-8, 0.01, 4, gscale, finf))
    return dict(errs=errs, ok=errs["norm"] < 1e-3 and errs["master"] < 1e-5 and errs["lp"] < 1e-2, adam_ms=med,
                adam_gbs=n * (4 * 3 * 2 + 2 + 2) / med / 1e6)


def check_topp():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    bs, V = 8, 50304
    probs = torch.softmax(torch.randn(bs, V, device="cuda") * 3, -1)
    top_ps = torch.full((bs,), 0.8, device="cuda")
    # empirical distribution vs renormalised nucleus
    counts = torch.zeros(bs, V, device="cuda")
    trials = 2000
    for t in range(trials):
        _, ids = lib.topp_sampling(probs, top_ps, 42, t * bs)
        counts.scatter_add_(1, ids, torch.ones_like(ids, dtype=torch.float))
    sp, si = probs.sort(-1, descending=True)
    cum = sp.cumsum(-1)
    in_nucleus_sorted = (cum - sp) < 0.8
    nucleus = torch.zeros_like(probs).scatter(1, si, in_nucleus_sorted.float())
    outside = float((counts * (1 - nucleus)).sum() / counts.sum())
    emp = counts / trials
    # exact law of the sorted-prefix search: u ~ U(0, top_p); token j (sorted) wins on (cum_{j-1}, cum_j] clipped to top_p
    lo = (cum - sp).clamp(max=0.8)
    hi = cum.clamp(max=0.8)
    target = torch.zeros_like(probs).scatter(1, si, (hi - lo) / 0.8)
    tv = float((emp - target).abs().sum(-1).mean()) / 2
    ref_counts = torch.zeros_like(counts)
    ref_ids = torch.multinomial(target, trials, replacement=True)
    ref_counts.scatter_add_(1, ref_ids, torch.ones_like(ref_ids, dtype=torch.float))
    tv_ref = float((ref_counts / trials - target).abs().sum(-1).mean()) / 2
    # half / bf16 inputs run
    _, ids16 = lib.topp_sampling(probs.half(), top_ps, 1, 0)
    med, _ = _time(lambda: lib.topp_sampling(probs, top_ps, 42, 0), flush_mb=1)
    return dict(outside_frac=outside, tv=tv, tv_ref=tv_ref, ok=outside < 2e-3 and tv < 1.3 * tv_ref + 0.01, ms=med, ids16=ids16.flatten().tolist()[:4])


def check_rope_softmax():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    b, s, h, d = 2, 128, 4, 64
    x = torch.randn(b, s, h, d, device="cuda", dtype=torch.bfloat16)
    y = lib.rope(x.view(b * s, h, d), None, s, 10000.0, False).view(b, s, h, d)
    pos = torch.arange(s, device="cuda").float()
    inv = 10000.0 ** (-torch.arange(0, d, 2, device="cuda").float() / d)
    ang = pos[:, None] * inv[None]
    cs, sn = ang.cos()[None, :, None, :], ang.sin()[None, :, None, :]
    xf = x.float(); x1, x2 = xf[..., : d // 2], xf[..., d // 2:]
    ref = torch.cat([x1 * cs - x2 * sn, x2 * cs + x1 * sn], -1)
    back = lib.rope(y.view(b * s, h, d), None, s, 10000.0, True).view(b, s, h, d)
    errs = dict(rope=_relerr(y, ref), rope_inv=_relerr(back, x))
    sc = torch.randn(b * h, s, s, device="cuda", dtype=torch.bfloat16)
    p = lib.causal_softmax_fwd(sc, 0.125)
    scf = sc.float().requires_grad_(True)
    mask = torch.triu(torch.ones(s, s, device="cuda", dtype=torch.bool), 1)
    pref = torch.softmax((scf * 0.125).masked_fill(mask, float("-inf")), -1)
    dyy = torch.randn_like(pref)
    pref.backward(dyy)
    dx = lib.causal_softmax_bwd(dyy.bfloat16(), p, 0.125)
    errs.update(csm=_relerr(p, pref), dcsm=_relerr(dx, scf.grad))
    return dict(errs=errs, ok=all(v < 2e-2 for v in errs.values()))


def check_lowp(kind="int8", M=512, N=512, K=512, cfg=0, time_it=False):
    import torch
    lib = _lib()
    torch.manual_seed(0)
    x = (torch.randn(M, K, device="cuda")).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    bias = torch.randn(N, device="cuda").bfloat16()
    fp8 = kind == "fp8"
    xq, xs = lib.quantize_rows(x, None, fp8)
    wq, ws = lib.quantize_rows(w, None, fp8)
    y = lib.gemm_lowp(xq, wq, xs, ws, bias, cfg)
    torch.cuda.synchronize()
    deq = (xq.float() * xs[:, None]) @ (wq.float() * ws[:, None]).t() + bias.float()
    ref_full = x.float() @ w.float().t() + bias.float()
    res = dict(err_vs_dequant=_relerr(y, deq), err_vs_bf16=_relerr(y, ref_full), quant_err=_relerr(xq.float() * xs[:, None], x))
    res["ok"] = res["err_vs_dequant"] < 1e-2 and res["err_vs_bf16"] < (8e-2 if fp8 else 3e-2)
    if time_it:
        med, best = _time(lambda: lib.gemm_lowp(xq, wq, xs, ws, bias, cfg))
        res.update(ms=med, tops=2.0 * M * N * K / med / 1e9, tops_best=2.0 * M * N * K / best / 1e9)
        med2, _ = _time(lambda: torch.matmul(x, w.t()))
        res.update(bf16_cublas_ms=med2)
    return res


def check_gemv():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    res, ok = {}, True
    for (M, N, K) in [(1, 4096, 4096), (3, 12288, 4096), (8, 4096, 16384), (5, 50304, 4096), (2, 1000, 1032)]:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        y = lib.gemv_skinny(x, w, b)
        ref = x.float() @ w.float().t() + b.float()
        e = _relerr(y, ref)
        ok = ok and e < 1e-2
        med, best = _time(lambda: lib.gemv_skinny(x, w, b))
        med_c, _ = _time(lambda: torch.nn.functional.linear(x, w, b))
        med_t, _ = _time(lambda: lib.gemm(x, w, b, None, True, True, 1, 0, 0))
        res[f"{M}x{N}x{K}"] = dict(err=round(e, 5), ms=round(med, 4), gbs=round(N * K * 2 / med / 1e6, 1), cublas_ms=round(med_c, 4),
                                   wgmma_gemm_ms=round(med_t, 4))
    return dict(ok=ok, shapes=res)


def check_smallm():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    res, ok = {}, True
    for (M, N, K, split) in [(4, 512, 512, 1), (16, 512, 1024, 2), (7, 4096, 4096, 0), (16, 12288, 4096, 0), (33, 4096, 16384, 0),
                             (128, 16384, 4096, 0), (100, 50304, 4096, 0), (8, 4096, 16384, 8), (1, 4096, 4096, 0), (2, 16384, 4096, 0),
                             (128, 4096, 4096, 4)]:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        y = lib.gemm_smallm(x, w, b, split)
        torch.cuda.synchronize()
        ref = x.float() @ w.float().t() + b.float()
        e = _relerr(y, ref)
        ok = ok and e < 1e-2
        med, best = _time(lambda: lib.gemm_smallm(x, w, b, split))
        med_c, _ = _time(lambda: torch.nn.functional.linear(x, w, b))
        row = dict(err=round(e, 5), ms=round(med, 4), gbs=round(N * K * 2 / med / 1e6, 1), cublas_ms=round(med_c, 4))
        if M <= 8:
            med_g, _ = _time(lambda: lib.gemv_skinny(x, w, b))
            row["gemv_ms"] = round(med_g, 4)
        res[f"{M}x{N}x{K}/s{split}"] = row
    return dict(ok=ok, shapes=res)


def check_attention_fwd():
    import torch
    import torch.nn.functional as F
    lib = _lib()
    torch.manual_seed(0)
    res, ok = {}, True
    for (B, Sq, Sk, H, D, causal, timed) in [(1, 128, 128, 2, 128, True, False), (2, 256, 256, 4, 128, False, False), (1, 300, 300, 3, 128, True, False),
                                             (2, 577, 577, 4, 64, False, False), (1, 128, 384, 2, 64, True, False), (8, 1024, 1024, 32, 128, True, True), (2, 4096, 4096, 32, 128, True, True), (16, 512, 512, 32, 128, True, True),
                                             (32, 577, 577, 16, 64, False, True)]:
        q = torch.randn(B, Sq, H, D, device="cuda").bfloat16()
        k = torch.randn(B, Sk, H, D, device="cuda").bfloat16()
        v = torch.randn(B, Sk, H, D, device="cuda").bfloat16()
        scale = D ** -0.5
        out, lse = lib.attention_fwd(q, k, v, causal, scale)
        torch.cuda.synchronize()
        if B * H * Sq * Sk <= (1 << 28):
            s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * scale
            if causal:
                mask = torch.ones(Sq, Sk, dtype=torch.bool, device="cuda").tril(Sk - Sq)
                s = s.masked_fill(~mask, float("-inf"))
            ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v.float())
            e_lse = _relerr(lse, torch.logsumexp(s, -1))
            del s
        else:               # long sequences: compare with the library kernel instead of materialising the score matrix
            ref = F.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), is_causal=causal, scale=scale).transpose(1, 2)
            e_lse = 0.0
        e = _relerr(out, ref)
        ok = ok and e < 1e-2 and e_lse < 1e-3
        row = dict(err=round(e, 5), err_lse=round(e_lse, 6))
        if timed:
            med, _ = _time(lambda: lib.attention_fwd(q, k, v, causal, scale))
            qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
            med_c, _ = _time(lambda: F.scaled_dot_product_attention(qt, kt, vt, is_causal=causal, scale=scale))
            flops = 4.0 * B * H * Sq * Sk * D * (0.5 if causal else 1.0)
            row.update(ms=round(med, 4), tflops=round(flops / med / 1e9, 1), sdpa_ms=round(med_c, 4), sdpa_tflops=round(flops / med_c / 1e9, 1))
        res[f"B{B}_Sq{Sq}_Sk{Sk}_H{H}_D{D}_{'causal' if causal else 'full'}"] = row
    return dict(ok=ok, shapes=res)


def _attn_reference(q, k, v, scale, causal, keep, p):
    """fp32 attention with an explicit keep mask [B,H,Sq,Sk] (or None); returns out and, with autograd, the input grads."""
    import torch
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) * scale
    Sq, Sk = q.shape[1], k.shape[1]
    if causal:
        mask = torch.ones(Sq, Sk, dtype=torch.bool, device=q.device).tril(Sk - Sq)
        s = s.masked_fill(~mask, float("-inf"))
    pr = torch.softmax(s, -1)
    if keep is not None:
        pr = pr * keep.to(pr.dtype) / (1.0 - p)
    return torch.einsum("bhqk,bkhd->bqhd", pr, v)


def check_attention_train(perf=False):
    """forward (with dropout) + backward of the flash kernels against fp32 autograd with the SAME dropout mask, on contiguous, packed-QKV and
    sequence-major layouts; optional timing against library SDPA."""
    import torch
    import torch.nn.functional as F
    from paddlefleetx_b200.ops import attention as ATT
    lib = _lib()
    torch.manual_seed(0)
    res, ok = {}, True
    cases = [  # B, Sq, Sk, H, causal, p, layout, D
        (1, 128, 128, 1, True, 0.0, "plain", 128), (2, 256, 256, 2, True, 0.0, "plain", 128), (1, 320, 320, 2, True, 0.1, "plain", 128),
        (2, 200, 200, 3, False, 0.0, "plain", 128), (1, 128, 256, 2, True, 0.0, "plain", 128), (2, 512, 512, 4, True, 0.1, "packed", 128),
        (2, 384, 384, 2, True, 0.1, "seq_major", 128), (1, 1024, 1024, 4, True, 0.0, "packed", 128),
        # 64-wide heads (GPT-345M, ViT, ERNIE-base): full and causal, ragged, dropout, packed projection layout
        (2, 256, 256, 2, True, 0.0, "plain", 64), (2, 577, 577, 4, False, 0.1, "plain", 64), (1, 1024, 1024, 16, True, 0.1, "packed", 64),
        (2, 197, 197, 3, False, 0.0, "seq_major", 64)]
    for (B, Sq, Sk, H, causal, p, layout, D) in cases:
        scale = D ** -0.5
        if layout == "plain":
            q = torch.randn(B, Sq, H, D, device="cuda").bfloat16(); k = torch.randn(B, Sk, H, D, device="cuda").bfloat16(); v = torch.randn(B, Sk, H, D, device="cuda").bfloat16()
            dq = torch.empty_like(q); dk = torch.empty_like(k); dv = torch.empty_like(v)
        elif layout == "packed":
            mix = torch.randn(B, Sq, H, 3, D, device="cuda").bfloat16(); q, k, v = mix.unbind(3)
            dmix = torch.empty_like(mix); dq, dk, dv = dmix.unbind(3)
        else:
            mix = torch.randn(Sq, B, H, 3, D, device="cuda").bfloat16().transpose(0, 1); q, k, v = mix.unbind(3)
            dmix = torch.empty(Sq, B, H, 3, D, device="cuda", dtype=torch.bfloat16).transpose(0, 1); dq, dk, dv = dmix.unbind(3)
        seed = 0x1234567 + 977 * Sq
        out, lse = lib.attention_fwd_v2(q, k, v, causal, scale, p, seed)
        go = (torch.randn(B, Sq, H, D, device="cuda") * 0.5).bfloat16()
        lib.attention_bwd(q, k, v, out, go, lse, dq, dk, dv, causal, scale, p, seed)
        torch.cuda.synchronize()
        keep = ATT.attn_keep_mask(seed, B, H, Sq, Sk, p, "cuda") if p > 0 else None
        qr, kr, vr = (t.detach().float().requires_grad_(True) for t in (q, k, v))
        ref = _attn_reference(qr, kr, vr, scale, causal, keep, p)
        ref.backward(go.float())
        errs = dict(out=_relerr(out, ref), dq=_relerr(dq, qr.grad), dk=_relerr(dk, kr.grad), dv=_relerr(dv, vr.grad))
        if keep is not None:
            errs["keep_rate"] = round(float(keep.float().mean()), 4)
        good = all(errs[n] < 2e-2 for n in ("out", "dq", "dk", "dv"))
        ok = ok and good
        res[f"B{B}_Sq{Sq}_Sk{Sk}_H{H}_D{D}_{'causal' if causal else 'full'}_p{p}_{layout}"] = {n: round(float(e), 5) for n, e in errs.items()}
    out_d = dict(ok=ok, shapes=res)
    if perf:
        for (B, S, H, D) in [(8, 1024, 32, 128), (2, 4096, 32, 128), (16, 1024, 16, 64)]:
            mix = torch.randn(B, S, H, 3, D, device="cuda").bfloat16(); q, k, v = mix.unbind(3)
            dmix = torch.empty_like(mix); dq, dk, dv = dmix.unbind(3)
            go = torch.randn(B, S, H, D, device="cuda").bfloat16()
            scale = D ** -0.5
            for p in (0.0, 0.1):
                out, lse = lib.attention_fwd_v2(q, k, v, True, scale, p, 7)
                t_f, _ = _time(lambda: lib.attention_fwd_v2(q, k, v, True, scale, p, 7))
                t_b, _ = _time(lambda: lib.attention_bwd(q, k, v, out, go, lse, dq, dk, dv, True, scale, p, 7))
                qt, kt, vt = (t.transpose(1, 2).detach().requires_grad_(True) for t in (q.contiguous(), k.contiguous(), v.contiguous()))
                got = go.transpose(1, 2)
                t_sf, _ = _time(lambda: F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, dropout_p=p, scale=scale))

                def sd_fb():
                    o = F.scaled_dot_product_attention(qt, kt, vt, is_causal=True, dropout_p=p, scale=scale)
                    o.backward(got)
                    qt.grad = kt.grad = vt.grad = None
                t_sfb, _ = _time(sd_fb)
                fl = 4.0 * B * H * S * S * D * 0.5
                out_d[f"perf_B{B}_S{S}_H{H}{'' if D == 128 else '_D64'}_p{p}"] = dict(fwd_ms=round(t_f, 4), fwd_tflops=round(fl / t_f / 1e9, 1), bwd_ms=round(t_b, 4),
                                                         bwd_tflops=round(2.5 * fl / t_b / 1e9, 1), sdpa_fwd_ms=round(t_sf, 4),
                                                         sdpa_fwd_bwd_ms=round(t_sfb, 4), ours_fwd_bwd_ms=round(t_f + t_b, 4))
    return out_d


def check_attention_autograd():
    """The autograd wrappers (plain and packed) against fp32 autograd; no dropout (mask replication is covered by attention_train)."""
    import torch
    from paddlefleetx_b200.ops import attention as ATT
    torch.manual_seed(1)
    B, S, H, D = 2, 256, 4, 128
    mix = torch.randn(B, S, H, 3, D, device="cuda").bfloat16().requires_grad_(True)
    go = torch.randn(B, S, H, D, device="cuda").bfloat16()
    out = ATT.flash_attention_packed(mix, causal=True)
    assert out is not None
    out.backward(go)
    q, k, v = (t.detach().float().requires_grad_(True) for t in mix.detach().unbind(3))
    ref = _attn_reference(q, k, v, D ** -0.5, True, None, 0.0)
    ref.backward(go.float())
    gref = torch.stack([q.grad, k.grad, v.grad], dim=3)
    e1, e2 = _relerr(out, ref), _relerr(mix.grad, gref)
    q2, k2, v2 = (torch.randn(B, S, H, D, device="cuda").bfloat16().requires_grad_(True) for _ in range(3))
    o2 = ATT.attention(q2, k2, v2, causal=False)
    o2.backward(go)
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q2, k2, v2))
    r2 = _attn_reference(qf, kf, vf, D ** -0.5, False, None, 0.0)
    r2.backward(go.float())
    e3 = max(_relerr(q2.grad, qf.grad), _relerr(k2.grad, kf.grad), _relerr(v2.grad, vf.grad), _relerr(o2, r2))
    return dict(ok=bool(max(e1, e2, e3) < 2e-2), err_out=e1, err_packed_grad=e2, err_plain=e3)


def check_fused_ffn():
    """Dual-output bias+GELU epilogue, dGELU epilogue and the FFN autograd node built on them vs fp32 PyTorch; timing vs the unfused chain."""
    import torch
    import torch.nn.functional as F
    lib = _lib()
    from paddlefleetx_b200.ops import functional as OF
    torch.manual_seed(0)
    errs = {}
    for (M, H, Fh) in [(300, 256, 1032), (1024, 512, 2048)]:
        x = torch.randn(M, H, device="cuda").bfloat16()
        w1 = (torch.randn(Fh, H, device="cuda") * 0.05).bfloat16()
        b1 = (torch.randn(Fh, device="cuda") * 0.1).bfloat16()
        z, g = lib.gemm_bias_gelu_dual(x, w1, b1)
        zr = x.float() @ w1.float().t() + b1.float()
        errs[f"dual_z_{M}"] = _relerr(z, zr)
        errs[f"dual_g_{M}"] = _relerr(g, F.gelu(zr, approximate="tanh"))
        dy = torch.randn(M, H, device="cuda").bfloat16()
        w2 = (torch.randn(H, Fh, device="cuda") * 0.05).bfloat16()
        dz = lib.gemm_dgelu(dy, w2, z)
        zf = z.float().requires_grad_(True)
        (F.gelu(zf, approximate="tanh") * (dy.float() @ w2.float())).sum().backward()
        errs[f"dgelu_{M}"] = _relerr(dz, zf.grad)
    # autograd node vs the unfused chain (same kernels otherwise) and vs fp32
    M, H, Fh = 2048, 1024, 4096
    xs = [torch.randn(M, H, device="cuda").bfloat16().requires_grad_(True) for _ in range(2)]
    xs[1].data.copy_(xs[0].data)
    mk = lambda: [(torch.randn(Fh, H, device="cuda") * 0.03).bfloat16().requires_grad_(True), (torch.randn(Fh, device="cuda") * 0.1).bfloat16().requires_grad_(True),
                  (torch.randn(H, Fh, device="cuda") * 0.03).bfloat16().requires_grad_(True)]
    torch.manual_seed(1); pa = mk()
    torch.manual_seed(1); pb = mk()
    gy = torch.randn(M, H, device="cuda").bfloat16()
    ya = OF.fused_ffn(xs[0], pa[0], pa[1], pa[2]); ya.backward(gy)
    yb = OF.linear(OF.bias_gelu(OF.linear(xs[1], pb[0], None), pb[1]), pb[2], None); yb.backward(gy)
    errs["ffn_y"] = _relerr(ya, yb)
    errs["ffn_dx"] = _relerr(xs[0].grad, xs[1].grad)
    for n, a, b in zip(("dw1", "db1", "dw2"), pa, pb):
        errs["ffn_" + n] = _relerr(a.grad, b.grad)
    ok = all(e < 1.5e-2 for e in errs.values())
    M, H, Fh = 8192, 4096, 16384
    x = torch.randn(M, H, device="cuda").bfloat16().requires_grad_(True)
    w1 = (torch.randn(Fh, H, device="cuda") * 0.02).bfloat16().requires_grad_(True)
    b1 = torch.zeros(Fh, device="cuda").bfloat16().requires_grad_(True)
    w2 = (torch.randn(H, Fh, device="cuda") * 0.02).bfloat16().requires_grad_(True)
    gy = torch.randn(M, H, device="cuda").bfloat16()
    def fused():
        OF.fused_ffn(x, w1, b1, w2).backward(gy)
    def chain():
        OF.linear(OF.bias_gelu(OF.linear(x, w1, None), b1), w2, None).backward(gy)
    t_f, _ = _time(fused, iters=8, warmup=2)
    t_c, _ = _time(chain, iters=8, warmup=2)
    return dict(ok=ok, errs={k: round(v, 5) for k, v in errs.items()}, fwd_bwd_ms_fused=round(t_f, 4), fwd_bwd_ms_unfused=round(t_c, 4))


def check_gemv_tuning():
    """Sweep the GEMV launch shape (weight rows per warp x K-slices per block) on the decode shapes of GPT-6.7B, L2 cold and warm."""
    import torch
    lib = _lib()
    torch.manual_seed(0)
    out = {}
    for (M, N, K) in [(1, 4096, 4096), (1, 12288, 4096), (1, 16384, 4096), (1, 4096, 16384), (1, 50304, 4096)]:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        row = {}
        for cols in (2, 4):
            for split in (1, 2, 4, 8):
                lib.gemv_set_tuning(cols, split)
                med, best = _time(lambda: lib.gemv_skinny(x, w, None), iters=15)
                row[f"c{cols}s{split}"] = round(N * K * 2 / med / 1e6)
        lib.gemv_set_tuning(0, 0)
        med, _ = _time(lambda: lib.gemv_skinny(x, w, None), iters=15)
        row["auto"] = round(N * K * 2 / med / 1e6)
        # back-to-back (no L2 flush, as inside the decode graph): 8 different weight matrices round-robin > L2
        ws = [w] + [(torch.randn(N, K, device="cuda") * 0.05).bfloat16() for _ in range(3)]
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(3):
            for wi in ws:
                lib.gemv_skinny(x, wi, None)
        e0.record()
        for _ in range(10):
            for wi in ws:
                lib.gemv_skinny(x, wi, None)
        e1.record(); torch.cuda.synchronize()
        row["auto_back_to_back"] = round(N * K * 2 * 40 / e0.elapsed_time(e1) / 1e6)
        out[f"{M}x{N}x{K}"] = row
    return dict(ok=True, gbs=out)


def check_decode_fused():
    import torch
    import torch.nn.functional as F
    lib = _lib()
    torch.manual_seed(0)
    errs = {}
    for (M, N, K) in [(1, 12288, 4096), (2, 4096, 16384), (1, 1000, 1032)]:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.03).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        g = (1 + 0.1 * torch.randn(K, device="cuda")).bfloat16()
        be = (0.1 * torch.randn(K, device="cuda")).bfloat16()
        res = torch.randn(M, N, device="cuda").bfloat16()
        y = lib.gemv_fused(x, w, b, g, be, 1e-5, res, 1)
        ref = F.gelu(F.layer_norm(x.float(), (K,), g.float(), be.float(), 1e-5) @ w.float().t() + b.float(), approximate="tanh") + res.float()
        errs[f"ln_gelu_res_{M}x{N}x{K}"] = _relerr(y, ref)
        y2 = lib.gemv_fused(x, w, None, None, None, 1e-5, res, 0)
        errs[f"res_{M}x{N}x{K}"] = _relerr(y2, x.float() @ w.float().t() + res.float())
    B, H, D, Lmax = 2, 32, 128, 136
    qkv = torch.randn(B, 1, H, 3, D, device="cuda").bfloat16()
    k = torch.randn(B, Lmax, H, D, device="cuda").bfloat16()
    v = torch.randn(B, Lmax, H, D, device="cuda").bfloat16()
    pos = 77
    valid = torch.zeros(B, Lmax, dtype=torch.bool, device="cuda")
    valid[:, :pos + 1] = True
    mask = torch.zeros(B, 1, 1, Lmax, device="cuda").masked_fill(~valid.view(B, 1, 1, Lmax), -1e4).bfloat16()
    k_ref, v_ref = k.clone(), v.clone()
    k_ref[:, pos], v_ref[:, pos] = qkv[:, 0, :, 1], qkv[:, 0, :, 2]
    idx = torch.tensor([pos], device="cuda")
    out = lib.attention_decode_packed(qkv, k, v, mask, idx, D ** -0.5)
    sc = torch.einsum("bqhd,bkhd->bhqk", qkv[:, :, :, 0].float(), k_ref.float()) * D ** -0.5 + mask.float()
    ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(sc, -1), v_ref.float())
    errs["attn_packed"] = _relerr(out, ref)
    errs["cache_k"] = float((k - k_ref).abs().max())
    errs["cache_v"] = float((v - v_ref).abs().max())
    ok = all(e < 1e-2 for kk, e in errs.items() if not kk.startswith("cache")) and errs["cache_k"] == 0 and errs["cache_v"] == 0
    return dict(ok=ok, errs={kk: round(e, 5) for kk, e in errs.items()})


def check_gemv_w8a8():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    res, ok = {}, True
    for (M, N, K) in [(1, 4096, 4096), (2, 12288, 4096), (8, 4096, 16384), (4, 16384, 4096), (1, 1000, 1040)]:
        x = torch.randn(M, K, device="cuda").bfloat16()
        w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
        b = torch.randn(N, device="cuda").bfloat16()
        xq, xs = lib.quantize_rows(x, None, False)
        wq, ws = lib.quantize_rows(w, None, False)
        y = lib.gemv_w8a8(xq, wq, xs, ws, b)
        deq = (xq.float() * xs[:, None]) @ (wq.float() * ws[:, None]).t() + b.float()
        e = _relerr(y, deq)
        ok = ok and e < 5e-3
        med, _ = _time(lambda: lib.gemv_w8a8(xq, wq, xs, ws, b))
        med_b, _ = _time(lambda: lib.gemv_skinny(x, w, b))
        res[f"{M}x{N}x{K}"] = dict(err=round(e, 5), ms=round(med, 4), gbs=round(N * K / med / 1e6, 1), bf16_gemv_ms=round(med_b, 4))
    return dict(ok=ok, shapes=res)


def check_attention_decode():
    import torch
    lib = _lib()
    torch.manual_seed(0)
    res, ok = {}, True
    for (B, H, D, Lmax, L) in [(1, 32, 128, 136, 136), (4, 32, 128, 1024, 1024), (3, 16, 64, 200, 200), (16, 32, 128, 136, 136)]:
        q = torch.randn(B, 1, H, D, device="cuda").bfloat16()
        k = torch.randn(B, Lmax, H, D, device="cuda").bfloat16()
        v = torch.randn(B, Lmax, H, D, device="cuda").bfloat16()
        valid = torch.rand(B, Lmax, device="cuda") > 0.3
        valid[:, 0] = True
        mask = torch.zeros(B, 1, 1, Lmax, device="cuda").masked_fill(~valid.view(B, 1, 1, Lmax), -1e4).bfloat16()
        scale = D ** -0.5
        y = lib.attention_decode(q, k, v, mask, L, scale)
        s = torch.einsum("bqhd,bkhd->bhqk", q.float(), k.float()) * scale + mask.float()
        ref = torch.einsum("bhqk,bkhd->bqhd", torch.softmax(s, -1), v.float())
        e = _relerr(y, ref)
        ok = ok and e < 1e-2
        med, _ = _time(lambda: lib.attention_decode(q, k, v, mask, L, scale))
        med_s, _ = _time(lambda: torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=mask, scale=scale))
        res[f"B{B}xH{H}xD{D}xL{L}"] = dict(err=round(e, 5), ms=round(med, 4), gbs=round(2 * B * L * H * D * 2 / med / 1e6, 1), sdpa_ms=round(med_s, 4))
    return dict(ok=ok, shapes=res)


def check_embedding():
    """Fused word + position look-up and the sorted scatter-add gradient against F.embedding autograd in fp32 (repeated ids, a vocabulary shard
    with foreign ids, the main_grad store / accumulate protocol, > 16 K tokens)."""
    import torch
    import torch.nn.functional as F
    from paddlefleetx_b200.ops import functional as OF
    torch.manual_seed(0)
    res, ok = {}, True
    for (V, H, B, S, start, with_pos) in [(1000, 256, 4, 128, 0, True), (512, 1024, 2, 64, 256, False), (50304, 512, 20, 1024, 0, True)]:
        w = (torch.randn(V if start == 0 else 256, H, device="cuda") * 0.1).bfloat16().requires_grad_(True)
        pw = (torch.randn(S, H, device="cuda") * 0.1).bfloat16().requires_grad_(True) if with_pos else None
        ids = torch.randint(0, V, (B, S), device="cuda")
        ids[0, :8] = ids[0, 0]                        # a run of repeats
        pos = torch.arange(S, device="cuda").expand(B, S).contiguous()
        go = torch.randn(B, S, H, device="cuda").bfloat16()
        out = OF.embedding(ids, w, start, pos if with_pos else None, pw)
        out.backward(go)
        wr = w.detach().float().requires_grad_(True)
        local = ids - start
        oob = (local < 0) | (local >= wr.shape[0])
        ref = F.embedding(local.masked_fill(oob, 0), wr).masked_fill(oob.unsqueeze(-1), 0.0)
        if with_pos:
            pr = pw.detach().float().requires_grad_(True)
            ref = ref + F.embedding(pos, pr)
        ref.backward(go.float())
        errs = dict(out=_relerr(out, ref), dw=_relerr(w.grad, wr.grad))
        if with_pos:
            errs["dpos"] = _relerr(pw.grad, pr.grad)
        good = all(e < 1e-2 for e in errs.values())
        ok = ok and good
        res[f"V{V}_H{H}_T{B * S}_start{start}"] = {k: round(float(v), 5) for k, v in errs.items()}
    # main_grad protocol: fresh -> zero + rows; then accumulate on top of an existing gradient
    w = (torch.randn(300, 128, device="cuda") * 0.1).bfloat16().requires_grad_(True)
    w.main_grad = torch.full((300, 128), 7.0, device="cuda", dtype=torch.float32)
    w._grad_fresh = True
    ids = torch.randint(0, 300, (3, 50), device="cuda")
    go = torch.randn(3, 50, 128, device="cuda").bfloat16()
    OF.embedding(ids, w).backward(go)
    want = torch.zeros(300, 128, device="cuda").index_add_(0, ids.reshape(-1), go.float().reshape(-1, 128))
    e1 = _relerr(w.main_grad, want)
    w.grad = None
    OF.embedding(ids, w).backward(go)                  # second micro-batch: accumulates
    e2 = _relerr(w.main_grad, 2 * want)
    ok = ok and e1 < 1e-5 and e2 < 1e-5 and not w._grad_fresh
    res["main_grad"] = dict(store=e1, accumulate=e2)
    return dict(ok=ok, cases=res)


def check_norm_residual():
    """Pre-norm block pattern: out = x_res + f(norm(x)); the residual gradient is added inside the norm-backward kernel."""
    import torch
    from paddlefleetx_b200.ops import functional as OF
    torch.manual_seed(0)
    ok, res = True, {}
    for rms in (False, True):
        x = torch.randn(512, 1024, device="cuda").bfloat16().requires_grad_(True)
        w = (1 + 0.1 * torch.randn(1024, device="cuda")).bfloat16().requires_grad_(True)
        b = None if rms else (0.1 * torch.randn(1024, device="cuda")).bfloat16().requires_grad_(True)
        g = torch.randn(512, 1024, device="cuda").bfloat16()
        OF.reset_launch_count()
        h, xr = OF.norm_with_residual(x, w, b, 1e-5, rms)
        out = xr + torch.tanh(h)
        out.backward(g)
        xf, wf = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True)
        if rms:
            hf = xf * torch.rsqrt(xf.pow(2).mean(-1, keepdim=True) + 1e-5) * wf
        else:
            bf = b.detach().float().requires_grad_(True)
            hf = torch.nn.functional.layer_norm(xf, (1024,), wf, bf, 1e-5)
        (xf + torch.tanh(hf)).backward(g.float())
        e = dict(dx=_relerr(x.grad, xf.grad), dw=_relerr(w.grad, wf.grad))
        ok = ok and max(e.values()) < 2e-2
        res["rms" if rms else "ln"] = {k: round(float(v), 5) for k, v in e.items()}
    return dict(ok=ok, cases=res)


def check_gemm_big_sweep():
    """Multi-tile shapes (several tiles per CTA, dozens of k-blocks, ragged edges) for every
    (CTA-group, operand majors, output mode) against fp32."""
    worst, rows, ok = 0.0, {}, True
    for cfg in (1, 2, 3, 4):
        for (a_k, b_k) in ((True, True), (True, False), (False, False), (False, True)):
            for out_mode in (0, 1, 2):
                M, N, K = (4096 + 128, 2048 + 64, 1536) if cfg in (1, 2) else (3072, 1024 + 128, 2048)
                r = check_gemm(a_k, b_k, cfg, M, N, K, out_mode=out_mode, epilogue=1 if out_mode == 0 else 0)
                rows[f"cfg{cfg}_{'K' if a_k else 'M'}{'K' if b_k else 'N'}_out{out_mode}"] = round(r["err"], 5)
                worst = max(worst, r["err"])
                ok = ok and r["ok"]
    return dict(ok=ok, worst=worst, cases=rows)


def check_moe_grouped(perf=False):
    """Grouped expert GEMMs against an fp32 per-expert loop: synthetic segment tables (an expert without tokens, unused blocks at the end, 128-
    and 256-row alignment = 1-CTA and 2-CTA tiles), the tile-table kernel, forward + backward of the whole grouped FFN."""
    import torch
    import torch.nn.functional as F
    from paddlefleetx_b200.models.language_model.moe.grouped_experts import GroupedExperts, grouped_ffn
    from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer
    from paddlefleetx_b200.ops import _native
    lib = _native.require()
    res, ok = {}, True
    cases = [(4, 256, 512, [300, 0, 129, 700], 256, 4096), (3, 128, 384, [5, 640, 130], 128, 1536), (8, 1024, 4096, [1500, 2100, 1800, 0, 2500, 1900, 2222, 1777], 256, 20480)]
    if perf:
        cases = cases[-1:]
    for (E, hm, ffn, counts, align, cap) in cases:
        torch.manual_seed(E)
        ex = [ExpertLayer(hm, ffn, init_std=0.05, dtype=torch.bfloat16, device="cuda") for _ in range(E)]
        holder = torch.nn.ModuleList(ex)
        ge = GroupedExperts(ex)
        with torch.no_grad():
            ge.b1.normal_(0, 0.1); ge.b2.normal_(0, 0.1)
        starts, pos = [], 0
        for c in counts:
            starts.append(pos)
            pos += (c + align - 1) // align * align
        seg = torch.tensor(starts + counts + [pos, 0], dtype=torch.int32, device="cuda")
        sticky = torch.zeros(1, dtype=torch.int32, device="cuda")
        tile_group, seg2 = lib.moe_tile_table(seg, E, align, cap, sticky)
        tg = tile_group.tolist()
        want = [-1] * (cap // 128)
        for e, (s0, c) in enumerate(zip(starts, counts)):
            for t in range(s0 // 128, (s0 + (c + align - 1) // align * align) // 128):
                want[t] = e
        table_ok = tg == want and int(sticky) == 0
        xs = torch.full((cap, hm), float("nan"), device="cuda", dtype=torch.bfloat16)     # unused rows are poisoned: nothing may read them
        go = torch.full((cap, hm), float("nan"), device="cuda", dtype=torch.bfloat16)
        for s0, c in zip(starts, counts):
            pad = (c + align - 1) // align * align
            xs[s0:s0 + pad] = 0; go[s0:s0 + pad] = 0
            xs[s0:s0 + c] = (torch.randn(c, hm, device="cuda") * 0.5).bfloat16()
            go[s0:s0 + c] = (torch.randn(c, hm, device="cuda") * 0.1).bfloat16()
        xs.requires_grad_(True)
        ys = grouped_ffn(xs, tile_group, seg2, ge, None, align)
        ys.backward(go)
        # fp32 reference over the real rows
        errs = {}
        w1, b1, w2, b2 = (t.detach().float() for t in (ge.w1, ge.b1, ge.w2, ge.b2))
        for e, (s0, c) in enumerate(zip(starts, counts)):
            dw1 = torch.zeros_like(w1[e]); dw2 = torch.zeros_like(w2[e]); db1 = torch.zeros_like(b1[e]); db2 = torch.zeros_like(b2[e])
            if c:
                xe = xs.detach()[s0:s0 + c].float().requires_grad_(True)
                pw = [t.clone().requires_grad_(True) for t in (w1[e], b1[e], w2[e], b2[e])]
                ye = F.linear(F.gelu(F.linear(xe, pw[0], pw[1]), approximate="tanh"), pw[2], pw[3])
                ye.backward(go[s0:s0 + c].float())
                errs[f"y{e}"] = _relerr(ys.detach()[s0:s0 + c], ye.detach())
                errs[f"dx{e}"] = _relerr(xs.grad[s0:s0 + c], xe.grad)
                dw1, db1, dw2, db2 = (t.grad for t in pw)
                for nm, got, ref in (("dw1", ge.w1.grad[e], dw1), ("db1", ge.b1.grad[e], db1), ("dw2", ge.w2.grad[e], dw2), ("db2", ge.b2.grad[e], db2)):
                    errs[f"{nm}_{e}"] = _relerr(got, ref)
            else:   # an expert without tokens: exact zero gradients, written (not left uninitialised)
                errs[f"empty{e}"] = float(max(ge.w1.grad[e].float().abs().max(), ge.w2.grad[e].float().abs().max(), ge.b1.grad[e].float().abs().max()))
        worst = max(errs.values())
        finite = bool(torch.isfinite(ge.w1.grad.float()).all() and torch.isfinite(ge.w2.grad.float()).all())
        case_ok = table_ok and worst < 2e-2 and finite
        ok = ok and case_ok
        r = dict(ok=case_ok, tile_table_ok=table_ok, worst=round(worst, 5), finite=finite)
        if perf:
            def step():
                xs.grad = None
                grouped_ffn(xs, tile_group, seg2, ge, None, align).backward(go)
            ms, _ = _time(step)
            rows = sum(counts)
            r["fwd_bwd_ms"] = round(ms, 4)
            r["tflops"] = round(3 * 2 * 2 * rows * hm * ffn / ms / 1e9, 1)
            def loop():
                for e, (s0, c) in enumerate(zip(starts, counts)):
                    if c:
                        xe = xs.detach()[s0:s0 + c].requires_grad_(True)
                        ge.bind_views()
                        ex[e](xe).backward(go[s0:s0 + c])
            ms_loop, _ = _time(loop)
            r["per_expert_loop_ms"] = round(ms_loop, 4)
        res[f"E{E}_h{hm}_ffn{ffn}_align{align}"] = r
    return dict(ok=ok, cases=res)


def check_evoformer_attention(perf=False):
    """Evoformer gated attention kernel against the fp32 expression: both biases, gating, ragged lengths, several key tiles, heads 4 / 8; the
    chunked backward against autograd of the same expression."""
    import torch
    from paddlefleetx_b200.ops import evoformer_attention as EA
    torch.manual_seed(0)
    res, ok = {}, True
    #        G   gpp Sq   Sk   H  mask  pair  gate
    cases = [(4, 4, 128, 128, 4, True, True, True), (6, 3, 200, 200, 8, True, True, True), (2, 1, 300, 77, 2, True, False, True),
             (3, 3, 64, 384, 4, False, True, False), (8, 8, 256, 256, 8, True, True, True)]
    if perf:
        cases = [(256, 256, 256, 256, 8, True, True, True), (128, 128, 384, 384, 8, True, True, True)]
    for (G, gpp, Sq, Sk, H, wm, wp, wg) in cases:
        mk = lambda *sh: (torch.randn(*sh, device="cuda") * 0.7).bfloat16()
        q, k, v = mk(G, Sq, H, 32), mk(G, Sk, H, 32), mk(G, Sk, H, 32)
        mask = None
        if wm:
            keep = (torch.rand(G, Sk, device="cuda") > 0.15).float()
            keep[:, 0] = 1
            mask = (keep - 1.0) * 1e9
        pair = mk(G // gpp, H, Sq, Sk) if wp else None
        gate = mk(G, Sq, H, 32) if wg else None
        name = f"G{G}_Sq{Sq}_Sk{Sk}_H{H}" + ("_mask" if wm else "") + ("_pair" if wp else "") + ("_gate" if wg else "")
        if perf:
            out = EA.evoformer_attention(q, k, v, mask, pair, gate, gpp)
            ms, _ = _time(lambda: EA.evoformer_attention(q, k, v, mask, pair, gate, gpp))
            def eager():
                return EA.reference(q, k, v, mask, pair, gate, gpp, 32 ** -0.5).to(q.dtype)
            ms_ref, _ = _time(eager)
            def sdpa():
                m = mask.view(G, 1, 1, Sk) + pair.float().repeat_interleave(gpp, 0)
                o = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2), attn_mask=m.to(q.dtype))
                return o.transpose(1, 2) * torch.sigmoid(gate)
            ms_sdpa, _ = _time(sdpa)
            flops = 4.0 * G * H * Sq * Sk * 32
            # forward + backward through autograd: native kernel pair vs the chunked recomputation vs SDPA autograd with a materialised mask
            leaves = [t.clone().requires_grad_(True) for t in (q, k, v, pair, gate)]
            go = torch.randn_like(out)

            def fb():
                for t in leaves:
                    t.grad = None
                EA.evoformer_attention(leaves[0], leaves[1], leaves[2], mask, leaves[3], leaves[4], gpp).backward(go)
            ms_fb, _ = _time(fb)
            EA._BWD = "torch"
            ms_fb_torch, _ = _time(fb)
            EA._BWD = "native"

            def sdpa_fb():
                for t in leaves:
                    t.grad = None
                m = mask.view(G, 1, 1, Sk) + leaves[3].float().repeat_interleave(gpp, 0)
                o = torch.nn.functional.scaled_dot_product_attention(leaves[0].transpose(1, 2), leaves[1].transpose(1, 2), leaves[2].transpose(1, 2), attn_mask=m.to(q.dtype))
                (o.transpose(1, 2) * torch.sigmoid(leaves[4])).backward(go)
            ms_fb_sdpa, _ = _time(sdpa_fb)
            res[name] = dict(ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1), eager_fp32_ms=round(ms_ref, 4), sdpa_masked_ms=round(ms_sdpa, 4),
                             err=round(_relerr(out, eager()), 5), fwd_bwd_ms=round(ms_fb, 4), fwd_bwd_chunked_torch_ms=round(ms_fb_torch, 4),
                             fwd_bwd_sdpa_ms=round(ms_fb_sdpa, 4))
            continue
        leaves = [t.clone().requires_grad_(True) for t in (q, k, v)] + [t.clone().requires_grad_(True) if t is not None else None for t in (pair, gate)]
        out = EA.evoformer_attention(leaves[0], leaves[1], leaves[2], mask, leaves[3], leaves[4], gpp)
        ref_leaves = [t.detach().float().requires_grad_(True) for t in (q, k, v)] + [t.detach().float().requires_grad_(True) if t is not None else None for t in (pair, gate)]
        ref = EA.reference(ref_leaves[0], ref_leaves[1], ref_leaves[2], mask, ref_leaves[3], ref_leaves[4], gpp, 32 ** -0.5)
        go = torch.randn_like(ref)
        out.backward(go.to(out.dtype))
        ref.backward(go)
        errs = {"out": _relerr(out, ref)}
        for nm, a, b in zip(("dq", "dk", "dv", "dpair", "dgate"), leaves, ref_leaves):
            if a is not None:
                errs[nm] = _relerr(a.grad, b.grad)
        case_ok = max(errs.values()) < 2e-2
        ok = ok and case_ok
        res[name] = dict(ok=case_ok, **{k_: round(v_, 5) for k_, v_ in errs.items()})
    return dict(ok=ok, cases=res)


def _mx_decode(q, sf):
    """(e4m3 [R, K], scale atoms) -> fp32 [R, K]: the value the tensor core sees."""
    import torch
    R, K = q.shape
    r = torch.arange(R, device=q.device).view(R, 1)
    kb = torch.arange(K // 32, device=q.device).view(1, -1)
    idx = ((r // 128) * (K // 128) + kb // 4) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + (kb % 4)
    e = sf.reshape(-1)[idx].float()                                   # [R, K / 32]
    return q.float() * torch.exp2(e - 127).repeat_interleave(32, dim=1)


def _mx_encode_sf(e_rows_kb):
    """[R, K / 32] uint8 exponents -> atom-ordered scale tensor."""
    import torch
    R, KB = e_rows_kb.shape
    sf = torch.full(((R + 127) // 128, KB // 4, 512), 127, dtype=torch.uint8, device=e_rows_kb.device)
    r = torch.arange(R, device=sf.device).view(R, 1)
    kb = torch.arange(KB, device=sf.device).view(1, -1)
    idx = ((r // 128) * (KB // 4) + kb // 4) * 512 + (r % 32) * 16 + ((r % 128) // 32) * 4 + (kb % 4)
    sf.view(-1)[idx.reshape(-1)] = e_rows_kb.reshape(-1)
    return sf


def check_gemm_mxfp8(perf=False):
    """MX block-scaled fp8 GEMM in stages that isolate each piece of the protocol: unit
    scales, per-row A scales (lane / column mapping), per-K-block scales (sf_id), B scales, then quantiser + GEMM against fp32."""
    import torch
    lib = _lib()
    torch.manual_seed(0)
    res, ok = {}, True
    M, N, K = 300, 384, 512
    a = (torch.randn(M, K, device="cuda") * 2).to(torch.float8_e4m3fn)
    b = (torch.randn(N, K, device="cuda") * 2).to(torch.float8_e4m3fn)
    ones = lambda R: torch.full((R, K // 32), 127, dtype=torch.uint8, device="cuda")
    rnd = lambda R, per_row, per_k: (127 + torch.randint(-6, 7, (R if per_row else 1, K // 32 if per_k else 1), device="cuda")).to(torch.uint8).expand(R, K // 32).contiguous()
    stages = {"unit_scales": (ones(M), ones(N)), "a_row_scales": (rnd(M, True, False), ones(N)), "a_kblock_scales": (rnd(M, False, True), ones(N)),
              "b_row_scales": (ones(M), rnd(N, True, False)), "b_kblock_scales": (ones(M), rnd(N, False, True)), "all_scales": (rnd(M, True, True), rnd(N, True, True))}
    for name, (ea, eb) in stages.items():
        sfa, sfb = _mx_encode_sf(ea), _mx_encode_sf(eb)
        d = lib.gemm_mxfp8(a, sfa, b, sfb)
        ref = _mx_decode(a, sfa) @ _mx_decode(b, sfb).t()
        e = _relerr(d, ref)
        res[name] = round(e, 5)
        ok = ok and e < 1e-2
    # quantiser: round trip and layout
    x = (torch.randn(M, K, device="cuda") * torch.logspace(-2, 2, K // 32, device="cuda").repeat_interleave(32)).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    qx, sx = lib.quantize_mxfp8(x)
    qw, sw = lib.quantize_mxfp8(w)
    res["quant_roundtrip"] = round(_relerr(_mx_decode(qx, sx), x), 5)
    bias = torch.randn(N, device="cuda").bfloat16()
    d = lib.gemm_mxfp8(qx, sx, qw, sw, bias)
    res["gemm_vs_dequantised"] = round(_relerr(d, _mx_decode(qx, sx) @ _mx_decode(qw, sw).t() + bias.float()), 5)
    res["gemm_vs_fp32"] = round(_relerr(d, x.float() @ w.float().t() + bias.float()), 5)
    ok = ok and res["quant_roundtrip"] < 6e-2 and res["gemm_vs_dequantised"] < 1e-2 and res["gemm_vs_fp32"] < 6e-2
    out = dict(ok=ok, **res)
    if perf:
        M2, N2, K2 = 8192, 8192, 8192
        x2, w2 = torch.randn(M2, K2, device="cuda").bfloat16(), torch.randn(N2, K2, device="cuda").bfloat16()
        qx2, sx2 = lib.quantize_mxfp8(x2); qw2, sw2 = lib.quantize_mxfp8(w2)
        ms, _ = _time(lambda: lib.gemm_mxfp8(qx2, sx2, qw2, sw2))
        mq, _ = _time(lambda: lib.quantize_mxfp8(x2))
        out["perf_8192"] = dict(gemm_ms=round(ms, 4), tflops=round(2.0 * M2 * N2 * K2 / ms / 1e9, 1), quantize_ms=round(mq, 4),
                                quantize_gbs=round(M2 * K2 * 3 / mq / 1e6, 1))
    return out


def check_sync_audit():
    """Host <-> device synchronisations inside a training step, found with torch's sync debug mode: steps of a small GPT and of a small
    GPT-MoE on the sync-free path (expert group of one rank).  Reports every distinct Python call site that made the host wait."""
    import collections
    import traceback
    import warnings

    import torch
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_gpu_models as T                     # reuse the tiny recipes and the engine builder
    from paddlefleetx_b200.utils import config as C

    out, ok = {}, True
    for name, recipe, extra in (("gpt", "nlp/gpt/pretrain_gpt_345M_single_card.yaml", []),
                                ("moe_sync_free", "nlp/moe/pretrain_moe_345M_single_card.yaml", ["Model.moe_configs.fused_p2p=True"])):
        cfg = C.get_config(os.path.join(T.CFG, recipe), T.SMALL_GPT + extra, nranks=1)
        eng = T._engine(cfg)
        batch = [t.cuda() for t in T._gpt_batches(cfg, 1)[0]]
        for _ in range(3):
            eng.train_step(batch)                   # warm-up: lazy initialisation may sync
        torch.cuda.synchronize()
        sites = collections.Counter()
        torch.cuda.set_sync_debug_mode(1)
        try:
            with warnings.catch_warnings(record=True) as rec:
                warnings.simplefilter("always")
                for _ in range(2):
                    loss = eng.train_step(batch)
                n_warn = len(rec)
                for w in rec:
                    sites[f"{os.path.relpath(w.filename, ROOT) if w.filename.startswith(ROOT) else os.path.basename(w.filename)}:{w.lineno}"] += 1
        finally:
            torch.cuda.set_sync_debug_mode(0)
        out[name] = dict(syncs_in_2_steps=n_warn, sites=dict(sites.most_common(12)), loss=float(loss))
    return dict(ok=ok, **out)


CHECKS = {
    "sync_audit": check_sync_audit,
    "gemm_mxfp8": check_gemm_mxfp8,
    "gemm_mxfp8_perf": lambda: check_gemm_mxfp8(perf=True),
    "evoformer_attention": check_evoformer_attention,
    "evoformer_attention_perf": lambda: check_evoformer_attention(perf=True),
    "moe_grouped": check_moe_grouped,
    "moe_grouped_perf": lambda: check_moe_grouped(perf=True),
    "attention_train": check_attention_train,
    "attention_train_perf": lambda: check_attention_train(perf=True),
    "attention_autograd": check_attention_autograd,
    "gemm_big_sweep": check_gemm_big_sweep,
    "embedding": check_embedding,
    "norm_residual": check_norm_residual,
    "attention_decode": check_attention_decode,
    "gemv_w8a8": check_gemv_w8a8,
    "decode_fused": check_decode_fused,
    "gemv_tuning": check_gemv_tuning,
    "fused_ffn": check_fused_ffn,
    "attention_fwd": check_attention_fwd,
    "gemm_smallm": check_smallm,
    "gemv_skinny": check_gemv,
    "gemm_nt_1cta": lambda: check_gemm(True, True, 1),
    "gemm_nt_1cta_n128": lambda: check_gemm(True, True, 3),
    "gemm_nt_2cta": lambda: check_gemm(True, True, 2),
    "gemm_nt_2cta_n128": lambda: check_gemm(True, True, 4),
    "gemm_nn_1cta": lambda: check_gemm(True, False, 1),
    "gemm_tn_1cta": lambda: check_gemm(False, False, 1),
    "gemm_tk_1cta": lambda: check_gemm(False, True, 1),
    "gemm_nn_2cta": lambda: check_gemm(True, False, 2),
    "gemm_tn_2cta": lambda: check_gemm(False, False, 2),
    "gemm_tail": lambda: check_gemm(True, True, 1, M=300, N=264, K=136),
    "gemm_tail_2cta": lambda: check_gemm(True, True, 2, M=300, N=264, K=136),
    "gemm_bias_gelu": lambda: check_gemm(True, True, 1, epilogue=2),
    "gemm_f32_acc": lambda: check_gemm(False, False, 2, out_mode=2),
    "gemm_f32": lambda: check_gemm(True, True, 1, out_mode=1),
    "gemm_perf_1cta": lambda: check_gemm(True, True, 1, 8192, 8192, 8192, time_it=True),
    "gemm_perf_2cta": lambda: check_gemm(True, True, 2, 8192, 8192, 8192, time_it=True),
    "gemm_perf_ffn1": lambda: check_gemm(True, True, 2, 8192, 16384, 4096, epilogue=1, time_it=True),
    "gemm_perf_dgrad": lambda: check_gemm(True, False, 2, 8192, 4096, 16384, time_it=True),
    "gemm_perf_wgrad": lambda: check_gemm(False, False, 2, 16384, 4096, 8192, out_mode=1, time_it=True),
    "gemm_int8": lambda: check_lowp("int8"),
    "gemm_int8_pair": lambda: check_lowp("int8", 1024, 1024, 1024, 2),
    "gemm_fp8": lambda: check_lowp("fp8"),
    "gemm_fp8_pair": lambda: check_lowp("fp8", 1024, 1024, 1024, 2),
    "gemm_int8_perf": lambda: check_lowp("int8", 8192, 8192, 8192, 2, True),
    "gemm_fp8_perf": lambda: check_lowp("fp8", 8192, 8192, 8192, 2, True),
    "layernorm": lambda: check_norm(False),
    "rmsnorm": lambda: check_norm(True),
    "gelu_dropout": check_gelu_dropout,
    "cross_entropy": check_ce,
    "adamw": check_adam,
    "topp": check_topp,
    "rope_softmax": check_rope_softmax,
}


def main():
    os.makedirs(OUT, exist_ok=True)
    if len(sys.argv) == 2 and sys.argv[1] in CHECKS:
        name = sys.argv[1]
        try:
            res = CHECKS[name]()
        except Exception as e:  # noqa: BLE001
            res = dict(ok=False, error=repr(e)[:500])
        print("RESULT " + json.dumps(dict(check=name, **res)))
        return
    names = sys.argv[1:] or list(CHECKS)
    log = open(os.path.join(OUT, "selftest.log"), "a")
    n_ok = 0
    n_timeouts = 0
    for name in names:
        t0 = time.time()
        if n_timeouts >= 3 and name.startswith("gemm"):
            print(json.dumps(dict(check=name, ok=False, error="skipped after repeated timeouts")), flush=True)
            continue
        try:
            p = subprocess.run([sys.executable, os.path.abspath(__file__), name], capture_output=True, text=True, timeout=180)
            line = [l for l in p.stdout.splitlines() if l.startswith("RESULT ")]
            res = json.loads(line[-1][7:]) if line else dict(check=name, ok=False, rc=p.returncode,
                                                             tail=(p.stdout[-600:] + p.stderr[-1200:]))
        except subprocess.TimeoutExpired:
            res = dict(check=name, ok=False, error="timeout")
            n_timeouts += 1
        res["wall_s"] = round(time.time() - t0, 1)
        n_ok += bool(res.get("ok"))
        msg = json.dumps(res)
        print(msg, flush=True)
        log.write(msg + "\n"); log.flush()
    print(f"SELFTEST {n_ok}/{len(names)} ok")


if __name__ == "__main__":
    main()
