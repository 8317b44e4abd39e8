"""The grouped expert FFN (``GroupedFFN``) on one H100: GELU experts, SwiGLU experts with the activation inside the grouped GEMM epilogues,
and the unfused SwiGLU composition the fused epilogues replace.

    python tools/bench_moe_ffn.py                 # one JSON line per arm and alignment, then a table
    python tools/bench_moe_ffn.py --rounds 5 --iters 20

Shape: E = 8 experts, H = 2048, F = 5632 (SwiGLU; 8H/3 rounded up to 256) or 8192 (GELU, 4H), bf16, 16384 routed rows (8192 tokens,
top-2) spread unevenly over the experts in a capacity buffer of twice that, with 128- and 256-row expert alignment.  Arms:

    gelu       GroupedFFN, GELU experts: EPI_BIAS_GELU_DUAL -> EPI_BIAS, backward EPI_DGELU
    swiglu     GroupedFFN, SwiGLU experts: EPI_BIAS_SWIGLU_DUAL -> EPI_BIAS, backward EPI_DSWIGLU
    unfused    the same SwiGLU FFN as EPI_BIAS + ``bias_swiglu_fwd`` over the capacity buffer -> EPI_BIAS, backward EPI_NONE +
               ``bias_swiglu_bwd``; every other launch as in GroupedFFN

Forward and forward + backward from CUDA events around ``--iters`` repetitions (medians over rounds, the arms alternating inside every
round).  The fused and unfused SwiGLU outputs are compared on the same inputs.  The card name and power limit are read in the same process.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_doc_attention import _card, _time_ms  # noqa: E402

E, H, ROWS = 8, 2048, 16384
F_OF = {"gelu": 8192, "swiglu": 5632, "unfused": 5632}


def _layout(lib, align, device):
    """Uneven per-expert row counts summing to ROWS, each expert padded to ``align``, in a capacity buffer of 2 ROWS."""
    import torch

    g = torch.Generator().manual_seed(0)
    w = torch.rand(E, generator=g) + 0.5
    counts = (w / w.sum() * ROWS).long()
    counts[-1] += ROWS - int(counts.sum())
    starts, pos = [], 0
    for c in counts.tolist():
        starts.append(pos)
        pos += (c + align - 1) // align * align
    cap = 2 * ROWS
    seg = torch.tensor(starts + counts.tolist() + [pos, 0], dtype=torch.int32, device=device)
    tile_group, seg2 = lib.moe_tile_table(seg, E, align, cap, torch.zeros(1, dtype=torch.int32, device=device))
    return starts, counts.tolist(), cap, tile_group, seg2


def _unfused(lib, xs, tile_group, seg2, ge, align, go=None):
    """The SwiGLU expert FFN without the fused epilogues: returns ys, or runs the backward too when ``go`` is given."""
    import torch

    from paddlefleetx_b200.models.language_model.moe.grouped_experts import EPI_BIAS, EPI_NONE

    rows = xs.shape[0]
    pre = torch.empty(rows, ge.w1.shape[1], dtype=xs.dtype, device=xs.device)
    lib.gemm_grouped(xs, ge.w1, ge.b1, tile_group, pre, True, EPI_BIAS, None, None, align)
    h = lib.bias_swiglu_fwd(pre, None)
    ys = torch.empty_like(xs)
    lib.gemm_grouped(h, ge.w2, ge.b2, tile_group, ys, True, EPI_BIAS, None, None, align)
    if go is None:
        return ys
    dw2 = torch.empty_like(ge.w2)
    lib.gemm_grouped_wgrad(go, h, seg2, dw2)
    lib.grouped_colsum(go, seg2, E)
    dh = torch.empty(rows, ge.w2.shape[2], dtype=xs.dtype, device=xs.device)
    lib.gemm_grouped(go, ge.w2, None, tile_group, dh, False, EPI_NONE, None, None, align)
    dpre = lib.bias_swiglu_bwd(dh, pre, None)
    dw1 = torch.empty_like(ge.w1)
    lib.gemm_grouped_wgrad(dpre, xs, seg2, dw1)
    lib.grouped_colsum(dpre, seg2, E)
    dxs = torch.empty_like(xs)
    lib.gemm_grouped(dpre, ge.w1, None, tile_group, dxs, False, EPI_NONE, None, None, align)
    return ys


def main():
    """Time the three arms at both alignments, print one JSON line per arm and a Markdown table."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch

    from paddlefleetx_b200.models.language_model.moe.grouped_experts import GroupedExperts, grouped_ffn
    from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer
    from paddlefleetx_b200.ops import _native

    if not torch.cuda.is_available():
        raise SystemExit("bench_moe_ffn needs a CUDA device")
    lib = _native.require()
    card = _card()
    dev, dt = torch.device("cuda"), torch.bfloat16
    experts = {}
    for act in ("gelu", "swiglu"):
        torch.manual_seed(1)
        ex = [ExpertLayer(H, F_OF[act], init_std=0.02, dtype=dt, device=dev, activation=act) for _ in range(E)]
        experts[act] = (ex, GroupedExperts(ex))
    results = []
    for align in (128, 256):
        starts, counts, cap, tile_group, seg2 = _layout(lib, align, dev)
        g = torch.Generator(device=dev).manual_seed(align)
        xs = torch.zeros(cap, H, device=dev, dtype=dt)
        go = torch.zeros(cap, H, device=dev, dtype=dt)
        for s0, c in zip(starts, counts):
            xs[s0:s0 + c] = (torch.randn(c, H, device=dev, generator=g) * 0.5).to(dt)
            go[s0:s0 + c] = (torch.randn(c, H, device=dev, generator=g) * 0.1).to(dt)
        xg = xs.clone().requires_grad_(True)

        def arm(name, backward):
            ge = experts["gelu" if name == "gelu" else "swiglu"][1]
            if name == "unfused":
                return lambda: _unfused(lib, xs, tile_group, seg2, ge, align, go if backward else None)
            if backward:
                def step():
                    xg.grad = None
                    grouped_ffn(xg, tile_group, seg2, ge, None, align).backward(go)
                return step
            return lambda: grouped_ffn(xs, tile_group, seg2, ge, None, align)

        with torch.no_grad():
            fused_y = grouped_ffn(xs, tile_group, seg2, experts["swiglu"][1], None, align)
            unfused_y = _unfused(lib, xs, tile_group, seg2, experts["swiglu"][1], align)
            real = torch.cat([torch.arange(s0, s0 + c, device=dev) for s0, c in zip(starts, counts)])
            diff = float((fused_y[real].float() - unfused_y[real].float()).norm() / unfused_y[real].float().norm())
        names = ("gelu", "swiglu", "unfused")
        times = {(n, b): [] for n in names for b in (False, True)}
        for n in names:
            for b in (False, True):
                for _ in range(a.warmup):
                    arm(n, b)()
        for _ in range(a.rounds):
            for b in (False, True):
                for n in names:
                    times[(n, b)].append(_time_ms(arm(n, b), a.iters))
        for n in names:
            f = F_OF[n]
            ffn1 = 2 * f if n != "gelu" else f
            flops = 2 * ROWS * H * (ffn1 + f)
            fwd, fb = statistics.median(times[(n, False)]), statistics.median(times[(n, True)])
            r = dict(arm=n, align=align, experts=E, hidden=H, ffn=f, rows=ROWS, capacity=cap, fwd_ms=round(fwd, 4), fwd_bwd_ms=round(fb, 4),
                     fwd_tflops=round(flops / fwd / 1e9, 1), fwd_bwd_tflops=round(3 * flops / fb / 1e9, 1), card=card)
            if n == "unfused":
                r["fused_vs_unfused_rel_diff"] = diff
            results.append(r)
            print(json.dumps(r), flush=True)
    print(f"\n{card}, E {E}, H {H}, {ROWS} routed rows, bf16; medians of {a.rounds} rounds of {a.iters} calls\n")
    print("| align | arm | F | fwd ms | fwd+bwd ms | fwd+bwd TFLOP/s |")
    print("|---|---|---|---|---|---|")
    for r in results:
        print(f"| {r['align']} | {r['arm']} | {r['ffn']} | {r['fwd_ms']} | {r['fwd_bwd_ms']} | {r['fwd_bwd_tflops']} |")


if __name__ == "__main__":
    main()
