"""Grouped-query attention kernels on one H100: flash forward + backward and the decode step for several K/V head counts.

    python tools/bench_gqa.py                      # prints one JSON line per shape and arm, then a summary line
    python tools/bench_gqa.py --rounds 5 --iters 50

Flash: forward + backward (causal, bf16) on the packed ``[b, s, Hkv, G + 2, d]`` projection output the GPT model hands the kernels, at
b 8, s 1024, H 16, d 128 (GPT-1.3B's attention) for Hkv in {16, 4, 1}, and b 1, s 1024 for Hkv in {16, 1}: with one K/V head and one
sequence the backward grid has only 16 CTAs (one per 64-key tile), the underfill listed in docs/design.md.
Decode: the packed decode step (cache append + attention over the whole static cache) at cache length 2048, batch {1, 8, 32}, for the
same Hkv.  ``kv_bytes`` is the unique K/V cache bytes one step must read (2 x b x L x Hkv x d x 2 bytes); ``kv_GBps`` is those bytes over
the step time.  Query heads of one group read the same cache rows, so traffic beyond the unique bytes may be served from L2.

The arms of one shape alternate within each round, every shape is warmed up before timing, and every time comes from CUDA events around
``--iters`` launches.  The card name and power limit are read in the same process (``nvidia-smi --query-gpu=name,power.limit``, read only).
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

H, D, S_FLASH, L_DECODE = 16, 128, 1024, 2048
KV_HEADS = (16, 4, 1)


def _time_ms(fn, iters: int) -> float:
    import torch

    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def flash_arm(lib, b: int, hkv: int):
    import torch

    g = H // hkv
    mix = torch.randn(b, S_FLASH, hkv, g + 2, D, device="cuda", dtype=torch.bfloat16)
    dmix = torch.empty_like(mix)
    go = torch.randn(b, S_FLASH, H, D, device="cuda", dtype=torch.bfloat16)
    split = (lambda m: m.unbind(3)) if g == 1 else (lambda m: (m[:, :, :, :g], m[:, :, :, g], m[:, :, :, g + 1]))
    (q, k, v), (dq, dk, dv) = split(mix), split(dmix)
    scale = D ** -0.5

    def step():
        out, lse = lib.attention_fwd_v2(q, k, v, True, scale, 0.0, 0)
        lib.attention_bwd(q, k, v, out, go, lse, dq, dk, dv, True, scale, 0.0, 0)
    return step


def decode_arm(lib, b: int, hkv: int):
    import torch

    g = H // hkv
    qkv = torch.randn(b, 1, hkv, g + 2, D, device="cuda", dtype=torch.bfloat16)
    kc = torch.randn(b, L_DECODE, hkv, D, device="cuda", dtype=torch.bfloat16)
    vc = torch.randn_like(kc)
    mask = torch.zeros(b, L_DECODE, device="cuda", dtype=torch.bfloat16)
    idx = torch.tensor([L_DECODE - 1], device="cuda")
    return lambda: lib.attention_decode_packed(qkv, kc, vc, mask, idx, D ** -0.5)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5, help="alternating rounds per shape")
    ap.add_argument("--iters", type=int, default=30, help="launches per timed window (flash); decode uses 10x")
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()

    import torch

    from bench_precision import gpu_info
    from paddlefleetx_b200.ops import _native

    assert torch.cuda.is_available(), "bench_gqa.py needs a CUDA device"
    lib = _native.require()
    info = gpu_info()
    groups = [("flash_fwd_bwd", 8, KV_HEADS, flash_arm, a.iters), ("flash_fwd_bwd", 1, (16, 1), flash_arm, a.iters)]
    groups += [("decode", b, KV_HEADS, decode_arm, 10 * a.iters) for b in (1, 8, 32)]
    summary = []
    for kind, b, kvs, make, iters in groups:
        arms = {hkv: make(lib, b, hkv) for hkv in kvs}
        for fn in arms.values():
            for _ in range(a.warmup):
                fn()
        times = {hkv: [] for hkv in kvs}
        for _ in range(a.rounds):
            for hkv, fn in arms.items():
                times[hkv].append(_time_ms(fn, iters))
        for hkv in kvs:
            t = times[hkv]
            rec = dict(info, kind=kind, b=b, H=H, Hkv=hkv, d=D, ms=round(statistics.median(t), 4), ms_min=round(min(t), 4), ms_max=round(max(t), 4))
            if kind == "decode":
                kv_bytes = 2 * b * L_DECODE * hkv * D * 2
                rec.update(L=L_DECODE, kv_bytes=kv_bytes, kv_GBps=round(kv_bytes / (rec["ms"] * 1e-3) / 1e9, 1))
            else:
                rec.update(s=S_FLASH)
            print(json.dumps(rec), flush=True)
            summary.append(rec)
        del arms
        torch.cuda.empty_cache()
    print(json.dumps(dict(info, summary=[{k: r[k] for k in ("kind", "b", "Hkv", "ms")} for r in summary])))


if __name__ == "__main__":
    main()
