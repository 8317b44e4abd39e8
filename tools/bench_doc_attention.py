"""Intra-document causal attention (``DocumentMask``) against plain causal attention on one H100.

    python tools/bench_doc_attention.py                      # one JSON line per shape, dtype and document length, then a table
    python tools/bench_doc_attention.py --rounds 5 --iters 20

Shapes hold b x s at 16 k tokens (s 2048 / 4096 / 8192), H 16, D 128, in bf16 and fp16; every row is packed from documents of 128, 512 or
2048 tokens, or holds one document ("row").  For each shape the plain causal kernel runs at the same size, alternating with the document
arms inside every round.  Times are forward and forward + backward from CUDA events around ``--iters`` launches (medians over rounds).
``tflops`` counts only the useful work, from the attended pairs sum_i (i - key_start[i] + 1): 4 D FLOPs per pair forward, 10 D backward,
so a kernel that skips masked tiles shows a higher time saving than rate.  The bounds derivation (one small launch per step in training)
is outside the timed window.  The card name and power limit are read in the same process (``nvidia-smi --query-gpu=name,power.limit``).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TOKENS, H, D = 16384, 16, 128
SEQS = (2048, 4096, 8192)
DOC_LENS = (128, 512, 2048, "row")


def pairs(key_start) -> int:
    """Attended (query, key) pairs of a [b, s] key_start: sum over rows of i - key_start[i] + 1."""
    import torch

    i = torch.arange(key_start.shape[1], device=key_start.device)
    return int((i - key_start.long() + 1).sum())


def positions(b: int, s: int, doc_len, device="cpu"):
    import torch

    i = torch.arange(s, device=device)
    pos = i if doc_len == "row" else i % doc_len
    return pos.unsqueeze(0).expand(b, s).contiguous()


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


def _card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return "unknown"


def main():
    """Time the causal and document-mask arms of every shape, alternating within each round, and print one JSON line per arm and a
    Markdown table of times, useful TFLOP/s and speed-ups."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch

    from paddlefleetx_b200.ops import _native
    from paddlefleetx_b200.ops.attention import DocumentMask

    if not torch.cuda.is_available():
        raise SystemExit("bench_doc_attention needs a CUDA device")
    lib = _native.require()
    card = _card()
    print(json.dumps({"card": card, "torch": torch.__version__}), flush=True)
    rows = []
    for dt in (torch.bfloat16, torch.float16):
        for s in SEQS:
            b = TOKENS // s
            mix = torch.randn(b, s, H, 3, D, device="cuda", dtype=dt)
            q, k, v = mix.unbind(3)
            dmix = torch.empty_like(mix)
            dq, dk, dv = dmix.unbind(3)
            go = torch.randn(b, s, H, D, device="cuda", dtype=dt)
            scale = D ** -0.5
            arms = {"causal": None}
            for L in DOC_LENS:
                if L == "row" or L < s:
                    arms[L] = DocumentMask.from_positions(positions(b, s, L, "cuda"))

            def fns(doc):
                if doc is None:
                    fwd = lambda: lib.attention_fwd_v2(q, k, v, True, scale, 0.0, 0)
                    bwd = lambda o, l: lib.attention_bwd(q, k, v, o, go, l, dq, dk, dv, True, scale, 0.0, 0)
                else:
                    fwd = lambda: lib.attention_fwd_doc(q, k, v, *doc.bounds(), scale, 0.0, 0)
                    bwd = lambda o, l: lib.attention_bwd_doc(q, k, v, o, go, l, dq, dk, dv, *doc.bounds(), scale, 0.0, 0)

                def both():
                    o, l = fwd()
                    bwd(o, l)
                return fwd, both

            times = {name: ([], []) for name in arms}
            for name, doc in arms.items():
                f, fb = fns(doc)
                for _ in range(a.warmup):
                    fb()
            for _ in range(a.rounds):
                for name, doc in arms.items():
                    f, fb = fns(doc)
                    times[name][0].append(_time_ms(f, a.iters))
                    times[name][1].append(_time_ms(fb, a.iters))
            causal_pairs = b * s * (s + 1) // 2
            base_f, base_fb = (statistics.median(t) for t in times["causal"])
            for name, doc in arms.items():
                n = causal_pairs if doc is None else pairs(doc.key_start)
                mf, mfb = (statistics.median(t) for t in times[name])
                r = {"dtype": str(dt).split(".")[-1], "s": s, "b": b, "doc_len": name, "pairs": n, "fwd_ms": round(mf, 3),
                     "fwd_bwd_ms": round(mfb, 3), "fwd_tflops": round(4 * D * n * H / mf / 1e9, 1),
                     "fwd_bwd_tflops": round(14 * D * n * H / mfb / 1e9, 1), "fwd_speedup": round(base_f / mf, 2),
                     "fwd_bwd_speedup": round(base_fb / mfb, 2), "card": card}
                rows.append(r)
                print(json.dumps(r), flush=True)
    print(f"\n{card}: b*s = {TOKENS}, H {H}, D {D}; speed-up against the plain causal kernel at the same shape")
    print("| dtype | s | doc length | fwd ms | fwd+bwd ms | fwd TFLOP/s | fwd+bwd TFLOP/s | fwd speed-up | fwd+bwd speed-up |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['dtype']} | {r['s']} | {r['doc_len']} | {r['fwd_ms']} | {r['fwd_bwd_ms']} | {r['fwd_tflops']} | {r['fwd_bwd_tflops']} | "
              f"{r['fwd_speedup']} | {r['fwd_bwd_speedup']} |")


if __name__ == "__main__":
    main()
