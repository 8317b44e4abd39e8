"""Ring attention with packed documents (``RingDocumentMask``) against the plain causal ring, on one H100.

    python tools/bench_ring_doc_attention.py                 # one JSON line per shape, dtype and document length, then a table
    python tools/bench_ring_doc_attention.py --rounds 5 --iters 10

One GPU plays every rank of a ring of c in turn: for rank r it runs the c attention blocks that rank computes in a step (the diagonal block
and the c - 1 blocks from the other ranks, with the ``_block_plan`` shapes of parallel/ring_attention.py), each one flash-kernel call.  A
step waits for the slowest rank, so the reported time is the maximum over ranks of the time of its blocks.  The transfers, the
online-softmax merge and the dK / dV accumulation are outside the timed window (they are the same with and without documents), and so is
the bounds launch (one per step in training).  Shapes: c 4 and 8, s 32 k and 64 k, one sequence, H 16, D 128, bf16 and fp16; every row
is packed from documents of 512, 2048 or 8192 tokens, or holds one document ("row"); one grouped shape (Hkv 4).  Times are forward and
forward + backward from CUDA events around ``--iters`` repetitions (medians over rounds, the arms alternating inside every round).  The
card name and power limit are read in the same process (``nvidia-smi --query-gpu=name,power.limit``).
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

from bench_doc_attention import _card, _time_ms, positions  # noqa: E402

H, D = 16, 128
SHAPES = [(c, s, H) for c in (4, 8) for s in (32768, 65536)] + [(8, 32768, 4)]     # (c, s, kv heads)
DOC_LENS = (512, 2048, 8192, "row")


def rank_schedule(lib, q, k, v, go, c, r, mask, scale):
    """(forward, forward + backward) closures over rank r's c blocks; ``mask`` is the rank's RingDocumentMask or None (causal ring)."""
    import torch

    from paddlefleetx_b200.parallel.ring_attention import _block_plan

    half = q.shape[1] // 2
    blocks = []
    for src in range(c):
        qs, ks, causal = _block_plan(True, r, src, half)
        qb, kb, vb, gb = q[:, qs], k[:, ks], v[:, ks], go[:, qs]
        grads = [torch.empty_like(t) for t in (qb, kb, vb)]
        blocks.append((qb, kb, vb, gb, grads, causal, None if mask is None else mask.block(src)))

    def fwd(b):
        qb, kb, vb, _, _, causal, doc = b
        if doc is None:
            return lib.attention_fwd_v2(qb, kb, vb, causal, scale, 0.0, 0)
        return lib.attention_fwd_doc(qb, kb, vb, *doc.bounds(), scale, 0.0, 0, causal)

    def bwd(b, o, l):
        qb, kb, vb, gb, g, causal, doc = b
        if doc is None:
            lib.attention_bwd(qb, kb, vb, o, gb, l, *g, causal, scale, 0.0, 0)
        else:
            lib.attention_bwd_doc(qb, kb, vb, o, gb, l, *g, *doc.bounds(), scale, 0.0, 0, causal)

    def forward():
        for b in blocks:
            fwd(b)

    def both():
        for b in blocks:
            o, l = fwd(b)
            bwd(b, o, l)

    return forward, both


def main():
    """Time the causal ring and the document arms of every shape, rank by rank, and print one JSON line per arm and a Markdown table."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    import torch

    from paddlefleetx_b200.ops import _native
    from paddlefleetx_b200.parallel.ring_attention import RingDocumentMask, zigzag_slice

    if not torch.cuda.is_available():
        raise SystemExit("bench_ring_doc_attention needs a CUDA device")
    lib = _native.require()
    card = _card()
    print(json.dumps({"card": card, "torch": torch.__version__}), flush=True)
    rows = []
    for dt in (torch.bfloat16, torch.float16):
        for c, s, hkv in SHAPES:
            if hkv != H and dt != torch.bfloat16:
                continue
            s_l = s // c
            q, go = (torch.randn(1, s_l, H, D, device="cuda", dtype=dt) for _ in range(2))
            k, v = (torch.randn(1, s_l, hkv, D, device="cuda", dtype=dt) for _ in range(2))
            scale = D ** -0.5
            arms = {"causal": [None] * c}
            for L in DOC_LENS:
                pos = positions(1, s, L, "cuda")
                arms[L] = [RingDocumentMask.from_positions(zigzag_slice(pos, c, r), c, r) for r in range(c)]
            sched = {name: [rank_schedule(lib, q, k, v, go, c, r, m[r], scale) for r in range(c)] for name, m in arms.items()}
            for per_rank in sched.values():
                for _, fb in per_rank:
                    for _ in range(a.warmup):
                        fb()
            times = {name: [([], []) for _ in range(c)] for name in arms}
            for _ in range(a.rounds):
                for name, per_rank in sched.items():
                    for r, (f, fb) in enumerate(per_rank):
                        times[name][r][0].append(_time_ms(f, a.iters))
                        times[name][r][1].append(_time_ms(fb, a.iters))
            step = {name: tuple(max(statistics.median(t[i]) for t in per) for i in (0, 1)) for name, per in times.items()}
            base_f, base_fb = step["causal"]
            for name in arms:
                mf, mfb = step[name]
                r_ = {"dtype": str(dt).split(".")[-1], "c": c, "s": s, "kv_heads": hkv, "doc_len": name, "fwd_ms": round(mf, 3),
                      "fwd_bwd_ms": round(mfb, 3), "fwd_speedup": round(base_f / mf, 2), "fwd_bwd_speedup": round(base_fb / mfb, 2), "card": card}
                rows.append(r_)
                print(json.dumps(r_), flush=True)
    print(f"\n{card}: one sequence, H {H}, D {D}; the slowest rank's attention blocks per step, speed-up against the causal ring")
    print("| dtype | c | s | Hkv | doc length | fwd ms | fwd+bwd ms | fwd speed-up | fwd+bwd speed-up |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r_ in rows:
        print(f"| {r_['dtype']} | {r_['c']} | {r_['s']} | {r_['kv_heads']} | {r_['doc_len']} | {r_['fwd_ms']} | {r_['fwd_bwd_ms']} | "
              f"{r_['fwd_speedup']} | {r_['fwd_bwd_speedup']} |")


if __name__ == "__main__":
    main()
