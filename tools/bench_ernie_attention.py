"""ERNIE's padded attention: the key-padding flash kernels (``KeyPaddingMask``) against PyTorch SDPA on the additive ``[b, 1, 1, s]`` mask
that ERNIE used before, on one H100.

    python tools/bench_ernie_attention.py                 # one JSON line per shape, dtype and padding pattern, then a table
    python tools/bench_ernie_attention.py --rounds 5 --iters 20

Shapes at s = 512, batch 8: ERNIE-base (H 12, D 64) and the 10B-class encoder (H 32, D 128, the heads of one rank at mp 2), bf16 and
fp16.  Padding: none, 25 % and 50 % right padding on every row, and a random interior pattern (each key padding with probability 0.25).
Both arms run through autograd as a training step does (``attention(..., attn_mask=mask)`` and ``F.scaled_dot_product_attention``); the
mask is built once outside the timed window, as it is built once per step for all layers.  Times are forward and forward + backward from
CUDA events around ``--iters`` repetitions (medians over rounds, the arms alternating inside every round).  The card name and power limit
are read in the same process.
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

B, S = 8, 512
SHAPES = [("ernie-base", 12, 64), ("ernie-10b", 32, 128)]
PADDING = ("0%", "25%", "50%", "interior")


def valid_rows(kind: str, device):
    """bool [B, S]: the real tokens of each row."""
    import torch

    if kind == "interior":
        g = torch.Generator().manual_seed(0)
        return (torch.rand(B, S, generator=g) >= 0.25).to(device)
    n = S - S * int(kind[:-1]) // 100
    return (torch.arange(S, device=device) < n).expand(B, S).contiguous()


def main():
    """Time SDPA and the key-padding kernels for every shape, dtype and padding, print one JSON line per case and a Markdown table."""
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch
    import torch.nn.functional as F

    from paddlefleetx_b200.ops import _native
    from paddlefleetx_b200.ops import attention as ATT

    if not torch.cuda.is_available():
        raise SystemExit("bench_ernie_attention needs a CUDA device")
    _native.require()
    card = _card()
    print(json.dumps({"card": card, "torch": torch.__version__}), flush=True)
    rows = []
    for name, H, D in SHAPES:
        for dt in (torch.bfloat16, torch.float16):
            q, k, v, go = (torch.randn(B, S, H, D, device="cuda", dtype=dt) for _ in range(4))
            for t in (q, k, v):
                t.requires_grad_(True)
            for kind in PADDING:
                valid = valid_rows(kind, "cuda")
                pad = ATT.KeyPaddingMask.from_valid(valid.float(), dt)
                additive = pad.additive().to(dt)

                def sdpa():
                    return F.scaled_dot_product_attention(*(t.transpose(1, 2) for t in (q, k, v)), attn_mask=additive).transpose(1, 2)

                def native():
                    return ATT.attention(q, k, v, causal=False, attn_mask=pad)

                arms = {}
                for arm, fn in (("sdpa", sdpa), ("keypad", native)):
                    def fwd(fn=fn):
                        with torch.no_grad():
                            fn()

                    def both(fn=fn):
                        fn().backward(go)
                    arms[arm] = (fwd, both)
                for fwd, both in arms.values():
                    for _ in range(a.warmup):
                        fwd(); both()
                times = {arm: ([], []) for arm in arms}
                for _ in range(a.rounds):
                    for arm, (fwd, both) in arms.items():
                        times[arm][0].append(_time_ms(fwd, a.iters))
                        times[arm][1].append(_time_ms(both, a.iters))
                med = {arm: (statistics.median(t[0]), statistics.median(t[1])) for arm, t in times.items()}
                r = {"shape": name, "H": H, "D": D, "b": B, "s": S, "dtype": str(dt).split(".")[-1], "padding": kind,
                     "valid_frac": round(float(valid.float().mean()), 3),
                     "sdpa_fwd_ms": round(med["sdpa"][0], 3), "keypad_fwd_ms": round(med["keypad"][0], 3),
                     "sdpa_fwd_bwd_ms": round(med["sdpa"][1], 3), "keypad_fwd_bwd_ms": round(med["keypad"][1], 3),
                     "fwd_speedup": round(med["sdpa"][0] / med["keypad"][0], 2), "fwd_bwd_speedup": round(med["sdpa"][1] / med["keypad"][1], 2),
                     "card": card}
                rows.append(r)
                print(json.dumps(r), flush=True)
    print(f"\n{card}: b {B}, s {S}; key-padding kernels against SDPA with the additive [b, 1, 1, s] mask")
    print("| shape | dtype | padding | SDPA fwd ms | ours fwd ms | SDPA fwd+bwd ms | ours fwd+bwd ms | fwd speed-up | fwd+bwd speed-up |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in rows:
        print(f"| {r['shape']} | {r['dtype']} | {r['padding']} | {r['sdpa_fwd_ms']} | {r['keypad_fwd_ms']} | {r['sdpa_fwd_bwd_ms']} | "
              f"{r['keypad_fwd_bwd_ms']} | {r['fwd_speedup']} | {r['fwd_bwd_speedup']} |")


if __name__ == "__main__":
    main()
