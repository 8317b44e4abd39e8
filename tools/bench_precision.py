"""float16 against bfloat16 on the headline GPT-1.3B single-GPU step, and the kernels behind it, on one H100.

    python tools/bench_precision.py --steps 20 --warmup 5            # arms fp16, bf16, fp16, bf16: one subprocess each
    python tools/bench_precision.py --kernels                         # GEMM, flash-attention and SwiGLU timings in both dtypes

Step mode builds the exact configuration of ``bench.py --gpus 1`` (``bench.build_config``) and changes only
``Engine.mix_precision.dtype``.  Each arm runs in its own process under bench.py's rules: W untimed warm-up steps, then K steps
bracketed by synchronisation and CUDA events.  float16 trains with the dynamic loss scaler (initial scale ``scale_loss`` = 32768): the
line reports the final scale and how many timed steps it skipped.  Every line carries the GPU name and power limit read in the same
process (``nvidia-smi --query-gpu=name,power.limit``, read only).

Kernel mode times the persistent GEMM at GPT-1.3B's Linear shapes (8 x 1024 tokens, hidden 2048: QKV, attention output, FFN1, FFN2 and
the tied LM head with vocabulary 50304) in the forward and dgrad forms and in three wgrad forms: ``wgrad_bf16`` stores into a 16-bit
[out, in] gradient buffer (out mode 0, what a training step without fp32 main gradients runs on a fresh gradient), ``wgrad_f32`` stores
into an fp32 main gradient (out mode 1) and ``wgrad_f32acc`` accumulates into it (out mode 2).  Each row gives TFLOP/s and the share of
the H100 SXM data-sheet dense rate (989 TFLOP/s).  The backward forms a training step runs (every dgrad, the FFN2 dgrad with the GELU
derivative in its epilogue, ``dgelu``, and the 16-bit wgrad) are timed at both tiles of the GEMM, ``tile`` 128x128 (config 0) and
128x256 (config 1, what the backward asks for), alternating, two windows each; ``ms`` is their mean.  Flash attention forward + backward runs at b 8, s 1024, h 16, d 128 (causal).  The
SwiGLU kernels run at the shapes of the SwiGLU GPT-1.3B recipe (F = 5632): ``bias_swiglu`` forward and backward over 8 x 1024 tokens, and
the LayerNorm + FFN1 + SwiGLU decode GEMV for 1 and 8 rows.  They are bandwidth-bound, so their rows give the bytes the kernel must move
over its time and the share of the data-sheet HBM3 bandwidth (3.35 TB/s).  Both dtypes.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=10).stdout.strip()
        name, power = [s.strip() for s in out.split(",")[:2]]
        return dict(gpu=name, power_limit=power)
    except Exception as e:          # the measurement still stands; say why the card is not named
        return dict(gpu=None, power_limit=None, gpu_info_error=repr(e))


def run_arm(dtype: str, steps: int, warmup: int) -> dict:
    """One arm in this process: the headline GPT-1.3B single-GPU configuration of bench.py with ``Engine.mix_precision.dtype = dtype``,
    ``warmup`` untimed steps, then ``steps`` steps between CUDA events.  Returns the JSON-ready result (ms/step, tokens/s, final loss, for
    float16 the loss scale after the timed steps and how many of them the dynamic scaler skipped, and the GPU name and power limit)."""
    import torch

    import bench
    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module

    assert torch.cuda.is_available(), "bench_precision.py needs a CUDA device"
    args = types.SimpleNamespace(model="gpt-1.3b", layout="auto", local_batch=8, micro_batch=0, recompute="auto", seq_len=1024, layers=0,
                                 step_overlap=-1, fused_tp=0, p2p=-1)
    env.init_process_group("gpu")
    torch.cuda.set_device(0)
    cfg, lay = bench.build_config(args, 1)
    cfg.Engine.mix_precision.dtype = dtype
    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    engine = EagerEngine(configs=cfg, module=build_module(cfg))
    dev = torch.device("cuda", 0)
    assert next(engine._module.model.parameters()).dtype == getattr(torch, dtype)
    seq, local, vocab = args.seq_len, lay["local"], cfg.Model.vocab_size
    gen = torch.Generator().manual_seed(1234)
    pool = []
    for _ in range(4):
        toks = torch.randint(0, vocab, (local, seq + 1), generator=gen, dtype=torch.int64)
        pos = torch.arange(seq, dtype=torch.int64).unsqueeze(0).expand(local, seq).contiguous()
        pool.append([t.to(dev) for t in (toks[:, :-1].contiguous(), pos, toks[:, 1:].contiguous(), torch.ones(local, seq))])
    scaler = engine._scaler if dtype == "float16" else None

    def device_step(i):
        loss = engine._fit_impl(list(pool[i % len(pool)]))
        engine._lr_scheduler.step(epoch=cfg.Global.global_batch_size)
        engine._optimizer.clear_grad()
        return loss

    for i in range(warmup):
        device_step(i)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    skipped = 0
    e0.record()
    for i in range(steps):
        loss = device_step(i)
        if scaler is not None and scaler.found_inf:           # the scaler has already read the flag to the host inside step()
            skipped += 1
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return dict(dtype=dtype, model="gpt-1.3b", steps=steps, warmup=warmup, ms_per_step=round(ms, 2),
                tokens_per_s=round(local * seq / ms * 1e3, 1), final_loss=round(float(loss), 4),
                loss_scale=scaler.get_scale() if scaler is not None else None, skipped_steps=skipped if scaler is not None else None, **gpu_info())


def _time_ms(fn, warmup=5, window_ms=500.0) -> float:
    """Mean device time of one call over a window of at least ``window_ms`` (at least 30 calls): a few milliseconds of back-to-back
    launches measure the clock state as much as the kernel."""
    import time

    import torch

    t0 = time.perf_counter()
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    iters = max(30, int(window_ms / max((time.perf_counter() - t0) * 1e3 / warmup, 1e-3)))
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


WIDE_FORMS = ("dgrad", "dgelu", "wgrad_bf16")   # the backward forms: timed at config 0 (128 x 128) and config 1 (128 x 256)
TILES = {0: "128x128", 1: "128x256"}


def run_kernels() -> list:
    """One JSON-ready row per kernel and dtype: the GEMM forms at GPT-1.3B's Linear shapes (the backward forms at both tiles), flash
    attention forward and backward, and the SwiGLU kernels, each with the GPU name and power limit."""
    import torch

    from paddlefleetx_b200.ops import _native

    lib = _native.require()
    tokens, h = 8 * 1024, 2048
    linears = {"qkv": (3 * h, h), "attn_out": (h, h), "ffn1": (4 * h, h), "ffn2": (h, 4 * h), "lm_head": (50304, h)}   # (out, in) features
    rows = []
    info = gpu_info()
    for dt in (torch.float16, torch.bfloat16):
        torch.manual_seed(0)
        for name, (n_out, n_in) in linears.items():
            x = torch.randn(tokens, n_in, device="cuda", dtype=dt)
            w = torch.randn(n_out, n_in, device="cuda", dtype=dt) * 0.02
            dy = torch.randn(tokens, n_out, device="cuda", dtype=dt)
            main_grad = torch.zeros(n_out, n_in, device="cuda")
            grad = torch.empty(n_out, n_in, device="cuda", dtype=dt)
            forms = {"fwd": lambda c: lib.gemm(x, w, None, None, True, True, 0, 0, c),                    # y = x W^T
                     "dgrad": lambda c: lib.gemm(dy, w, None, None, True, False, 0, 0, c),                # dx = dy W
                     "wgrad_bf16": lambda c: lib.gemm(dy, x, None, grad, False, False, 0, 0, c),          # grad = dy^T x (16-bit)
                     "wgrad_f32": lambda c: lib.gemm(dy, x, None, main_grad, False, False, 0, 1, c),      # main_grad = dy^T x
                     "wgrad_f32acc": lambda c: lib.gemm(dy, x, None, main_grad, False, False, 0, 2, c)}   # main_grad += dy^T x
            z = None
            if name == "ffn2":            # what the fused FFN's backward runs in place of the plain FFN2 dgrad: dz = (dy W2) * gelu'(z)
                z = torch.randn(tokens, n_in, device="cuda", dtype=dt)
                forms["dgelu"] = lambda c: lib.gemm_dgelu(dy, w, z, c)
            for form, fn in forms.items():
                configs = (0, 1) if form in WIDE_FORMS else (0,)
                times = {c: [] for c in configs}
                for _ in range(2 if len(configs) > 1 else 1):
                    for c in configs:
                        times[c].append(_time_ms(lambda: fn(c)))
                for c in configs:
                    ms = sum(times[c]) / len(times[c])
                    tflops = 2.0 * tokens * n_out * n_in / ms / 1e9
                    rows.append(dict(kernel=f"gemm_{name}_{form}", tile=TILES[c], dtype=str(dt).split(".")[-1], ms=round(ms, 4),
                                     ms_windows=[round(t, 4) for t in times[c]], tflops=round(tflops, 1),
                                     pct_of_989=round(100.0 * tflops / 989.0, 1), **info))
            del x, w, dy, main_grad, grad, z
        b, s, nh, d = 8, 1024, 16, 128
        mix = torch.randn(b, s, nh, 3, d, device="cuda", dtype=dt)
        q, k, v = mix.unbind(3)
        dmix = torch.empty_like(mix)
        dq, dk, dv = dmix.unbind(3)
        go = torch.randn(b, s, nh, d, device="cuda", dtype=dt)
        out, lse = lib.attention_fwd_v2(q, k, v, True, d ** -0.5, 0.0, 0)
        flops = 4.0 * b * nh * s * s * d * 0.5
        ms_f = _time_ms(lambda: lib.attention_fwd_v2(q, k, v, True, d ** -0.5, 0.0, 0))
        ms_b = _time_ms(lambda: lib.attention_bwd(q, k, v, out, go, lse, dq, dk, dv, True, d ** -0.5, 0.0, 0))
        rows.append(dict(kernel="attention_fwd_b8_s1024_h16_d128_causal", dtype=str(dt).split(".")[-1], ms=round(ms_f, 4),
                         tflops=round(flops / ms_f / 1e9, 1), **info))
        rows.append(dict(kernel="attention_bwd_b8_s1024_h16_d128_causal", dtype=str(dt).split(".")[-1], ms=round(ms_b, 4),
                         tflops=round(2.5 * flops / ms_b / 1e9, 1), **info))
        rows += _swiglu_rows(lib, dt, tokens, h, info)
    return rows


def _swiglu_rows(lib, dt, tokens: int, h: int, info: dict) -> list:
    """bias_swiglu forward / backward and the SwiGLU decode GEMV at GPT-1.3B SwiGLU shapes (F = 5632), as bytes moved / time."""
    import torch

    f, e = 5632, 2                                            # F, bytes per 16-bit element
    z = torch.randn(tokens, 2 * f, device="cuda", dtype=dt)
    bias = torch.randn(2 * f, device="cuda", dtype=dt) * 0.1
    dh = torch.randn(tokens, f, device="cuda", dtype=dt)
    w = torch.randn(2 * f, h, device="cuda", dtype=dt) * 0.02
    gamma, beta = torch.ones(h, device="cuda", dtype=dt), torch.zeros(h, device="cuda", dtype=dt)
    cases = [("bias_swiglu_fwd_8192x5632", lambda: lib.bias_swiglu_fwd(z, bias), e * (tokens * 3 * f + 2 * f)),   # z + bias in, h out
             ("bias_swiglu_bwd_8192x5632", lambda: lib.bias_swiglu_bwd(dh, z, bias), e * (tokens * 5 * f + 2 * f))]  # dh, z, bias in, dz out
    for m in (1, 8):
        x = torch.randn(m, h, device="cuda", dtype=dt)
        cases.append((f"gemv_ln_ffn1_swiglu_rows{m}_{2 * f}x{h}", lambda x=x: lib.gemv_fused(x, w, bias, gamma, beta, 1e-5, None, 2),
                      e * (2 * f * h + 2 * f + m * h + 2 * h + m * f)))
    rows = []
    for name, fn, nbytes in cases:
        ms = _time_ms(fn)
        rows.append(dict(kernel=name, dtype=str(dt).split(".")[-1], ms=round(ms, 4), gb_per_s=round(nbytes / ms / 1e6, 1),
                         pct_of_3350=round(100.0 * nbytes / ms / 1e6 / 3350.0, 1), **info))
    return rows


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=20)
    p.add_argument("--warmup", type=int, default=5)
    p.add_argument("--rounds", type=int, default=2, help="fp16 / bf16 pairs, alternated")
    p.add_argument("--kernels", action="store_true", help="time the GEMM and attention kernels instead of the training step")
    p.add_argument("--arm", default=None, choices=["float16", "bfloat16"], help=argparse.SUPPRESS)
    a = p.parse_args()
    if a.kernels:
        for row in run_kernels():
            print(json.dumps(row), flush=True)
        return
    if a.arm:
        print(json.dumps(run_arm(a.arm, a.steps, a.warmup)), flush=True)
        return
    for _ in range(a.rounds):
        for dtype in ("float16", "bfloat16"):
            res = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm", dtype, "--steps", str(a.steps), "--warmup", str(a.warmup)],
                                 capture_output=True, text=True)
            line = next((l for l in reversed(res.stdout.splitlines()) if l.startswith("{")), None)
            if res.returncode != 0 or line is None:
                sys.stderr.write(res.stdout[-4000:] + res.stderr[-4000:])
                raise SystemExit(f"{dtype} arm failed with exit code {res.returncode}")
            print(line, flush=True)


if __name__ == "__main__":
    main()
