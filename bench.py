"""Headline benchmark: GPT-3 pre-training throughput (tokens/s, whole job) on N H100s of one node (1.3B on one GPU by default).

    python bench.py --gpus 1 --steps 5 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...
    python bench.py --impl reference ...      # the unmodified reference (needs Paddle; reports `unavailable` otherwise)

Model/config = ``--model`` (GPT 1.3B: h=2048, L=24, heads=16; 6.7B: h=4096, L=32, heads=32), vocab=50304, seq=1024, bf16, synthetic tokens,
random-init weights, full step (forward + backward + clip + AdamW + LR step).  Timing: W untimed warm-up steps, then
exactly K steps bracketed by barrier + cuda synchronize, CUDA events on the compute stream, MAX over ranks.  One JSON
line on rank 0.  ``e2e`` repeats the measurement through the public ``EagerEngine.train_step`` API with per-step
pinned-host -> device input copies and a device -> host read of the loss.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

MODELS = {
    "gpt-6.7b": dict(cfg="pretrain_gpt_6.7B_single_card.yaml", hidden=4096, layers=32, heads=32),
    "gpt-1.3b": dict(cfg="pretrain_gpt_1.3B_single_card.yaml", hidden=2048, layers=24, heads=16),
    "gpt-345m": dict(cfg="pretrain_gpt_345M_single_card.yaml", hidden=1024, layers=24, heads=16),
}


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--impl", default="ours", choices=["ours", "reference", "torch_library"],
                   help="reference = the unmodified PaddleFleetX tree (needs Paddle); torch_library = a clearly-labelled stock-PyTorch arm "
                        "(cuBLAS + SDPA + torch fused AdamW + NCCL DDP) of the same model/config, NOT a substitute for the reference")
    p.add_argument("--model", default="gpt-1.3b", choices=sorted(MODELS),
                   help="gpt-1.3b trains on one 80 GB H100 (weights, fp32 master, AdamW state and gradients of gpt-6.7b alone need more than 100 GB: give it >= 2 GPUs)")
    p.add_argument("--dump-outputs", default=None, metavar="DIR",
                   help="after the timed steps write float32 DIR/<name>.npy: losses (every timed step), grad_norm (last timed step), params_sample (4096 "
                        "seeded positions of every parameter after it).  Inputs, weights and dropout are seeded; two runs agree to fp32 reduction order "
                        "(dQ tiles are added in no fixed order): on an H100 3e-5 relative in the loss, 1e-4 in the gradient norm")
    p.add_argument("--layout", default="auto", help="auto | sharding | mp2_pp2_sharding2 | dp | mpN")
    p.add_argument("--local-batch", type=int, default=8)
    p.add_argument("--micro-batch", type=int, default=0, help="0 = auto")
    p.add_argument("--recompute", default="auto", help="auto | none | full | full_attn | core_attn")
    p.add_argument("--seq-len", type=int, default=1024)
    p.add_argument("--no-e2e", action="store_true")
    p.add_argument("--p2p", type=int, default=-1, help="ZeRO traffic through our symmetric-memory kernels (NVLS multimem / peer stores): -1 auto (on for N > 1), 0 = NCCL, 1 on")
    p.add_argument("--fused-tp", type=int, default=0, help="1: all-gather->GEMM and GEMM->reduce-scatter as single kernels (TP+SP layouts)")
    p.add_argument("--step-overlap", type=int, default=-1, help="AdamW update issued per bucket on the side stream underneath the next forward pass: -1 auto (on), 0 off, 1 on")
    p.add_argument("--layers", type=int, default=0, help="debug only: override layer count (marks the result invalid)")
    p.add_argument("--named-layout", default="auto", help="at 8 GPUs also measure BASELINE config #2 (mp2 x pp2 x sharding2, fused TP kernels) in a child job after "
                                                         "the headline run and embed its line under \"named_layout\": auto (on at N = 8) | off")
    p.add_argument("--inner", action="store_true", help=argparse.SUPPRESS)
    p.add_argument("--profile", type=int, default=0, help="after the timed region, run this many extra steps under the CUPTI profiler and write "
                                                          "bench_trace_n<N>_rank0.json.gz into $PFX_BENCH_OUT, or a fresh temporary directory (kernel timeline; never part of the reported numbers)")
    return p.parse_args()


class ClockSampler:
    """nvidia-smi sampler running during the timed region (rank 0 only)."""

    FIELDS = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
              "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")

    def __init__(self, index: int = 0):
        self.index, self.rows, self._stop, self._t = index, [], threading.Event(), None

    def start(self):
        def run():
            while not self._stop.is_set():
                try:
                    out = subprocess.run(["nvidia-smi", f"--id={self.index}", f"--query-gpu={self.FIELDS}", "--format=csv,noheader,nounits"],
                                         capture_output=True, text=True, timeout=5).stdout.strip()
                    if out:
                        self.rows.append([x.strip() for x in out.split(",")])
                except (OSError, subprocess.SubprocessError):      # nvidia-smi missing / slow: the sample is simply skipped
                    pass
                self._stop.wait(0.2)
        self._t = threading.Thread(target=run, daemon=True)
        self._t.start()

    def stop(self) -> dict:
        self._stop.set()
        if self._t is not None:
            self._t.join(timeout=6)
        sm = sorted(int(float(r[0])) for r in self.rows if r and r[0].replace(".", "").isdigit())
        mx = max([int(float(r[1])) for r in self.rows if len(r) > 1 and r[1].replace(".", "").isdigit()] or [0])
        reasons = set()
        for r in self.rows:
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.strip().lower() == "active":
                    reasons.add(name)
        pw = sorted(float(r[2]) for r in self.rows if len(r) > 2 and r[2].replace(".", "").isdigit())
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx or None, "reasons": sorted(reasons), "samples": len(sm),
                "power_w": pw[len(pw) // 2] if pw else None}


def reference_arm(args):
    """Run the unmodified reference through its own tools/train.py.  It needs the Paddle framework; where that is not installed, say so in
    the result line."""
    why = None
    try:
        import paddle  # noqa: F401
    except Exception as e:  # noqa: BLE001
        why = f"the reference needs the Paddle framework and `import paddle` fails here ({type(e).__name__})"
    if why is None and not os.path.isdir(os.path.join(ROOT, "baseline", "_ref", "ppfleetx")):
        why = "baseline/_ref/ppfleetx not installed"
    if why is None:
        why = "paddle import unexpectedly succeeded but the reference launcher is not wired in this build"
    if int(os.environ.get("RANK", "0")) == 0:
        print(json.dumps({"impl": "reference", "unavailable": why}))
    return 0


_OUT_DIR = None


def _out_dir() -> str:
    """Where traces and child-job logs go: $PFX_BENCH_OUT, or ONE temporary directory per process whose path is printed on stderr — never the
    source tree, which may be read-only."""
    global _OUT_DIR
    if _OUT_DIR is None:
        _OUT_DIR = os.environ.get("PFX_BENCH_OUT")
        if _OUT_DIR:
            os.makedirs(_OUT_DIR, exist_ok=True)
        else:
            import tempfile

            _OUT_DIR = tempfile.mkdtemp(prefix="pfx_bench_")
        print(f"bench.py: traces and logs in {_OUT_DIR}", file=sys.stderr)
    return _OUT_DIR


def _profile_steps(args, device_step, barrier, rank, world):
    """Kernel timeline of a few steps (rank 0): name, stream, start, duration of every kernel — compact json.gz for offline analysis."""
    import gzip

    import torch

    barrier()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for i in range(args.profile):
            device_step(i)
        torch.cuda.synchronize()
    barrier()
    if rank != 0:
        return
    out_dir = _out_dir()
    tmp = os.path.join(out_dir, f"_trace_tmp_{os.getpid()}.json")
    prof.export_chrome_trace(tmp)
    with open(tmp) as f:
        trace = json.load(f)
    os.remove(tmp)
    rows = [[e.get("name", "")[:120], int(e.get("args", {}).get("stream", -1)), float(e["ts"]), float(e.get("dur", 0.0))]
            for e in trace.get("traceEvents", []) if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset") and "ts" in e]
    rows.sort(key=lambda r: r[2])
    with gzip.open(os.path.join(out_dir, f"bench_trace_n{world}_rank0.json.gz"), "wt") as f:
        json.dump({"steps": args.profile, "model": args.model, "n_gpus": world, "columns": ["name", "stream", "ts_us", "dur_us"], "kernels": rows}, f)


def child_job_env(parent_env, port_offset: int = 17) -> dict:
    """Environment of a child job started by every rank of a torchrun job: same ranks, its own rendezvous port.  Under torchrun the env://
    rendezvous connects to the elastic AGENT's store instead of creating one; nobody serves the child's port, so unless the agent-store
    marker is removed every child rank waits for a store that never comes up."""
    env = dict(parent_env)
    env["MASTER_PORT"] = str(int(env.get("MASTER_PORT", "29500")) + port_offset)
    env.pop("TORCHELASTIC_USE_AGENT_STORE", None)
    env.pop("TORCHELASTIC_RUN_ID", None)
    return env


def _run_named_layout(args, rank):
    """BASELINE config #2 (GPT-6.7B, mp2 x pp2 x sharding2) as a child job on the same 8 GPUs: one child per rank, its own rendezvous port, a hard
    timeout; returns the child's JSON line (rank 0) or a dict with the failure reason.  Never raises: the headline line must survive."""
    env = child_job_env(os.environ)
    forced = os.environ.get("PFX_NAMED_LAYOUT_FORCE")      # test hook: exercise the child-job path at another world size / layout (e.g. mp2 on 2 GPUs)
    cmd = [sys.executable, os.path.abspath(__file__), "--gpus", env.get("WORLD_SIZE", "8"), "--layout", forced or "mp2_pp2_sharding2", "--fused-tp", "1", "--steps", str(max(args.steps // 2, 3)),
           "--warmup", "3", "--no-e2e", "--inner", "--model", args.model, "--seq-len", str(args.seq_len), "--local-batch", str(args.local_batch)]
    if args.layers:
        cmd += ["--layers", str(args.layers)]
    log_path = os.path.join(_out_dir(), f"named_layout_child_rank{rank}.log")
    limit = float(os.environ.get("PFX_NAMED_LAYOUT_TIMEOUT", "300"))

    def tail():
        try:
            with open(log_path, "r", errors="replace") as f:
                return f.read()[-600:]
        except OSError:
            return ""

    try:
        with open(log_path, "w") as log:
            p = subprocess.Popen(cmd, env=env, stdout=subprocess.PIPE, stderr=log, text=True)
            try:
                out, _ = p.communicate(timeout=limit)
            except subprocess.TimeoutExpired:
                p.kill()                      # this exact child, by handle
                p.communicate()
                return {"unavailable": f"child job timed out after {limit:.0f} s", "stderr_tail": tail()} if rank == 0 else None
        if rank != 0:
            return None
        for line in reversed(out.strip().splitlines()):
            if line.startswith("{"):
                return json.loads(line)
        return {"unavailable": f"child exited {p.returncode} without a result", "stderr_tail": tail()}
    except Exception as e:  # noqa: BLE001
        return {"unavailable": repr(e)[:300]} if rank == 0 else None


def build_config(args, world: int):
    from paddlefleetx_b200.utils import config as C

    spec = MODELS[args.model]
    layout = args.layout
    if layout == "auto":
        layout = "sharding" if world > 1 else "single"
    mp = pp = 1
    sharding, dp = world, 1
    stage = 1
    if layout == "mp2_pp2_sharding2":
        assert world == 8, "mp2_pp2_sharding2 needs 8 GPUs"
        mp, pp, sharding = 2, 2, 2
    elif layout == "dp":
        sharding, dp = 1, world
    elif layout.startswith("mp"):            # "mp2", "mp4", ...: tensor + sequence parallel, rest of the world is ZeRO-1 sharding
        mp = int(layout[2:])
        assert world % mp == 0
        sharding = world // mp
    local = args.local_batch * mp * pp          # per data-rank batch: per-GPU work stays fixed (weak scaling)
    micro = args.micro_batch or (local if pp == 1 else max(args.local_batch // 2, 1))
    recompute = args.recompute
    if recompute == "auto":
        recompute = "none"
    ov = [
        f"Global.local_batch_size={local}", f"Global.micro_batch_size={micro}", "Global.global_batch_size=None",
        f"Distributed.dp_degree={dp}", f"Distributed.mp_degree={mp}", f"Distributed.pp_degree={pp}",
        f"Distributed.sharding.sharding_degree={sharding}", f"Distributed.sharding.sharding_stage={stage}",
        f"Distributed.sharding.reduce_overlap={world > 1}", f"Distributed.sharding.broadcast_overlap={world > 1}", f"Distributed.sharding.use_p2p={bool(args.p2p) if args.p2p >= 0 else world > 1}",
        f"Model.use_recompute={recompute != 'none'}", f"Model.recompute_granularity={'full' if recompute == 'none' else recompute}",
        f"Model.sequence_parallel={mp > 1}",
        "Engine.max_steps=1000000", "Engine.eval_freq=-1", "Engine.eval_iters=0", "Engine.logging_freq=1000000",
        "Engine.save_load.save_steps=-1", "Engine.mix_precision.dtype=bfloat16",
        f"Model.max_position_embeddings={args.seq_len}",
    ]
    if args.layers:
        ov.append(f"Model.num_layers={args.layers}")
    if args.step_overlap != 0:
        ov.append("Optimizer.step_overlap=True")
    if args.fused_tp:
        ov.append("Fused.tp_comm=True")
    cfg_path = os.path.join(ROOT, "paddlefleetx_b200", "configs", "nlp", "gpt", spec["cfg"])
    cfg = C.get_config(cfg_path, overrides=ov, show=False, nranks=world)
    # synthetic data of the named shape
    for mode in ("Train", "Eval"):
        cfg.Data[mode]["dataset"] = C.AttrDict(name="SyntheticGPTDataset", max_seq_len=args.seq_len, vocab_size=cfg.Model.vocab_size)
        cfg.Data[mode]["loader"] = C.AttrDict(num_workers=0, collate_fn="gpt_collate_fn")
    return cfg, dict(layout=layout, mp=mp, pp=pp, sharding=sharding, dp=dp, recompute=recompute, local=local, micro=micro)


def main():
    """Run one arm of the headline benchmark (``--impl``: ours, ``reference`` or ``torch_library``) on this rank and, on rank 0, print the ONE
    JSON result line: W untimed warm-up steps, exactly K device-timed steps between barriers (max over ranks), clocks sampled
    during the timed region, the end-to-end arm through the public engine API, launch and exposed-communication counts."""
    args = parse()
    if args.dump_outputs and args.impl != "ours":
        raise SystemExit("--dump-outputs is implemented for --impl ours only")
    if args.impl == "reference":
        return reference_arm(args)
    if args.impl == "torch_library":
        from tools.torch_library_baseline import run as run_library

        return run_library(args, MODELS[args.model], ClockSampler)
    import torch
    import torch.distributed as dist

    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module
    from paddlefleetx_b200.ops import functional as OF

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    assert world == args.gpus, f"--gpus {args.gpus} but WORLD_SIZE={world}; launch with torchrun for N>1"
    assert torch.cuda.is_available(), "bench.py needs a CUDA device"
    env.init_process_group("gpu")
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    cfg, lay = build_config(args, world)
    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    module = build_module(cfg)
    engine = EagerEngine(configs=cfg, module=module)
    dev = torch.device("cuda", torch.cuda.current_device())

    seq, local = args.seq_len, lay["local"]
    vocab = cfg.Model.vocab_size
    data_rank, data_world = env.get_data_world_rank(), env.get_data_world_size()
    global_batch = cfg.Global.global_batch_size
    gen = torch.Generator().manual_seed(1234 + data_rank)

    def host_batch():
        toks = torch.randint(0, vocab, (local, seq + 1), generator=gen, dtype=torch.int64)
        pos = torch.arange(seq, dtype=torch.int64).unsqueeze(0).expand(local, seq).contiguous()
        mask = torch.ones(local, seq, dtype=torch.float32)
        return [t.pin_memory() for t in (toks[:, :-1].contiguous(), pos, toks[:, 1:].contiguous(), mask)]

    pool = [host_batch() for _ in range(4)]
    dev_pool = [[t.to(dev) for t in b] for b in pool]

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def device_step(i):
        loss = engine._fit_impl([t for t in dev_pool[i % len(dev_pool)]])
        engine._lr_scheduler.step(epoch=global_batch)
        engine._optimizer.clear_grad()
        return loss

    # ---- warm-up
    for i in range(args.warmup):
        device_step(i)
    barrier()

    # ---- timed region (device inputs, no host sync inside)
    sampler = ClockSampler(int(os.environ.get("LOCAL_RANK", "0"))) if rank == 0 else None
    if sampler:
        sampler.start()
    OF.reset_launch_count()
    opt = engine._optimizer
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    barrier()
    if hasattr(opt, "comm_meter_start"):
        opt.comm_meter_start()
    e0.record()
    marks, step_losses = [], []
    for i in range(args.steps):
        loss = device_step(i)
        step_losses.append(loss.detach())
        ev = torch.cuda.Event(enable_timing=True)      # per-step marks: the spread inside the run (power-capped parts wander by several %)
        ev.record()
        marks.append(ev)
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    per_step = sorted(a.elapsed_time(b) for a, b in zip([e0] + marks[:-1], marks))
    launches = OF.native_launch_count()
    exposed = opt.comm_meter_read() / args.steps if hasattr(opt, "comm_meter_read") else None
    if exposed is not None and world > 1:
        te = torch.tensor([exposed], device=dev)
        dist.all_reduce(te, op=dist.ReduceOp.MAX)
        exposed = float(te.item())
    t = torch.tensor([ms], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_total = float(t.item())
    final_loss = float(loss)
    if args.dump_outputs and rank == 0:
        import numpy as np

        os.makedirs(args.dump_outputs, exist_ok=True)
        losses = torch.stack([l.float().reshape(()) for l in step_losses]).cpu().numpy().astype(np.float32)
        np.save(os.path.join(args.dump_outputs, "losses.npy"), losses)
        if hasattr(opt, "grad_norm"):
            np.save(os.path.join(args.dump_outputs, "grad_norm.npy"), np.asarray([opt.grad_norm()], dtype=np.float32))
        pick = torch.Generator().manual_seed(4321)
        sample = []
        for _, p in sorted(engine._module.model.named_parameters(), key=lambda kv: kv[0]):
            idx = torch.randint(0, p.numel(), (min(4096, p.numel()),), generator=pick)
            sample.append(p.detach().reshape(-1)[idx.to(p.device)].float().cpu())
        np.save(os.path.join(args.dump_outputs, "params_sample.npy"), torch.cat(sample).numpy())

    # ---- end-to-end through the public API: pinned host inputs copied every step + loss read back every step
    e2e = None
    if not args.no_e2e:
        barrier()
        f0, f1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        f0.record()
        for i in range(args.steps):
            l = engine.train_step(pool[i % len(pool)])
            _ = l.item()
        f1.record()
        barrier()
        t2 = torch.tensor([f0.elapsed_time(f1)], device=dev)
        if world > 1:
            dist.all_reduce(t2, op=dist.ReduceOp.MAX)
        h2d = sum(x.numel() * x.element_size() for x in pool[0])
        e2e = {"value": global_batch * seq * args.steps / (float(t2.item()) / 1e3), "unit": "tokens/s",
               "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4}
    clocks = sampler.stop() if sampler else None
    step_spread = {"median_ms": per_step[len(per_step) // 2], "min_ms": per_step[0], "max_ms": per_step[-1]} if per_step else None
    energy = None
    if clocks and clocks.get("power_w"):
        # energy-normalised throughput (rank 0's GPU): what a power-capped part can be compared on from box to box
        energy = {"power_w_median": clocks["power_w"], "tokens_per_joule_per_gpu": (global_batch * seq / world) / (ms_total / args.steps / 1e3) / clocks["power_w"]}
    if args.profile > 0:
        _profile_steps(args, device_step, barrier, rank, world)

    symm = getattr(opt, "_symm", None)
    if world == 1:
        collective = "none (1 GPU); exposed_comm = compute-stream waits on the side-stream AdamW update"
    elif getattr(opt, "use_p2p", False):
        collective = ("own kernels over symmetric memory: " + ("NVLS multimem.ld_reduce reduce-scatter + AdamW with multimem.st broadcast"
                      if (getattr(symm, "multicast", False) and any(g.meta.get("mc_grads") for g in opt.groups)) else "unicast peer pull reduce-scatter + AdamW with peer-store broadcast")
                      + "; NCCL only for the scalar grad-norm all-reduce" + (" and TP/PP traffic" if lay["mp"] > 1 or lay["pp"] > 1 else ""))
    else:
        collective = "NCCL"
    opt_overlapped = bool(getattr(opt, "step_overlap", False))
    named = None
    if (world == 8 or os.environ.get("PFX_NAMED_LAYOUT_FORCE")) and args.named_layout != "off" and args.layout == "auto" and not args.inner and (not args.layers or os.environ.get("PFX_NAMED_LAYOUT_FORCE")):
        # release this job's device memory, then every rank starts the same rank of a child job (fresh process groups, fresh topology)
        del loss
        engine = module = opt = dev_pool = None
        import gc

        gc.collect()
        torch.cuda.empty_cache()
        named = _run_named_layout(args, rank)
    if rank == 0:
        tokens = global_batch * seq * args.steps
        par = {"single": "single", "sharding": f"sharding{world}_stage1", "dp": f"dp{world}",
               "mp2_pp2_sharding2": "mp2_pp2_sharding2"}.get(lay["layout"])
        if par is None:
            par = f"mp{lay['mp']}_sp_sharding{lay['sharding']}_stage1" + ("_fusedtp" if args.fused_tp else "")
        out = {
            "metric": f"GPT-3 {args.model.split('-')[1].upper()} pre-training tokens/sec (whole job, device-timed, max over ranks)",
            "value": tokens / (ms_total / 1e3), "unit": "tokens/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
            "ms_per_step": ms_total / args.steps, "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
            "dtype": "bf16", "data": "synthetic (uniform random tokens, random-init weights)",
            "config": {"model": args.model if not args.layers else f"{args.model}-DEBUG-{args.layers}layers(INVALID)",
                       "global_batch": global_batch, "seq_len": seq, "parallelism": par, "local_batch": lay["local"],
                       "micro_batch": lay["micro"], "recompute": lay["recompute"], "dropout": cfg.Model.hidden_dropout_prob,
                       "optimizer": "FusedAdamW fp32 master + clip" + (" (update overlapped with the next forward)" if opt_overlapped else ""), "l2": "working set per step >> 50 MB L2, no explicit flush"},
            "gpu_launches": launches, "clocks": clocks, "e2e": e2e, "final_loss": final_loss,
            "collective": collective, "exposed_comm_ms_per_step": exposed, "step_spread": step_spread, "energy": energy, "named_layout": named,
            "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30,
        }
        print(json.dumps(out))
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


if __name__ == "__main__":
    sys.exit(main())
