"""Throughput of the other BASELINE.json workloads (bench.py is reserved for the GPT-3 6.7B headline):

    moe    GPT-MoE 8 x 1.3B, expert parallel over the data-parallel ranks, gshard top-2, 2 experts / rank   (tokens/s)
    vit    ViT-L/16 384^2 fine-tune, ZeRO stage 2 over all ranks, 32 images / GPU                            (images/s)
    ernie  ERNIE 10B-class encoder, mp x ZeRO stage 3                                                        (tokens/s)
    gpt-1.3b    GPT 1.3B (tanh-GELU FFN, 4h), data parallel, 8 x 1024 tokens / GPU                          (tokens/s)
    gpt-swiglu  the same model with the SwiGLU FFN (Model.ffn_activation: swiglu, F = 5632)                  (tokens/s)
    gpt-1.3b-docs  GPT 1.3B on rows packed from documents of 128 to 383 tokens (seeded lengths, mean 256),
                intra-document attention (Model.reset_attention_mask)                                          (tokens/s)

Synthetic data of the named shape, random-init weights, bf16.  Same contract as bench.py: W warm-up steps, K steps timed with CUDA
events between barriers, max over ranks, nvidia-smi clocks / throttle reasons sampled during the timed region, the exposed-
communication meter, the per-step host->device / device->host bytes (every step copies its batch from pinned memory and the harness reads
the loss back), one JSON line on rank 0.

    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/bench_workloads.py --workload moe --gpus 8 [--p2p 1]
"""
import argparse
import json
import os
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

CFG = os.path.join(ROOT, "paddlefleetx_b200", "configs")


def parse():
    p = argparse.ArgumentParser()
    p.add_argument("--workload", required=True, choices=["moe", "vit", "ernie", "gpt-1.3b", "gpt-swiglu", "gpt-1.3b-docs"])
    p.add_argument("--gpus", type=int, default=1)
    p.add_argument("--steps", type=int, default=5)
    p.add_argument("--warmup", type=int, default=3)
    p.add_argument("--p2p", type=int, default=0, help="moe: peer-memory dispatch/combine kernels; vit: peer-memory ZeRO kernels")
    p.add_argument("--local-batch", type=int, default=0)
    p.add_argument("--layers", type=int, default=0, help="debug: override depth (marks the result invalid)")
    p.add_argument("--mp", type=int, default=0, help="ernie: tensor-parallel degree (default 4 on 8 GPUs, else min(world, 2))")
    p.add_argument("--fp8", type=int, default=0, help="ernie: fp8 forward GEMMs in the tensor-parallel linears")
    p.add_argument("--sp", type=int, default=0, help="ernie: Megatron sequence parallelism over the tensor-parallel group")
    p.add_argument("--fused-tp", type=int, default=0, help="ernie (with --sp 1): all-gather->GEMM / GEMM->reduce-scatter as single peer-memory kernels")
    return p.parse_args()


def main():
    """Build the selected workload through the public engine, run warm-up + timed steps under the bench.py timing rules and print one JSON line."""
    a = parse()
    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module
    from paddlefleetx_b200.ops import functional as OF
    from paddlefleetx_b200.utils import config as C

    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    assert world == a.gpus
    env.init_process_group("gpu")
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dev = torch.device("cuda", torch.cuda.current_device())
    common = ["Engine.max_steps=1000000", "Engine.eval_freq=-1", "Engine.logging_freq=1000000", "Engine.save_load.save_steps=-1",
              "Engine.mix_precision.enable=True", "Engine.mix_precision.dtype=bfloat16", "Global.global_batch_size=None"]
    if a.workload in ("gpt-1.3b", "gpt-swiglu", "gpt-1.3b-docs"):
        local = a.local_batch or 8
        swiglu = a.workload == "gpt-swiglu"
        docs = a.workload == "gpt-1.3b-docs"
        ov = common + [f"Global.local_batch_size={local}", f"Global.micro_batch_size={local}", f"Distributed.dp_degree={world}",
                       "Distributed.mp_degree=1", "Distributed.pp_degree=1", "Distributed.sharding.sharding_degree=1"]
        if a.layers:
            ov.append(f"Model.num_layers={a.layers}")
        recipe = ("pretrain_gpt_1.3B_swiglu_single_card.yaml" if swiglu else
                  "pretrain_gpt_1.3B_packed_docs_single_card.yaml" if docs else "pretrain_gpt_1.3B_single_card.yaml")
        cfg = C.get_config(os.path.join(CFG, "nlp/gpt", recipe), ov, nranks=world)
        seq = 1024
        cfg.Data.Train["dataset"] = C.AttrDict(name="SyntheticGPTDataset", max_seq_len=seq, vocab_size=cfg.Model.vocab_size)
        cfg.Data.Train["loader"] = C.AttrDict(num_workers=0, collate_fn="gpt_collate_fn")
        unit, per_step = "tokens/s", local * seq * world
        from paddlefleetx_b200.models.language_model.gpt.model import swiglu_ffn_size

        h = cfg.Model.hidden_size
        ffn = cfg.Model.get("ffn_hidden_size") or (swiglu_ffn_size(h) if swiglu else 4 * h)
        name = f"GPT 1.3B ({'SwiGLU' if swiglu else 'GELU'} FFN, F = {ffn}), dp{world}, {local} x {seq} tokens/GPU, recompute {cfg.Model.get('use_recompute')}"
        if docs:
            from paddlefleetx_b200.data.dataset.gpt_dataset import SyntheticGPTDataset

            name += ", packed documents of 128-383 tokens, reset_attention_mask"
            doc_set = SyntheticGPTDataset(max_seq_len=seq, vocab_size=cfg.Model.vocab_size, reset_position_ids=True, document_length=256)

        def make_batch(g):
            t = torch.randint(0, cfg.Model.vocab_size, (local, seq + 1), generator=g)
            if docs:
                pos = torch.stack([torch.from_numpy(doc_set[int(torch.randint(0, 1 << 20, (1,), generator=g))][1]) for _ in range(local)])
            else:
                pos = torch.arange(seq).unsqueeze(0).expand(local, seq).contiguous()
            return [t[:, :-1].contiguous(), pos, t[:, 1:].contiguous(), torch.ones(local, seq)]
    elif a.workload == "moe":
        local = a.local_batch or 8
        ov = common + [f"Global.local_batch_size={local}", f"Global.micro_batch_size={local}", f"Distributed.dp_degree={world}",
                       "Distributed.mp_degree=1", "Distributed.pp_degree=1", "Distributed.sharding.sharding_degree=1",
                       f"Model.moe_configs.fused_p2p={bool(a.p2p)}", "Model.use_recompute=False"]
        if a.layers:
            ov.append(f"Model.num_layers={a.layers}")
        cfg = C.get_config(os.path.join(CFG, "nlp/moe/pretrain_moe_1.3B_dp8.yaml"), ov, nranks=world)
        seq = 1024
        cfg.Data.Train["dataset"] = C.AttrDict(name="SyntheticGPTDataset", max_seq_len=seq, vocab_size=cfg.Model.vocab_size)
        cfg.Data.Train["loader"] = C.AttrDict(num_workers=0, collate_fn="gpt_collate_fn")
        unit, per_step = "tokens/s", local * seq * world
        name = f"GPT-MoE {world}x1.3B (2 experts/rank, gshard top-2), expert parallel over dp{world}, {'peer-memory' if a.p2p else 'NCCL all-to-all'} dispatch"

        def make_batch(g):
            t = torch.randint(0, cfg.Model.vocab_size, (local, seq + 1), generator=g)
            pos = torch.arange(seq).unsqueeze(0).expand(local, seq).contiguous()
            return [t[:, :-1].contiguous(), pos, t[:, 1:].contiguous(), torch.ones(local, seq)]
    elif a.workload == "vit":
        local = a.local_batch or 32
        ov = common + [f"Global.local_batch_size={local}", f"Global.micro_batch_size={local}", "Distributed.dp_degree=1",
                       f"Distributed.sharding.sharding_degree={world}", "Distributed.sharding.sharding_stage=2",
                       f"Distributed.sharding.use_p2p={bool(a.p2p)}"]
        if a.layers:
            ov.append(f"Model.model.depth={a.layers}")
        cfg = C.get_config(os.path.join(CFG, "vis/vit/ViT_large_patch16_384_ft_in1k_dp8_sharding_stage2.yaml"), ov, nranks=world)
        unit, per_step = "images/s", local * world
        name = f"ViT-L/16 384^2 fine-tune, ZeRO stage 2 over {world} GPUs, {local} images/GPU"

        def make_batch(g):
            return [torch.randn(local, 3, 384, 384, generator=g), torch.randint(0, 1000, (local,), generator=g)]
    else:
        mp = a.mp or (4 if world == 8 else min(world, 2))
        sh = world // mp
        local = a.local_batch or 8
        seq = 512
        ov = common + [f"Global.local_batch_size={local}", f"Global.micro_batch_size={local}", "Distributed.dp_degree=1", f"Distributed.mp_degree={mp}",
                       f"Distributed.sharding.sharding_degree={sh}", "Distributed.sharding.sharding_stage=3", f"Fused.fp8_tp_gemm={bool(a.fp8)}",
                       f"Fused.tp_comm={bool(a.fused_tp and a.sp)}", f"Model.sequence_parallel={bool(a.sp)}", f"Data.Train.dataset.max_seq_length={seq}"]
        if a.layers:
            ov.append(f"Model.num_hidden_layers={a.layers}")
        cfg = C.get_config(os.path.join(CFG, "nlp/ernie/pretrain_ernie_10B_mp4_stage3_fp8.yaml"), ov, nranks=world)
        unit, per_step = "tokens/s", local * seq * sh
        name = (f"ERNIE 10B-class (h4096 L{cfg.Model.num_hidden_layers}), mp{mp} x ZeRO-3 sharding{sh}, {'fp8' if a.fp8 else 'bf16'} TP GEMMs"
                + (", sequence parallel" if a.sp else "") + (" with fused GEMM+collective kernels" if (a.fused_tp and a.sp) else ""))
        vocab = cfg.Model.vocab_size
        n_mask = 76

        def make_batch(g):
            ids = torch.randint(4, vocab, (local, seq), generator=g)
            seg = torch.zeros(local, seq, dtype=torch.long)
            mask = torch.ones(local, seq, dtype=torch.float32)
            pos = torch.stack([torch.randperm(seq, generator=g)[:n_mask].sort().values + i * seq for i in range(local)]).reshape(-1)
            labels = torch.randint(4, vocab, (local * n_mask,), generator=g)
            return [ids, seg, mask, pos, labels, torch.randint(0, 2, (local,), generator=g)]

    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    module = build_module(cfg)
    engine = EagerEngine(configs=cfg, module=module)
    g = torch.Generator().manual_seed(99 + env.get_data_world_rank())
    pool = [[t.pin_memory() for t in make_batch(g)] for _ in range(3)]

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    from bench import ClockSampler          # the headline bench's nvidia-smi sampler (repo root)

    for i in range(a.warmup):
        engine.train_step(pool[i % len(pool)])
    barrier()
    OF.reset_launch_count()
    opt = getattr(engine, "_optimizer", None)
    if hasattr(opt, "comm_meter_start"):
        opt.comm_meter_start()
    sampler = ClockSampler(int(os.environ.get("LOCAL_RANK", "0"))) if rank == 0 else None
    if sampler:
        sampler.start()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    loss_host = 0.0
    for i in range(a.steps):
        loss = engine.train_step(pool[i % len(pool)])
        loss_host = float(loss)             # device -> host read of the step's result, inside the timed region
    e1.record()
    barrier()
    clocks = sampler.stop() if sampler else None
    exposed = opt.comm_meter_read() / a.steps if hasattr(opt, "comm_meter_read") else None
    h2d = sum(t.numel() * t.element_size() for t in pool[0])
    t = torch.tensor([e0.elapsed_time(e1)], device=dev)
    if world > 1:
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms = float(t)
    if rank == 0:
        out = {"metric": name, "value": per_step * a.steps / (ms / 1e3), "unit": unit, "n_gpus": world, "steps": a.steps, "warmup": a.warmup,
               "ms_per_step": ms / a.steps, "higher_is_better": True, "scaling": "weak", "dtype": "bf16",
               "data": "synthetic, random-init weights; the timed region includes the pinned host->device copy of every batch and the loss read-back",
               "e2e": {"value": per_step * a.steps / (ms / 1e3), "unit": unit, "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": 4,
                       "note": "value IS end to end: engine.train_step(pinned host batch) -> float(loss) every step"},
               "clocks": clocks, "exposed_comm_ms_per_step": exposed,
               "final_loss": loss_host, "gpu_launches": OF.native_launch_count(), "peak_mem_gb": torch.cuda.max_memory_allocated() / 2 ** 30,
               "valid": not a.layers}
        print(json.dumps(out), flush=True)
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        tag = f"{a.workload}_{world}gpu" + ("_p2p" if a.p2p else "") + ("_fp8" if a.fp8 else "") + ("_sp" if a.sp else "") + ("_fusedtp" if a.fused_tp and a.sp else "")
        with open(os.path.join(ROOT, "gpurun_out", f"workload_{tag}.json"), "w") as f:
            json.dump(out, f)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
