"""Multi-GPU checks of the peer-memory kernels (run with torchrun, one rank per GPU):

    python -m torch.distributed.run --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/gpu_multi_selftest.py
"""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch
import torch.distributed as dist


def relerr(a, b):
    a, b = a.float(), b.float()
    return float((a - b).norm() / (b.norm() + 1e-12))


def timed(fn, iters=10, warmup=3):
    for _ in range(warmup):
        fn()
    dist.barrier(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    dist.barrier(); torch.cuda.synchronize()
    t = torch.tensor([e0.elapsed_time(e1) / iters], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


def main():
    """Run every multi-GPU check on this rank and print one ``RESULT {json}`` line per check (rank 0); exit status 1 if any check failed."""
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
    dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    from paddlefleetx_b200.ops import _native
    from paddlefleetx_b200.parallel import fused_tp
    from paddlefleetx_b200.parallel.symmetric_memory import SymmetricAllocator
    from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

    lib = _native.require()
    hcg = HybridCommunicateGroup(mp=world)
    grp = hcg.get_model_parallel_group()
    res = {}

    def report(name, **kw):
        res[name] = kw
        if rank == 0:
            print("RESULT " + json.dumps(dict(check=name, **kw)), flush=True)

    only = set(filter(None, os.environ.get("PFX_MULTI_ONLY", "").split(",")))

    def section(name):
        return not only or name in only

    # ---------------------------------------------------------------- cuMem-VMM symmetric memory + NVLS (multimem) kernels
    if section("nvls"):
        try:
            nvls_section(lib, grp, rank, world, report)
        except Exception as e:  # noqa: BLE001
            import traceback
            report("nvls_section", ok=False, error=repr(e), tb=traceback.format_exc()[-1500:])
    if only and only <= {"nvls"}:
        dist.barrier()
        finish(res, rank, world)
        return

    # ---------------------------------------------------------------- barrier + raw P2P
    sm = SymmetricAllocator(grp)
    n = 1 << 24
    buf = sm.alloc_tensor(n * world, torch.bfloat16)
    torch.manual_seed(100 + rank)
    local = (torch.randn(n * world, device="cuda") * 0.1).bfloat16()
    buf.copy_(local)
    torch.cuda.synchronize(); sm.barrier()
    ptrs = sm.peer_ptrs(buf)
    # reference reduce-scatter via NCCL
    ref = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    dist.reduce_scatter_tensor(ref, local.clone())
    out = torch.empty(n, dtype=torch.float32, device="cuda")
    lib.p2p_reduce_scatter(ptrs, out, rank, 1, False, 1.0, 128)
    torch.cuda.synchronize(); sm.barrier()
    report("p2p_reduce_scatter", err=relerr(out, ref), ok=relerr(out, ref) < 1e-2)

    def rs_p2p():
        sm.barrier(); lib.p2p_reduce_scatter(ptrs, out, rank, 1, False, 1.0, 128); sm.barrier()
    t_p2p = timed(rs_p2p)
    scratch = local.clone()
    t_nccl = timed(lambda: dist.reduce_scatter_tensor(ref, scratch))
    moved = n * (world - 1) * 2
    report("p2p_reduce_scatter_perf", ms=t_p2p, nccl_ms=t_nccl, gbs_in=moved / t_p2p / 1e6, nccl_gbs_in=moved / t_nccl / 1e6, ok=True)

    # push all-gather
    shard = (torch.arange(n, device="cuda") % 251 + rank).bfloat16()
    sm.barrier()
    lib.p2p_all_gather(ptrs, shard, rank, 32)
    torch.cuda.synchronize(); sm.barrier()
    ok = True
    for r in range(world):
        want = (torch.arange(n, device="cuda") % 251 + r).bfloat16()
        ok &= bool(torch.equal(buf[r * n:(r + 1) * n], want))
    report("p2p_all_gather", ok=ok)
    t_ag = timed(lambda: (sm.barrier(), lib.p2p_all_gather(ptrs, shard, rank, 32), sm.barrier()))
    gath = torch.empty(n * world, dtype=torch.bfloat16, device="cuda")
    t_ag_nccl = timed(lambda: dist.all_gather_into_tensor(gath, shard))
    report("p2p_all_gather_perf", ms=t_ag, nccl_ms=t_ag_nccl, gbs_out=moved / t_ag / 1e6, nccl_gbs=moved / t_ag_nccl / 1e6, ok=True)

    # ---------------------------------------------------------------- fused GEMM -> reduce-scatter
    torch.manual_seed(7)
    M, N, K = 8192, 4096, 4096 // world * world
    kl = K // world
    A = (torch.randn(M, K, device="cuda") * 0.05).bfloat16()
    W = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    a_loc, w_loc = A[:, rank * kl:(rank + 1) * kl].contiguous(), W[:, rank * kl:(rank + 1) * kl].contiguous()
    full = A.float() @ W.float().t()
    want = full[rank * (M // world):(rank + 1) * (M // world)]
    got = fused_tp.gemm_rs(a_loc, w_loc, grp)
    torch.cuda.synchronize()
    report("gemm_rs", err=relerr(got, want), ok=relerr(got, want) < 2e-2)
    t_f = timed(lambda: fused_tp.gemm_rs(a_loc, w_loc, grp))
    part = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    o2 = torch.empty(M // world, N, dtype=torch.bfloat16, device="cuda")

    def baseline_rs():
        torch.matmul(a_loc, w_loc.t(), out=part)
        dist.reduce_scatter_tensor(o2, part)
    t_b = timed(baseline_rs)
    t_g = timed(lambda: torch.matmul(a_loc, w_loc.t(), out=part))
    report("gemm_rs_perf", fused_ms=t_f, cublas_plus_nccl_ms=t_b, gemm_only_ms=t_g, ok=True)

    # ---------------------------------------------------------------- fused all-gather -> GEMM
    rows = M // world
    X = (torch.randn(M, K, device="cuda") * 0.05).bfloat16()        # same on all ranks (same seed)
    Wc = (torch.randn(N // world * world, K, device="cuda") * 0.05).bfloat16()
    nl = Wc.shape[0] // world
    w_col = Wc[rank * nl:(rank + 1) * nl].contiguous()
    x_shard = X[rank * rows:(rank + 1) * rows].contiguous()
    y, gathered = fused_tp.ag_gemm(x_shard, w_col, None, grp)
    torch.cuda.synchronize()
    want = X.float() @ w_col.float().t()
    report("ag_gemm", err=relerr(y, want), gathered_ok=bool(torch.equal(gathered, X)), ok=relerr(y, want) < 2e-2 and bool(torch.equal(gathered, X)))
    t_f = timed(lambda: fused_tp.ag_gemm(x_shard, w_col, None, grp))
    xg = torch.empty(M, K, dtype=torch.bfloat16, device="cuda")
    yo = torch.empty(M, nl, dtype=torch.bfloat16, device="cuda")

    def baseline_ag():
        dist.all_gather_into_tensor(xg, x_shard)
        torch.matmul(xg, w_col.t(), out=yo)
    t_b = timed(baseline_ag)
    t_g = timed(lambda: torch.matmul(xg, w_col.t(), out=yo))
    report("ag_gemm_perf", fused_ms=t_f, nccl_plus_cublas_ms=t_b, gemm_only_ms=t_g, ok=True)

    # ---------------------------------------------------------------- autograd parity of the fused SP linears
    from paddlefleetx_b200.ops import functional as OF
    from paddlefleetx_b200.parallel import comm_ops as C

    s, b, h = 1024, 2, 1024
    torch.manual_seed(3)
    xs = (torch.randn(s // world, b, h, device="cuda") * 0.5).bfloat16().requires_grad_(True)
    wq = (torch.randn(3 * h // world, h, device="cuda") * 0.05).bfloat16().requires_grad_(True)
    bq = (torch.randn(3 * h // world, device="cuda") * 0.05).bfloat16().requires_grad_(True)
    wo = (torch.randn(h, 3 * h // world, device="cuda") * 0.05).bfloat16().requires_grad_(True)
    go = (torch.randn(s // world, b, h, device="cuda") * 0.1).bfloat16()

    def run(fused):
        for t in (xs, wq, bq, wo):
            t.grad = None
        if fused:
            mid = fused_tp.all_gather_linear(xs, wq, bq, grp)
            out = fused_tp.linear_reduce_scatter(mid, wo, grp)
        else:
            mid = OF.linear(C.all_gather_seq(xs, grp), wq, bq)
            out = C.reduce_scatter_seq(OF.linear(mid, wo, None), grp)
        out.backward(go)
        return [out.detach().clone()] + [t.grad.detach().clone() for t in (xs, wq, bq, wo)]

    ref_out = run(False)
    fus_out = run(True)
    errs = [relerr(a, b_) for a, b_ in zip(fus_out, ref_out)]
    report("fused_sp_linear_autograd", errs=errs, ok=max(errs) < 3e-2)

    # ---------------------------------------------------------------- flat optimizer: P2P path == NCCL path
    from paddlefleetx_b200.optims import ClipGradByGlobalNorm, FusedAdamW

    hc2 = HybridCommunicateGroup(sharding=world)
    torch.manual_seed(11)
    def make():
        m = torch.nn.Sequential(torch.nn.Linear(1024, 2048), torch.nn.Linear(2048, 1024)).cuda().bfloat16()
        return m
    m1, m2 = make(), make()
    m2.load_state_dict(m1.state_dict())
    o1 = FusedAdamW(1e-2, named_parameters=list(m1.named_parameters()), multi_precision=True, hcg=hc2, grad_clip=ClipGradByGlobalNorm(1.0, hc2))
    o2_ = FusedAdamW(1e-2, named_parameters=list(m2.named_parameters()), multi_precision=True, hcg=hc2, use_p2p=True,
                     grad_clip=ClipGradByGlobalNorm(1.0, hc2))
    for step in range(3):
        # the SAME batch on every rank: the cross-rank gradient sum is then exact in bf16 (x world), so the NCCL ring (bf16
        # accumulation) and the peer-memory pull (fp32 accumulation) must agree bit for bit at any world size
        torch.manual_seed(50 + 10 * step)
        xin = torch.randn(64, 1024, device="cuda").bfloat16()
        for m, o in ((m1, o1), (m2, o2_)):
            m(xin).float().pow(2).mean().backward()
            o.step(); o.clear_grad()
    errs = [relerr(a, b_) for a, b_ in zip(m2.parameters(), m1.parameters())]
    report("zero_p2p_vs_nccl", errs=errs, ok=max(errs) < 5e-3)

    # ---------------------------------------------------------------- ZeRO-3: symmetric-memory gathers / reduce-scatter == NCCL path
    try:
        from paddlefleetx_b200.parallel.sharding import GroupShardedStage3

        class Block(torch.nn.Module):          # the wrapper cuts units at classes named like this
            def __init__(self):
                super().__init__()
                self.a, self.b = torch.nn.Linear(1024, 2048), torch.nn.Linear(2048, 1024)

            def forward(self, x):
                return x + self.b(torch.nn.functional.gelu(self.a(x)))

        def make3(nccl):
            os.environ["PFX_ZERO3_NCCL"] = "1" if nccl else "0"
            torch.manual_seed(21)
            net = torch.nn.Sequential(*[Block() for _ in range(4)]).cuda().bfloat16()
            w = GroupShardedStage3(net, hc2)
            o = FusedAdamW(1e-2, named_parameters=w.optimizer_named_parameters(), multi_precision=True, hcg=hc2, params_are_shards=True,
                           apply_decay_param_fun=w.shard_decay_fn())
            return w, o
        (wa, oa), (wb, ob) = make3(True), make3(False)
        assert wb._symm is not None and wa._symm is None
        for step in range(3):
            torch.manual_seed(70 + step)
            xin = torch.randn(32, 1024, device="cuda").bfloat16()
            for w, o in ((wa, oa), (wb, ob)):
                with w.backward_phase():
                    w(xin).float().pow(2).mean().backward()
                o.step(); o.clear_grad(); w.after_optimizer_step()
        sa, sb = wa.state_dict(), wb.state_dict()
        errs = [relerr(sb[k], sa[k]) for k in sa]
        report("zero3_symm_vs_nccl", errs=[round(e, 6) for e in errs[:6]], ok=max(errs) < 5e-3, pool_buffers=sum(len(v) for v in wb._pool.values()))
    except Exception as e:  # noqa: BLE001
        import traceback
        report("zero3_symm_vs_nccl", ok=False, error=repr(e), tb=traceback.format_exc()[-1200:])

    # ---------------------------------------------------------------- MoE: peer-memory dispatch/combine == NCCL all-to-all path
    from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer, MoELayer

    hc3 = HybridCommunicateGroup(dp=world)
    mg = hc3.get_moe_group()
    hm, e_local, tok = 1024, 2, 8192
    def make_moe(fused, grouped=True):
        torch.manual_seed(7 + rank)
        ex = [ExpertLayer(hm, 4 * hm, dtype=torch.bfloat16, device="cuda") for _ in range(e_local)]
        return MoELayer(hm, ex, gate={"type": "naive", "top_k": 2}, moe_group=mg, dtype=torch.bfloat16, device="cuda", fused_p2p=fused,
                        grouped_gemm=grouped)

    def named_grads(layer):      # per-expert names whether the experts' parameters are stacked (grouped path) or not
        names = {"w1": ("htoh4", "weight"), "b1": ("htoh4", "bias"), "w2": ("h4toh", "weight"), "b2": ("h4toh", "bias")}
        out = {}
        for n, p_ in layer.named_parameters():
            if p_.grad is None:
                continue
            if n.startswith("grouped."):
                lin, attr = names[n.split(".")[1]]
                for e in range(p_.shape[0]):
                    out[f"experts.{e}.{lin}.{attr}"] = p_.grad[e].detach().float()
            else:
                out[n] = p_.grad.detach().float()
        return out

    try:
        l_ref, l_loop, l_grp = make_moe(False), make_moe(True, grouped=False), make_moe(True)
        sd = l_ref.state_dict()
        l_loop.load_state_dict(sd); l_grp.load_state_dict(sd)
        same_names = sorted(l_grp.state_dict().keys()) == sorted(sd.keys())
        torch.manual_seed(99 + rank)
        xin = (torch.randn(tok, hm, device="cuda") * 0.5).bfloat16()
        gout = (torch.randn(tok, hm, device="cuda") * 0.1).bfloat16()
        outs = []
        for layer in (l_ref, l_loop, l_grp):
            xi = xin.clone().requires_grad_(True)
            y = layer(xi)
            y.backward(gout)
            g = named_grads(layer)
            outs.append({"y": y.detach(), "dx": xi.grad.detach(), **g})
        keys = sorted(outs[0].keys())
        errs_loop = {k: round(relerr(outs[1][k], outs[0][k]), 5) for k in keys}
        errs_grp = {k: round(relerr(outs[2][k], outs[0][k]), 5) for k in keys}

        def moe_step(layer):
            def f():
                xi = xin.clone().requires_grad_(True)
                layer(xi).backward(gout)
            return f
        t_ref, t_loop, t_grp = timed(moe_step(l_ref), iters=5), timed(moe_step(l_loop), iters=5), timed(moe_step(l_grp), iters=5)
        report("moe_p2p_dispatch_combine", errs=list(errs_loop.values()), ok=max(errs_loop.values()) < 3e-2, ms_nccl=t_ref, ms_p2p=t_loop,
               shape=dict(tokens=tok, hidden=hm, experts_per_rank=e_local, topk=2))
        report("moe_grouped_sync_free", errs=errs_grp, ok=max(errs_grp.values()) < 3e-2 and same_names, checkpoint_names_unchanged=same_names,
               ms_nccl_loop=t_ref, ms_p2p_loop=t_loop, ms_p2p_grouped=t_grp, host_syncs_in_layer=0)
    except Exception as e:  # noqa: BLE001
        import traceback
        report("moe_grouped_sync_free", ok=False, error=repr(e), tb=traceback.format_exc()[-1500:])

    dist.barrier()
    finish(res, rank, world)


def finish(res, rank, world):
    if rank == 0:
        n_ok = sum(1 for v in res.values() if v.get("ok"))
        print(f"MULTI_SELFTEST {n_ok}/{len(res)} ok")
        os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
        with open(os.path.join(ROOT, "gpurun_out", f"multi_selftest_{world}gpu.json"), "w") as f:
            json.dump(res, f, indent=1)
    dist.destroy_process_group()


def nvls_section(lib, grp, rank, world, report):
    """Symmetric memory on cuMem VMM, multicast (NVLS) and unicast variants of the ZeRO kernels against NCCL, and the experiment the
    design rests on: does a communication kernel overlap with a stream of persistent wgmma GEMMs, or serialise with it?"""
    from paddlefleetx_b200.parallel.symmetric_memory import VmmSymmetricAllocator

    caps = lib.vmm_caps()
    report("vmm_caps", ok=bool(caps["vmm"] and caps["fd_export"]), **{k: (int(v) if not isinstance(v, bool) else v) for k, v in caps.items()},
           mc_gran_min=int(lib.vmm_mc_granularity(world, 2 << 20, False)), mc_gran_rec=int(lib.vmm_mc_granularity(world, 2 << 20, True)))
    sm = VmmSymmetricAllocator(grp)
    report("vmm_allocator", ok=True, multicast=bool(sm.multicast), granularity=sm._gran)
    n = 1 << 25                              # elements per shard: 64 MiB of bf16 per rank-shard, bucket = world x that
    buf = sm.alloc_tensor(n * world, torch.bfloat16)
    torch.manual_seed(100 + rank)
    local = (torch.randn(n * world, device="cuda") * 0.1).bfloat16()
    buf.copy_(local)
    torch.cuda.synchronize(); sm.barrier(); torch.cuda.synchronize()
    report("symm_barrier", ok=True, kind="nvls" if sm.multicast else "p2p")
    t_bar = timed(lambda: sm.barrier(), iters=50)
    report("symm_barrier_perf", ok=True, us=t_bar * 1e3)

    ref = torch.empty(n, dtype=torch.bfloat16, device="cuda")
    dist.reduce_scatter_tensor(ref, local.clone())
    peers, mc = sm.peer_ptrs(buf), sm.mc_ptr(buf)
    variants = [("unicast", 0)] + ([("nvls", mc)] if mc else [])
    scratch = local.clone()
    t_nccl = timed(lambda: dist.reduce_scatter_tensor(ref, scratch))
    moved_in = n * 2 * (world - 1)
    for name, mcp in variants:
        out = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        sq = torch.zeros(1, device="cuda")
        lib.symm_reduce_scatter(mcp, peers, rank * n, out, rank, 1, 1.0, False, sq, 64)
        torch.cuda.synchronize(); sm.barrier(); torch.cuda.synchronize()
        want_sq = float(out.float().pow(2).sum())
        e = relerr(out, ref)
        report(f"symm_reduce_scatter_{name}", err=e, sumsq_rel=abs(float(sq) - want_sq) / max(want_sq, 1e-9), ok=e < 1e-2 and abs(float(sq) - want_sq) < 1e-3 * want_sq)
        # fp32 output + accumulate
        o32 = torch.ones(n, dtype=torch.float32, device="cuda")
        lib.symm_reduce_scatter(mcp, peers, rank * n, o32, rank, 1, 0.5, True, None, 64)
        torch.cuda.synchronize(); sm.barrier(); torch.cuda.synchronize()
        e2 = relerr(o32 - 1.0, ref.float() * 0.5)
        report(f"symm_reduce_scatter_{name}_f32acc", err=e2, ok=e2 < 1e-2)
        perf = {}
        for ctas in (16, 32, 64, 128, 264):
            perf[str(ctas)] = timed(lambda: (sm.barrier(), lib.symm_reduce_scatter(mcp, peers, rank * n, out, rank, 1, 1.0, False, None, ctas)))
        best = min(perf.values())
        report(f"symm_reduce_scatter_{name}_perf", ms_by_ctas=perf, nccl_ms=t_nccl, shard_mib=n * 2 / 2 ** 20,
               gbs_link_out=moved_in / best / 1e6, frac_of_770=moved_in / best / 1e6 / 770.0, ok=True)

    # all-gather
    shard = ((torch.arange(n, device="cuda") % 251) + rank).bfloat16()
    gath = torch.empty(n * world, dtype=torch.bfloat16, device="cuda")
    t_ag_nccl = timed(lambda: dist.all_gather_into_tensor(gath, shard))
    for name, mcp in variants:
        buf.zero_()
        torch.cuda.synchronize(); sm.barrier()
        lib.symm_all_gather(mcp, peers, rank * n * 2, shard, rank, 64)
        sm.barrier(); torch.cuda.synchronize()
        ok = all(bool(torch.equal(buf[r * n:(r + 1) * n], ((torch.arange(n, device="cuda") % 251) + r).bfloat16())) for r in range(world))
        perf = {}
        for ctas in (16, 32, 64, 128):
            perf[str(ctas)] = timed(lambda: (lib.symm_all_gather(mcp, peers, rank * n * 2, shard, rank, ctas), sm.barrier()))
        best = min(perf.values())
        report(f"symm_all_gather_{name}", ok=ok, ms_by_ctas=perf, nccl_ms=t_ag_nccl, gbs_link_in=moved_in / best / 1e6, frac_of_770=moved_in / best / 1e6 / 770.0)

    # AdamW + broadcast vs adamw_flat_ + NCCL all-gather
    for name, mcp in variants:
        torch.manual_seed(5)
        pfull = sm.alloc_tensor(n * world, torch.bfloat16)
        master = torch.randn(n, device="cuda") * 0.02 + rank
        g = (torch.randn(n, device="cuda") * 0.01).bfloat16()
        m0, v0 = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        gs, fi = torch.ones(1, device="cuda"), torch.zeros(1, device="cuda")
        ref_master, ref_m, ref_v = master.clone(), m0.clone(), v0.clone()
        ref_lp = torch.empty(n, dtype=torch.bfloat16, device="cuda")
        lib.adamw_flat_(ref_lp, ref_master, g, ref_m, ref_v, 1e-3, 0.9, 0.999, 1e-8, 0.01, 1, gs, fi)
        ref_full = torch.empty(n * world, dtype=torch.bfloat16, device="cuda")
        dist.all_gather_into_tensor(ref_full, ref_lp)
        torch.cuda.synchronize(); sm.barrier()
        lib.adamw_symm_broadcast_(sm.mc_ptr(pfull) if mcp else 0, sm.peer_ptrs(pfull), rank * n, master, g, m0, v0, 1e-3, 0.9, 0.999, 1e-8, 0.01, 1, gs, fi, 1, rank, 264)
        sm.barrier(); torch.cuda.synchronize()
        ok = bool(torch.equal(pfull, ref_full)) and bool(torch.equal(master, ref_master))
        t = timed(lambda: (lib.adamw_symm_broadcast_(sm.mc_ptr(pfull) if mcp else 0, sm.peer_ptrs(pfull), rank * n, master, g, m0, v0, 1e-3, 0.9, 0.999,
                                                     1e-8, 0.01, 2, gs, fi, 1, rank, 264), sm.barrier()))
        t_ref = timed(lambda: (lib.adamw_flat_(ref_lp, ref_master, g, ref_m, ref_v, 1e-3, 0.9, 0.999, 1e-8, 0.01, 2, gs, fi),
                               dist.all_gather_into_tensor(ref_full, ref_lp)))
        report(f"adamw_symm_broadcast_{name}", ok=ok, ms=t, adamw_plus_nccl_ag_ms=t_ref, shard_melems=n / 1e6)

    # ---- overlap experiment: a stream of persistent GEMMs with a reduce-scatter running beside it
    M, N, K = 8192, 16384, 4096
    a = (torch.randn(M, K, device="cuda") * 0.05).bfloat16()
    w = (torch.randn(N, K, device="cuda") * 0.05).bfloat16()
    c = torch.empty(M, N, dtype=torch.bfloat16, device="cuda")
    side = torch.cuda.Stream()
    n_gemm = 24

    def gemms():
        for _ in range(n_gemm):
            lib.gemm(a, w, None, c, True, True, 0, 0, 0)

    big = sm.alloc_tensor(n * world * 2, torch.bfloat16)        # 128 MiB x world bucket
    big.normal_()
    bpeers, bmc = sm.peer_ptrs(big), sm.mc_ptr(big)
    bout = torch.empty(n * 2, dtype=torch.bfloat16, device="cuda")
    nccl_in = torch.randn(n * world * 2, device="cuda").bfloat16()
    reps = 4

    def comm_ours(ctas):
        def f():
            for _ in range(reps):
                sm.barrier()
                lib.symm_reduce_scatter(bmc, bpeers, rank * n * 2, bout, rank, 1, 1.0, False, None, ctas)
        return f

    def comm_nccl():
        for _ in range(reps):
            dist.reduce_scatter_tensor(bout, nccl_in)

    def both(comm):
        def f():
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                comm()
            gemms()
            torch.cuda.current_stream().wait_stream(side)
        return f

    t_g = timed(gemms, iters=3, warmup=1)
    res_ov = {"gemm_only_ms": t_g, "n_gemm": n_gemm, "bucket_mib": n * world * 4 / 2 ** 20, "reps": reps}
    for ctas in (32, 64, 132):
        res_ov[f"ours{ctas}_only_ms"] = timed(comm_ours(ctas), iters=3, warmup=1)
        res_ov[f"ours{ctas}_both_ms"] = timed(both(comm_ours(ctas)), iters=3, warmup=1)
    res_ov["nccl_only_ms"] = timed(comm_nccl, iters=3, warmup=1)
    res_ov["nccl_both_ms"] = timed(both(comm_nccl), iters=3, warmup=1)
    report("overlap_gemm_reduce_scatter", ok=True, **res_ov)


if __name__ == "__main__":
    main()
