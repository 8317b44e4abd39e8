"""Environment validation (the reference tells users to run ``paddle.utils.run_check()`` and a launcher check — docs/deployment_faq.md:75,107):

    python tools/run_check.py                 # this process: CUDA device, sm_90a, native library, one wgmma GEMM vs PyTorch
    python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 tools/run_check.py   # + NCCL all-reduce, P2P access, peer-memory barrier
"""
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

import torch  # noqa: E402


def main():
    """Validate this process's environment (device, architecture, native library, one GEMM) and, under a launcher, the collectives between ranks."""
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    ok = True

    def say(msg, good=True):
        nonlocal ok
        ok = ok and good
        if rank == 0:
            print(("[ OK ] " if good else "[FAIL] ") + msg, flush=True)

    say(f"torch {torch.__version__}, CUDA runtime {torch.version.cuda}")
    if not torch.cuda.is_available():
        say("no CUDA device visible: only the CPU functional path (Global.device=cpu, gloo) is usable", False)
        return 1
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    cap = torch.cuda.get_device_capability()
    props = torch.cuda.get_device_properties(local)
    say(f"device {local}: {props.name}, sm_{cap[0]}{cap[1]}, {props.multi_processor_count} SMs, {props.total_memory / 2**30:.0f} GiB", cap == (9, 0))
    from paddlefleetx_b200.ops import _native

    lib = _native.load()
    say(f"native kernel library loaded: {getattr(lib, '__file__', lib)}", lib is not None)
    if lib is not None and cap == (9, 0):
        a = torch.randn(512, 256, device="cuda").bfloat16()
        b = torch.randn(384, 256, device="cuda").bfloat16()
        y = lib.gemm(a, b, None, None, True, True, 0, 0, 0)
        err = float((y.float() - a.float() @ b.float().t()).norm() / (a.float() @ b.float().t()).norm())
        say(f"wgmma GEMM vs fp32 reference: rel. error {err:.2e}", err < 1e-2)
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
        t = torch.ones(1 << 20, device="cuda") * (rank + 1)
        dist.all_reduce(t)
        say(f"NCCL all-reduce over {world} ranks", abs(float(t[0]) - world * (world + 1) / 2) < 1e-3)
        peers = [torch.cuda.can_device_access_peer(local, p) for p in range(torch.cuda.device_count()) if p != local]
        say(f"P2P access to {sum(peers)}/{len(peers)} peers (needed by the peer-memory kernels)", all(peers))
        if all(peers) and lib is not None:
            from paddlefleetx_b200.parallel.symmetric_memory import SymmetricAllocator
            from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

            sm = SymmetricAllocator(HybridCommunicateGroup(sharding=world).get_sharding_parallel_group())
            buf = sm.alloc_tensor(1024, torch.float32)
            buf.fill_(rank)
            torch.cuda.synchronize(); sm.barrier(); torch.cuda.synchronize()
            nxt = sm.peer_tensor(buf, (rank + 1) % world)
            say("CUDA-IPC symmetric memory + device barrier", float(nxt[0]) == (rank + 1) % world)
        dist.barrier()
        dist.destroy_process_group()
    if rank == 0:
        print("run_check: " + ("all good" if ok else "problems found"), flush=True)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
