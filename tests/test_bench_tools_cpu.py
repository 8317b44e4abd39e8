"""Host-side pieces of the benchmark contract that need no GPU: the nvidia-smi sampler's parsing (clocks / throttle reasons / power in the
bench line), the interval arithmetic of tools/analyze_trace.py, and the reference-arm line of bench.py."""
import gzip
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def test_clock_sampler_summarises_rows():
    from bench import ClockSampler

    s = ClockSampler(0)
    s.rows = [["1410", "1965", "955.2", "Not Active", "Not Active", "Not Active", "Active"],
              ["1395", "1965", "981.0", "Not Active", "Not Active", "Not Active", "Active"],
              ["1425", "1965", "940.9", "Not Active", "Not Active", "Not Active", "Not Active"],
              ["[N/A]", "1965", "[N/A]", "Not Active", "Active", "Not Active", "Not Active"]]
    out = s.stop()
    assert out["sm_mhz"] == 1410 and out["sm_max_mhz"] == 1965 and out["samples"] == 3
    assert out["reasons"] == ["hw_thermal_slowdown", "sw_power_cap"] and abs(out["power_w"] - 955.2) < 1e-6
    assert ClockSampler(0).stop() == {"sm_mhz": None, "sm_max_mhz": None, "reasons": [], "samples": 0, "power_w": None}


def test_analyze_trace_interval_arithmetic_and_report(tmp_path, capsys):
    import analyze_trace as A

    assert A.merge([(5, 7), (0, 2), (1, 3), (7, 8)]) == [[0, 3], [5, 8]]
    assert A.total([[0, 3], [5, 8]]) == 6
    assert A.intersect([[0, 3], [5, 8]], [[2, 6], [7, 9]]) == 1 + 1 + 1
    trace = {"steps": 2, "model": "toy", "n_gpus": 1, "columns": ["name", "stream", "ts_us", "dur_us"],
             "kernels": [["void pfx::gemm_wgmma_kernel<128>", 7, 0.0, 100.0], ["pfx::(anonymous namespace)::adamw_flat_kernel", 9, 50.0, 100.0],
                         ["void pfx::gemm_wgmma_kernel<128>", 7, 200.0, 100.0], ["ncclDevKernel_ReduceScatter", 9, 250.0, 100.0]]}
    path = tmp_path / "t.json.gz"
    with gzip.open(path, "wt") as f:
        json.dump(trace, f)
    old = sys.argv
    sys.argv = ["analyze_trace.py", str(path), "--top", "5"]
    try:
        A.main()
    finally:
        sys.argv = old
    out = capsys.readouterr().out
    assert "4 kernels over 2 steps" in out and "gemm_wgmma_kernel" in out


def test_reference_arm_reports_unavailable_and_exits_zero():
    p = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "1", "--steps", "2", "--warmup", "1"],
                       capture_output=True, text=True, timeout=120, cwd=ROOT)
    assert p.returncode == 0, p.stderr[-800:]
    line = json.loads(p.stdout.strip().splitlines()[-1])
    assert line["impl"] == "reference" and "unavailable" in line and "paddle" in line["unavailable"].lower()


def test_child_job_of_a_torchrun_job_can_rendezvous(tmp_path):
    """bench.py --gpus 8 starts BASELINE config #2 as a child job from every rank.  The child must not inherit the elastic agent's store
    (it would wait forever on a port nobody serves): two gloo ranks under torchrun each start a child with child_job_env and the children
    complete an all-reduce."""
    parent = tmp_path / "parent.py"
    child = tmp_path / "child.py"
    child.write_text("import torch, torch.distributed as dist\ndist.init_process_group('gloo')\nt = torch.ones(1)\ndist.all_reduce(t)\nprint('CHILD_OK', int(t.item()))\n")
    parent.write_text(
        "import os, subprocess, sys\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "import torch.distributed as dist\n"
        "from bench import child_job_env\n"
        "dist.init_process_group('gloo')\n"
        f"p = subprocess.run([sys.executable, {str(child)!r}], env=child_job_env(os.environ), capture_output=True, text=True, timeout=60)\n"
        "print('PARENT', dist.get_rank(), p.stdout.strip(), p.stderr[-300:])\n")
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr=127.0.0.1", "--master-port=29733",
                        str(parent)], capture_output=True, text=True, timeout=180, cwd=ROOT)
    assert p.returncode == 0, p.stderr[-1500:]
    assert p.stdout.count("CHILD_OK 2") == 2, p.stdout[-1500:] + p.stderr[-500:]
