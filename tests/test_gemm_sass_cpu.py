"""The persistent wgmma GEMM keeps each k-block's tensor-core products in one unbroken chain.

Every ``gemm_wgmma_kernel`` instantiation in the built library is disassembled (``cuobjdump -sass``).  A k-block of 64 issues
``kBlockK / 16 = 4`` wgmma; compiled as one chain they follow a single ``WARPGROUP.ARRIVE`` back to back and only the last waits on the
scoreboard (``gsb0``).  When ptxas has to fence every wgmma on its own (C7519: for example a runtime choice between the bf16 and fp16
forms inside the k-loop), each HGMMA gets its own ARRIVE and its own ``gsb0``, and the tensor core drains between products.  No GPU needed.
"""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from paddlefleetx_b200.ops import build as B

K_BLOCK, MMA_K = 64, 16


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and Path("/usr/local/cuda/bin/cuobjdump").exists():
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


def _gemm_functions():
    lib, exe = B.lib_path(), _cuobjdump()
    if not lib.exists():
        pytest.skip(f"native library not built: {lib.name}")
    if exe is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([exe, "-sass", str(lib)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        if "gemm_wgmma_kernel" in name:
            funcs[name.strip()] = body
    assert funcs, "no gemm_wgmma_kernel in the library's SASS"
    return funcs


def _hgmma_runs(body: str):
    """HGMMA instructions grouped by the WARPGROUP.ARRIVE that precedes them: one list per group, True where the HGMMA carries gsb0."""
    runs, cur = [], None
    for line in body.splitlines():
        if "WARPGROUP.ARRIVE" in line:
            if cur:
                runs.append(cur)
            cur = []
        elif re.search(r"\bHGMMA\.", line):
            if cur is None:
                cur = []
            cur.append("gsb0" in line)
    if cur:
        runs.append(cur)
    return runs


def test_gemm_wgmma_chains_unbroken():
    funcs = _gemm_functions()
    bad = {}
    for name, body in funcs.items():
        runs = _hgmma_runs(body)
        if not runs or any(len(r) < K_BLOCK // MMA_K or r[-1] is not True or any(r[:-1]) for r in runs):
            bad[name] = [len(r) for r in runs]
    assert not bad, f"{len(bad)} of {len(funcs)} GEMM instantiations break the wgmma chain (HGMMAs per ARRIVE): " + \
        "; ".join(f"{n[:80]}: {r}" for n, r in list(bad.items())[:4])
