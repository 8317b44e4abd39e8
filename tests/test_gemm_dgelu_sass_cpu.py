"""The dGELU GEMM (out mode 6: z TMA-loaded into the epilogue staging buffers) is compiled for the FFN2 dgrad's operand majors at both tiles.

The built library is disassembled (``cuobjdump -sass``): each dtype has a 128 x 128 and a 128 x 256 instantiation for A K-major, B
MN-major, none spills to local memory, the wide one runs m64n256k16 products with register reallocation, and the epilogue reads z from
shared memory.  No GPU needed.
"""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from paddlefleetx_b200.ops import build as B


def _dgelu_functions():
    lib = B.lib_path()
    exe = shutil.which("cuobjdump") or ("/usr/local/cuda/bin/cuobjdump" if Path("/usr/local/cuda/bin/cuobjdump").exists() else None)
    if not lib.exists():
        pytest.skip(f"native library not built: {lib.name}")
    if exe is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([exe, "-sass", str(lib)], capture_output=True, text=True, check=True).stdout
    funcs = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        m = re.search(r"gemm_wgmma_kernelILi(\d+)ELb([01])ELb([01])ELi6ELb([01])E", name)
        if m:
            funcs[m.groups()] = body
    return funcs


def test_dgelu_instantiations():
    funcs = _dgelu_functions()
    assert sorted(funcs) == [(n, "1", "0", bf) for n in ("128", "256") for bf in ("0", "1")], sorted(funcs)
    for (n, _, _, bf), body in funcs.items():
        hgmma = set(re.findall(r"HGMMA\.(\d+x\d+x16)\.F32(\S*)", body))
        assert hgmma == {(f"64x{n}x16", ".BF16" if bf == "1" else "")}, f"dgelu 128 x {n} bf16={bf}: {sorted(hgmma)}"
        assert not re.search(r"\b(STL|LDL)\b", body), f"dgelu 128 x {n} bf16={bf} spills to local memory"
        assert re.search(r"\bLDS\b", body), f"dgelu 128 x {n} bf16={bf} does not read z from shared memory"
        assert ("USETMAXREG" in body) == (n == "256"), f"dgelu 128 x {n} bf16={bf}: register reallocation on the wide tile only"
