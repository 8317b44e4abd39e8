"""In-tree AOT build of the sm_90a kernel library (``_pfx_native*.so``) and the C++ data helper.

``nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo`` for every ``.cu`` (they include no torch
headers, so each compiles in seconds), ``g++`` for the single pybind/torch binding file, one link.  The
resulting ``.so`` lives next to this file so that it travels with the source tree to the GPU box; a content
hash of the sources is stored beside it and the library is rebuilt only when the hash changes.

Run ``python -m paddlefleetx_b200.ops.build`` (or ``__graft_entry__.build()``).
"""
from __future__ import annotations

import hashlib
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
BUILD_DIR = HERE / "csrc" / "build"
MODULE_NAME = "_pfx_native"
CUDA_SOURCES = ["gemm_sm90.cu", "norm_act.cu", "loss_optim.cu", "sampling_attn_misc.cu", "comm_p2p.cu",
                "gemm_lowp_sm90.cu", "quant_kernels.cu", "moe_kernels.cu", "gemv_skinny.cu", "gemm_smallm_sm90.cu", "attention_decode.cu", "attention_fwd_sm90.cu", "comm_nvls.cu", "attention_bwd_sm90.cu", "evoformer_attn_sm90.cu", "embedding.cu"]
CPP_SOURCES = ["bindings.cpp", "symm_vmm.cpp"]
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _ext_suffix() -> str:
    return sysconfig.get_config_var("EXT_SUFFIX") or ".so"


def lib_path() -> Path:
    return HERE / f"{MODULE_NAME}{_ext_suffix()}"


def _existing(sources):
    return [s for s in sources if (CSRC / s).exists()]


def _hash_sources() -> str:
    h = hashlib.sha256()
    files = sorted(p for p in CSRC.iterdir() if p.suffix in (".cu", ".cuh", ".h", ".cpp"))
    for p in files:
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(ARCH_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    stamp = HERE / f"{MODULE_NAME}.hash"
    return lib_path().exists() and stamp.exists() and stamp.read_text().strip() == _hash_sources()


def _run(cmd, verbose):
    if verbose:
        print(" ".join(map(str, cmd)), flush=True)
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"build step failed: {' '.join(map(str, cmd))}\n{res.stdout}")
    return res.stdout


def build(force: bool = False, verbose: bool = True) -> Path:
    if not force and is_fresh():
        return lib_path()
    import torch
    from torch.utils import cpp_extension as ce

    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    cuda_home = Path(nvcc).resolve().parent.parent
    BUILD_DIR.mkdir(parents=True, exist_ok=True)
    inc = [f"-I{p}" for p in ce.include_paths()] + [f"-I{cuda_home}/include", f"-I{sysconfig.get_paths()['include']}", f"-I{CSRC}"]
    cxx_abi = f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"

    jobs = []
    for src in _existing(CUDA_SOURCES):
        obj = BUILD_DIR / (src + ".o")
        cmd = [nvcc, *ARCH_FLAGS, "-std=c++17", "-O3", "-lineinfo", "--use_fast_math", "-Xcompiler", "-fPIC",
               f"-I{CSRC}", "-c", str(CSRC / src), "-o", str(obj)]
        jobs.append((cmd, obj))
    for src in _existing(CPP_SOURCES):
        obj = BUILD_DIR / (src + ".o")
        cmd = ["g++", "-std=c++17", "-O2", "-fPIC", cxx_abi, f"-DTORCH_EXTENSION_NAME={MODULE_NAME}",
               "-DTORCH_API_INCLUDE_EXTENSION_H", *inc, "-c", str(CSRC / src), "-o", str(obj)]
        jobs.append((cmd, obj))
    with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as pool:
        list(pool.map(lambda j: _run(j[0], verbose), jobs))

    torch_lib = Path(torch.__file__).parent / "lib"
    tmp_lib = BUILD_DIR / (lib_path().name + ".tmp")      # link beside, then rename: a concurrent reader never sees half a file
    link = ["g++", "-shared", "-o", str(tmp_lib), *[str(o) for _, o in jobs],
            f"-L{torch_lib}", f"-L{cuda_home}/lib64", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch_cuda", "-ltorch",
            "-ltorch_python", "-lcudart", f"-Wl,-rpath,{torch_lib}", f"-Wl,-rpath,{cuda_home}/lib64"]
    _run(link, verbose)
    import os

    os.replace(tmp_lib, lib_path())
    (HERE / f"{MODULE_NAME}.hash").write_text(_hash_sources())
    return lib_path()


def build_data_helper(force: bool = False, verbose: bool = True) -> Path:
    """C++ index-map helper for the datasets (pybind11, no torch)."""
    src = HERE.parent / "data" / "data_tools" / "cpp" / "fast_index_map_helpers.cpp"
    out = src.parent / f"fast_index_map_helpers{_ext_suffix()}"
    if not src.exists():
        return out
    if out.exists() and not force and out.stat().st_mtime >= src.stat().st_mtime:
        return out
    import pybind11

    cmd = ["g++", "-O3", "-std=c++17", "-shared", "-fPIC", f"-I{pybind11.get_include()}",
           f"-I{sysconfig.get_paths()['include']}", str(src), "-o", str(out)]
    _run(cmd, verbose)
    return out


if __name__ == "__main__":
    p = build(force="--force" in sys.argv)
    print(f"built {p}")
    print(f"built {build_data_helper(force='--force' in sys.argv)}")
