"""Which GEMMs ask for the 128 x 256 tile, and that the library contains it.  No GPU needed.

The wgmma GEMM's ``config`` argument asks for the wide tile.  The forward GEMMs must not ask for it: the overlapped AdamW update of the
previous step runs beside them and needs room on the SM.  The backward GEMMs ask for it unless an optimizer that overlaps gradient
collectives with the backward (more than one replica) has turned it off.  The first part routes a tiny ``linear`` and fused FFN through
a recording stand-in for the native library; the second reads the SASS of the built library.
"""
import re
import shutil
import subprocess
import types
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import build as B
from paddlefleetx_b200.ops import functional as OF


class _RecordingLib:
    """The GEMM entry points the linear and fused-FFN autograd functions call, computed with torch; each call records its config."""

    def __init__(self):
        self.calls = []

    def gemm(self, a, b, bias, out, a_kmajor, b_kmajor, epilogue, out_mode, config):
        self.calls.append(("gemm", out_mode, config))
        y = (a if a_kmajor else a.t()).float() @ (b if b_kmajor else b.t()).float().t()
        if bias is not None:
            y = y + bias.float()
        if out is None:
            return y.to(a.dtype)
        if out_mode == 2:
            out.add_(y.to(out.dtype))
        else:
            out.copy_(y.to(out.dtype))
        return out

    def gemm_bias_gelu_dual(self, x, w, bias):
        self.calls.append(("gemm_bias_gelu_dual", 0, 0))
        z = (x.float() @ w.float().t() + bias.float()).to(x.dtype)
        return z, F.gelu(z.float(), approximate="tanh").to(x.dtype)

    def gemm_dgelu(self, dy, w, z, config=0):
        self.calls.append(("gemm_dgelu", 0, config))
        with torch.enable_grad():                                # called from a backward, where grad mode is off
            zf = z.float().requires_grad_()
            dg = torch.autograd.grad(F.gelu(zf, approximate="tanh").sum(), zf)[0]
        return ((dy.float() @ w.float()) * dg).to(dy.dtype)

    def colsum(self, x, out_fp32):
        return x.float().sum(0).to(torch.float32 if out_fp32 else x.dtype)


@pytest.fixture
def lib(monkeypatch):
    fake = _RecordingLib()
    monkeypatch.setattr(_native, "require", lambda: fake)
    OF.set_wide_backward(True)
    yield fake
    OF.set_wide_backward(True)


def _leaf(*shape, scale=1.0):
    return (torch.randn(*shape) * scale).to(torch.bfloat16).requires_grad_()


def test_linear_forward_128_backward_wide(lib):
    torch.manual_seed(0)
    x, w, b = _leaf(4, 16, 32), _leaf(24, 32, scale=0.1), _leaf(24)
    y = OF._LinearFn.apply(x, w, b)
    assert lib.calls == [("gemm", 0, 0)]
    lib.calls.clear()
    y.float().sum().backward()
    assert lib.calls == [("gemm", 0, 1), ("gemm", 0, 1)]       # dgrad, wgrad


def test_wgrad_into_main_grad(lib):
    """A 16-bit main gradient is written by the wide tile (out mode 0); an fp32 one by the fp32 output modes, which stay 128 x 128."""
    torch.manual_seed(1)
    x, g = torch.randn(64, 32).to(torch.bfloat16), torch.randn(64, 24).to(torch.bfloat16)
    for dtype, out_modes, config in [(torch.bfloat16, [0, 0], 1), (torch.float32, [1, 2], 0)]:
        w = torch.zeros(24, 32, dtype=torch.bfloat16)
        w.main_grad = torch.zeros(24, 32, dtype=dtype)
        w._grad_fresh = True
        lib.calls.clear()
        OF._wgrad(lib, g, x, w)
        OF._wgrad(lib, g, x, w)                                 # second touch: accumulate
        assert lib.calls == [("gemm", m, config) for m in out_modes], dtype
        torch.testing.assert_close(w.main_grad.float(), 2 * (g.float().t() @ x.float()), rtol=2e-2, atol=2e-2)


def test_fused_ffn_forward_128_backward_wide(lib):
    torch.manual_seed(2)
    x, w1, b1, w2 = _leaf(2, 8, 32), _leaf(64, 32, scale=0.1), _leaf(64), _leaf(32, 64, scale=0.1)
    y = OF._FusedFFNFn.apply(x, w1, b1, w2, None)
    assert [c[2] for c in lib.calls] == [0, 0]
    lib.calls.clear()
    y.float().sum().backward()
    assert lib.calls == [("gemm_dgelu", 0, 1), ("gemm", 0, 1), ("gemm", 0, 1), ("gemm", 0, 1)]   # dgelu, wgrad 2, wgrad 1, dgrad


def test_switch_off_keeps_128(lib):
    torch.manual_seed(3)
    OF.set_wide_backward(False)
    x, w = _leaf(16, 32), _leaf(24, 32, scale=0.1)
    OF._LinearFn.apply(x, w, None).float().sum().backward()
    assert [c[2] for c in lib.calls] == [0, 0, 0]


def test_optimizer_with_replicas_turns_wide_off(lib):
    from paddlefleetx_b200.optims import FusedAdamW

    w = torch.nn.Parameter(torch.randn(8, 8))
    FusedAdamW(1e-3, named_parameters=[("w", w)])
    assert OF.wide_backward()                                   # one replica: the backward keeps the wide tile
    dp = types.SimpleNamespace(nranks=2, rank=0, process_group=None)
    hcg = types.SimpleNamespace(get_sharding_parallel_group=lambda: None, get_data_parallel_group=lambda: dp)
    FusedAdamW(1e-3, named_parameters=[("w", w)], hcg=hcg)
    assert not OF.wide_backward()


def _cuobjdump():
    exe = shutil.which("cuobjdump")
    if exe is None and Path("/usr/local/cuda/bin/cuobjdump").exists():
        exe = "/usr/local/cuda/bin/cuobjdump"
    return exe


def test_library_has_wide_gemm():
    """Every operand major and both 16-bit dtypes have a 128 x 256 instantiation: m64n256k16 products and register reallocation."""
    lib, exe = B.lib_path(), _cuobjdump()
    if not lib.exists():
        pytest.skip(f"native library not built: {lib.name}")
    if exe is None:
        pytest.skip("cuobjdump not found")
    sass = subprocess.run([exe, "-sass", str(lib)], capture_output=True, text=True, check=True).stdout
    wide = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        m = re.search(r"gemm_wgmma_kernelILi256ELb([01])ELb([01])ELi0ELb([01])E", name)
        if m:
            wide[m.groups()] = body
    assert len(wide) == 8, f"expected 8 wide GEMM instantiations (4 majors x 2 dtypes), found {sorted(wide)}"
    for key, body in wide.items():
        hgmma = re.findall(r"HGMMA\.64x256x16\.F32\S*", body)
        assert hgmma, f"wide GEMM {key} has no HGMMA.64x256x16"
        assert all(h.endswith(".BF16") == (key[2] == "1") for h in hgmma), f"wide GEMM {key}: {sorted(set(hgmma))}"   # fp16 has no suffix
        assert "USETMAXREG" in body, f"wide GEMM {key} does not reallocate registers"
        assert not re.search(r"\b(STL|LDL)\b", body), f"wide GEMM {key} spills to local memory"
