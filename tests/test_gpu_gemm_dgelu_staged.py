"""The FFN2 dgrad with the GELU derivative in its epilogue, dz = (dy W) * gelu'(z), whose saved pre-activation z is TMA-loaded into the
epilogue staging buffers (needs an H100).

Against a float64 reference (``kernel_refs.assert_close``, the bound the other dGELU tests use) at both tiles and in both 16-bit dtypes:
several waves of tiles per CTA, so every staging buffer is refilled many times; ragged M, N and K, where the last column tile has z boxes
partly or wholly right of the tensor and K has fewer k-blocks than the pipeline has stages; and the grouped expert GEMM, whose CTAs skip
the row blocks no expert owns.
"""
import pytest
import torch

import kernel_refs as R
from paddlefleetx_b200.ops import _native

pytestmark = pytest.mark.gpu

F16, B16 = torch.float16, torch.bfloat16
EPI_DGELU = 5
SHAPES = {
    "waves": (4096, 6144, 1024),   # 768 tiles of 128 x 256 / 1536 of 128 x 128: 6-12 per CTA on 132 SMs
    "ragged": (1000, 1864, 200),   # M % 128 = 104, N % 256 = 72 (z chunks 2 and 3 of the last wide tile lie right of the tensor), 4 k-blocks
}
SENTINEL = 7.0


@pytest.fixture(scope="module")
def lib():
    return _native.require()


def _gelu_grad(z):
    z64 = z.double().requires_grad_()
    return torch.autograd.grad(torch.nn.functional.gelu(z64, approximate="tanh").sum(), z64)[0]


def _check(got, dy, w, z, dtype, what):
    dy64, w64 = dy.double(), w.double()
    acc, terms = dy64 @ w64, dy64.abs() @ w64.abs()
    dg = _gelu_grad(z)
    scale = terms * dg.abs() + acc.abs() * (1.0 + 2.0 * z.double().abs() ** 3)
    R.assert_close(got, acc * dg, dtype, scale=scale, n=dy.shape[1], approx=R.MMA_ACC + R.TANH_APPROX, what=what)


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("config", [0, 1], ids=["128x128", "128x256"])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_dgelu_staged_against_float64(lib, shape, config, dtype):
    M, N, K = SHAPES[shape]
    g = torch.Generator(device="cuda").manual_seed(M + N + K + config)
    dy = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    w = (torch.randn(K, N, device="cuda", generator=g) * 0.05).to(dtype)
    z = (torch.randn(M, N, device="cuda", generator=g) * 2.0).to(dtype)
    got = lib.gemm_dgelu(dy, w, z, config)
    torch.cuda.synchronize()
    _check(got, dy, w, z, dtype, f"dgelu {shape} config {config}")


@pytest.mark.parametrize("dtype", [B16, F16], ids=["bf16", "fp16"])
def test_dgelu_staged_grouped(lib, dtype):
    """The GELU experts' dgrad: row block r runs expert owners[r]; blocks owned by no expert (-1) are neither loaded nor written."""
    G, K, N = 3, 256, 1096                 # N % 128 = 72
    owners = [0, -1, 2, 2, -1, 0, 1, -1, -1, 1, 0, 2] * 3
    M = 128 * len(owners)
    tile_group = torch.tensor(owners, dtype=torch.int32, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(31)
    dy = torch.randn(M, K, device="cuda", generator=g).to(dtype)
    w = (torch.randn(G, K, N, device="cuda", generator=g) * 0.05).to(dtype)   # MN-major B: [G, K, N]
    z = (torch.randn(M, N, device="cuda", generator=g) * 2.0).to(dtype)
    out = torch.full((M, N), SENTINEL, device="cuda", dtype=dtype)
    lib.gemm_grouped(dy, w, None, tile_group, out, False, EPI_DGELU, None, z, 128)
    torch.cuda.synchronize()
    for blk, e in enumerate(owners):
        rows = slice(128 * blk, 128 * (blk + 1))
        if e < 0:
            assert bool((out[rows] == SENTINEL).all()), f"row block {blk} is owned by no expert but was written"
            continue
        _check(out[rows], dy[rows], w[e], z[rows], dtype, f"grouped dgelu block {blk}")
