"""The text-generation kernels against exact and float64 references (needs an H100): the Philox stream the sampler draws from, the top-p
sampler on rows whose choice is exact and on realistic rows, the decode GEMVs (``gemv_skinny`` / ``gemv_fused``) and the small-M GEMM
(``gemm_smallm``) within the bounds of ``decode_refs`` / ``kernel_refs``, the router of ``OF.linear`` at its edges, and the refusals of
operands the kernels cannot read."""
import numpy as np
import pytest
import torch

import decode_refs as D
import kernel_refs as R
from paddlefleetx_b200.ops import _native
from paddlefleetx_b200.ops import functional as OF

pytestmark = pytest.mark.gpu

F32, B16, F16 = torch.float32, torch.bfloat16, torch.float16
DTYPES = [B16, F16]
_worst = {}


def _record(name, dtype, r):
    key = f"{name} {str(dtype).split('.')[-1]}"
    _worst[key] = max(_worst.get(key, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    for k, v in sorted(_worst.items()):
        print(f"largest error / bound: {k}: {v:.3g}")


def _lib():
    return _native.require()


def _randn(*shape, seed, scale=1.0, shift=0.0, dtype=B16):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale + shift).to(dtype)


# ---------------------------------------------------------------------------------------------------------------- Philox
def test_dropout_keep_mask_is_the_philox_port():
    """dropout_bwd of ones exposes Philox::keep8 bit for bit; the seed and offset fill both words of the key and of the counter."""
    seed, offset, rows, cols = 0x0123456789ABCDEF, 2 ** 33 + 5, 64, 1024
    ones = torch.ones(rows, cols, dtype=B16, device="cuda")
    kept = (_lib().dropout_bwd(ones, 0.5, seed, offset) != 0).reshape(-1).cpu().numpy()
    want = D.keep8(seed, offset, rows * cols // 8, 0x8000)
    assert kept.shape == want.shape and int((kept != want).sum()) == 0, np.flatnonzero(kept != want)[:8]


# ---------------------------------------------------------------------------------------------------------------- top-p, exact
UNIT = 2 ** 20
# (V, tie classes as (count, probability in units of 2^-20), top_p).  Every probability has at most 8 significant bits and is >= 2^-20, so
# it is exact in fp32, bf16 and fp16 (subnormal there below 2^-14); the rest of the unit mass is one token per set bit, the other tokens are
# 0.  Every partial sum is then exact in fp32, whatever the order, and the kernel's choice is fully determined.
EXACT_CASES = {
    "flat_1024": (1024, [(1024, 1024)], 1.0),
    "flat_1025_one_zero": (1025, [(1024, 1024)], 0.9),
    "single_token": (1, [(1, UNIT)], 0.5),
    "ties_2": (7, [(2, 3 << 17)], 0.9),
    "ties_31": (1000, [(31, 3 << 13)], 0.9),
    "ties_32": (1000, [(32, 3 << 13)], 1.0),
    "ties_33": (1000, [(33, 3 << 13)], 1.0),
    "ties_100_and_5000": (50304, [(100, 3 << 6), (5000, 191)], 1.0),
    "ties_100_and_5000_half": (50304, [(100, 3 << 6), (5000, 191)], 0.5),
    "ties_40000": (50304, [(40000, 26)], 0.9),
    "tied_maximum": (1025, [(3, 3 << 16), (400, 1024)], 0.9),
    "tied_maximum_small_p": (1025, [(3, 3 << 16), (400, 1024)], 2.0 ** -10),
}
EXACT_ROWS = 512


def _exact_row(V, classes, seed):
    vals = [unit for count, unit in classes for _ in range(count)]
    rest = UNIT - sum(vals)
    assert rest >= 0
    vals += [1 << b for b in range(21) if rest >> b & 1]
    assert len(vals) <= V
    units = np.zeros(V, np.int64)
    units[:len(vals)] = vals
    return np.random.default_rng(seed).permutation(units)


@pytest.mark.parametrize("dtype", [F32, B16, F16])
@pytest.mark.parametrize("case", list(EXACT_CASES))
def test_topp_exact(case, dtype):
    """R identical rows, each with its own Philox counter (offset + row): R independent draws, each of which has one right answer."""
    V, classes, top_p = EXACT_CASES[case]
    row = torch.tensor(_exact_row(V, classes, seed=V + len(classes)), dtype=torch.float64) / UNIT
    assert float(row.sum()) == 1.0
    probs = row.to(dtype)
    assert torch.equal(probs.double(), row), "the case's probabilities must be exact in this dtype"
    probs = probs.cuda().expand(EXACT_ROWS, V).contiguous()
    seed, offset = 20240917, 1000
    counters = offset + np.arange(EXACT_ROWS, dtype=np.uint64)
    tp = torch.full((EXACT_ROWS,), top_p, device="cuda")
    out_p, out_i = _lib().topp_sampling(probs, tp, seed, offset)
    want, _ = D.topp_expected(row.cuda().expand(EXACT_ROWS, V), tp.cpu().numpy(), D.uniform(seed, counters))
    got = out_i.reshape(-1)
    bad = (got != want).nonzero().reshape(-1)
    assert bad.numel() == 0, (f"{case} {dtype}: {bad.numel()} of {EXACT_ROWS} draws picked the wrong token; first rows "
                              f"{bad[:4].tolist()}: got {got[bad[:4]].tolist()}, want {want[bad[:4]].tolist()}")
    assert out_p.dtype == dtype and torch.equal(out_p.reshape(-1), probs[0, got])


# ---------------------------------------------------------------------------------------------------------------- top-p, realistic
@pytest.mark.parametrize("dtype", DTYPES)
def test_topp_realistic_rows_follow_the_float64_law(dtype):
    """LM-head-like rows: 16-bit logits (so that many fp32 probabilities tie exactly), an fp32 softmax, top_p 0.9 / 0.5 / 1.  The kernel
    sums up to V masses of at most 1 in fp32, so its cumulative masses are within delta = V 2^-24 of float64: the chosen token's interval
    must come within delta of the threshold, and where the threshold is farther than delta from every boundary the choice is the law's."""
    V, per_sd = 50304, 1024
    logits = torch.cat([_randn(per_sd, V, seed=sd, scale=sd, dtype=dtype) for sd in (1, 2, 3)]).float()
    probs = torch.softmax(logits, -1)
    rows = probs.shape[0]
    tp = torch.tensor([0.9, 0.5, 1.0], device="cuda").repeat(rows // 3 + 1)[:rows]
    seed, offset = 77, 2 ** 32 + 3
    counters = offset + np.arange(rows, dtype=np.uint64)
    out_p, out_i = _lib().topp_sampling(probs, tp, seed, offset)
    ids = out_i.reshape(-1)
    assert torch.equal(out_p.reshape(-1), probs.gather(1, out_i).reshape(-1))
    _, via_of = OF.topp_sampling(probs, tp, seed, offset)
    assert torch.equal(via_of.reshape(-1), ids)

    u = D.uniform(seed, counters)
    want, margin = D.topp_expected(probs, tp.cpu().numpy(), u)
    thr = torch.as_tensor(D.topp_threshold(seed, counters, tp.cpu().numpy())).to("cuda", torch.float64)
    order, cum = D.sorted_mass(probs)
    pos = torch.empty_like(order).scatter_(1, order, torch.arange(V, device="cuda").expand(rows, V))
    k = pos.gather(1, ids[:, None]).reshape(-1)
    hi = cum.gather(1, k[:, None]).reshape(-1)
    lo = hi - probs.double().gather(1, ids[:, None]).reshape(-1)
    delta = V * 2.0 ** -24
    outside = ((thr < lo - delta) | (thr > hi + delta)).nonzero().reshape(-1)
    assert outside.numel() == 0, f"rows {outside[:4].tolist()}: threshold {thr[outside[:4]].tolist()} outside [{lo[outside[:4]].tolist()}, " \
                                 f"{hi[outside[:4]].tolist()}]"
    clear = margin > delta
    assert torch.equal(ids[clear], want[clear])
    ties = int(((probs.gather(1, ids[:, None]) == probs).sum(-1) > 32).sum())
    print(f"top-p realistic {dtype}: {int((ids != want).sum())} of {rows} rows differ from the float64 choice "
          f"({int((~clear).sum())} thresholds within delta of a boundary); {ties} draws landed in a class of more than 32 tied tokens")


# ---------------------------------------------------------------------------------------------------------------- refusals
def test_gemv_refuses_operands_it_cannot_read():
    lib = _lib()
    M, K, N = 2, 64, 16
    x, w = _randn(M, K, seed=1), _randn(N, K, seed=2)
    lnw, lnb = torch.ones(K, dtype=B16, device="cuda"), torch.zeros(K, dtype=B16, device="cuda")

    def shifted(t):                                      # the same values at a 2-byte offset: contiguous, not 16-byte aligned
        flat = torch.empty(t.numel() + 8, dtype=t.dtype, device="cuda")
        v = flat[1:1 + t.numel()].view(t.shape)
        v.copy_(t)
        return v

    with pytest.raises(RuntimeError, match="x must be 16-byte aligned"):
        lib.gemv_skinny(shifted(x), w, None)
    with pytest.raises(RuntimeError, match="w must be 16-byte aligned"):
        lib.gemv_fused(x, shifted(w), None, None, None, 1e-5, None, 0)
    with pytest.raises(RuntimeError, match="ln params must be 16-byte aligned"):
        lib.gemv_fused(x, w, None, shifted(lnw), lnb, 1e-5, None, 0)
    with pytest.raises(RuntimeError, match="bias"):
        lib.gemv_skinny(x, w, torch.zeros(N, device="cuda"))                      # fp32 bias with bf16 operands
    with pytest.raises(RuntimeError, match="bias"):
        lib.gemv_fused(x, w, torch.zeros(N - 1, dtype=B16, device="cuda"), None, None, 1e-5, None, 0)
    with pytest.raises(RuntimeError, match="bias"):
        lib.gemv_skinny(x, w, torch.zeros(N, dtype=B16))                          # on the host
    with pytest.raises(RuntimeError, match="ln params"):
        lib.gemv_fused(x, w, None, lnw, lnb.half(), 1e-5, None, 0)
    with torch.no_grad(), pytest.raises(RuntimeError, match="bias"):
        OF.linear(x, w, torch.zeros(N, device="cuda"))                           # the router does not hand an fp32 bias to the GEMV


def test_topp_refuses_a_host_or_missized_top_ps():
    probs = torch.softmax(_randn(4, 1000, seed=3, dtype=F32), -1)
    with pytest.raises(RuntimeError, match="top_ps must be on"):
        _lib().topp_sampling(probs, torch.full((4,), 0.9), 1, 0)
    with pytest.raises(RuntimeError, match="one entry per row"):
        _lib().topp_sampling(probs, torch.full((3,), 0.9, device="cuda"), 1, 0)


# ---------------------------------------------------------------------------------------------------------------- decode GEMV
TUNINGS = [(0, 0)] + [(c, s) for c in (2, 4) for s in (1, 2, 4, 8)]       # the heuristic, then every column-group width x K split
# (K, N): K = 8 is one 16-byte vector, 1032 is not a multiple of a 32-lane sweep (256 elements), 16392 takes the 8-slice FFN2 split
GEMV_SHAPES = [(8, 1000), (1032, 50304), (16392, 4100), (1032, 3), (8, 1), (16392, 1000), (1032, 4100), (8, 50304), (16392, 3)]
ACTS = [None, "gelu", "swiglu"]


def _gemv_case(M, K, N, act, ln, bias, res, dtype, seed):
    N = N + N % 2 if act == "swiglu" else N
    x = _randn(M, K, seed=seed, shift=100.0 if ln else 0.0, dtype=dtype)         # +100: a one-pass variance would cancel
    w = _randn(N, K, seed=seed + 1, scale=2 * K ** -0.5, dtype=dtype)
    b = _randn(N, seed=seed + 2, scale=0.5, dtype=dtype) if bias else None
    lnp = None
    if ln:
        g = torch.Generator(device="cuda").manual_seed(seed + 3)
        lnp = ((torch.rand(K, generator=g, device="cuda") + 0.5).to(dtype), _randn(K, seed=seed + 4, scale=0.1, dtype=dtype), 1e-5)
    r = _randn(M, N // 2 if act == "swiglu" else N, seed=seed + 5, dtype=dtype) if res else None
    return x, w, b, lnp, r


def _run_gemv(x, w, b, lnp, r, act):
    if lnp is None and r is None and act is None:
        return _lib().gemv_skinny(x, w, b)
    return OF.gemv_fused(x, w, b, ln=lnp, residual=r, act=act)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", range(1, 9))
def test_gemv_against_float64(dtype, M):
    """Every (rows, tuning) pair once; shape, activation, LayerNorm, bias and residual rotate with it."""
    for t, (cols, split) in enumerate(TUNINGS):
        K, N = GEMV_SHAPES[(t + 4 * M) % len(GEMV_SHAPES)]
        act = ACTS[(t + 2 * M) % 3]
        ln, bias, res = (t // 3 + M) % 2 == 1, (t + M // 2) % 2 == 0, (t // 2 + M) % 2 == 1
        x, w, b, lnp, r = _gemv_case(M, K, N, act, ln, bias, res, dtype, seed=100 * M + t)
        _lib().gemv_set_tuning(cols, split)
        try:
            y = _run_gemv(x, w, b, lnp, r, act)
        finally:
            _lib().gemv_set_tuning(0, 0)
        torch.cuda.synchronize()
        what = f"gemv M {M} K {K} N {w.shape[0]} act {act} ln {ln} bias {bias} res {res} cols {cols} split {split}"
        want, kw = D.gemv_ref(x, w, b, lnp, r, act)
        assert y.shape == want.shape and y.dtype == dtype, what
        _record(f"gemv {act}", dtype, R.assert_close(y, want, dtype, **kw, what=what))


# ---------------------------------------------------------------------------------------------------------------- small-M GEMM
SMALLM_M = [1, 2, 3, 15, 16, 17, 32, 33, 64, 65, 127, 128]        # every 16 / 32 / 64 / 128-row bucket and both of its edges
SMALLM_SPLITS = [0, 1, 2, 4, 8]                                    # 0: the heuristic
SMALLM_K = [8, 72, 520, 4104]       # below 64 x split some CTAs of a cluster get no k-block; K % 64 != 0 leaves a TMA zero fill
SMALLM_N = [8, 136, 4104, 50304]


def _gemm_ref(x, w, b):
    xd, wd = R._d(x), R._d(w)
    ref, terms = xd @ wd.t(), xd.abs() @ wd.abs().t()
    if b is not None:
        ref, terms = ref + R._d(b), terms + R._d(b).abs()
    return ref, terms


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("M", SMALLM_M)
def test_gemm_smallm_against_float64(dtype, M):
    """Every (M, split) pair once, K, N and the bias rotating with it."""
    i = SMALLM_M.index(M)
    for j, split in enumerate(SMALLM_SPLITS):
        K, N = SMALLM_K[(i + j) % 4], SMALLM_N[(i + 2 * j + i // 4) % 4]
        bias = (i + j) % 2 == 0
        seed = 1000 * M + 10 * j
        x = _randn(M, K, seed=seed, dtype=dtype)
        w = _randn(N, K, seed=seed + 1, scale=2 * K ** -0.5, dtype=dtype)
        b = _randn(N, seed=seed + 2, scale=0.5, dtype=dtype) if bias else None
        y = _lib().gemm_smallm(x, w, b, split)
        torch.cuda.synchronize()
        ref, terms = _gemm_ref(x, w, b)
        what = f"gemm_smallm M {M} K {K} N {N} split {split} bias {bias}"
        assert y.shape == (M, N) and y.dtype == dtype, what
        _record("gemm_smallm", dtype, R.assert_close(y, ref, dtype, scale=terms, n=K, approx=R.MMA_ACC, what=what))


# ---------------------------------------------------------------------------------------------------------------- router edges
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("rows", [2, 3, 128, 129])
def test_linear_router_edges_against_float64(dtype, rows):
    """At the GEMV / small-M / tiled-GEMM boundaries OF.linear returns the float64 result within the tensor-core GEMM's bound, which
    also covers the GEMV's fp32 chain at this K."""
    K, N = 1032, 1000
    x = _randn(rows, K, seed=rows, dtype=dtype)
    w = _randn(N, K, seed=rows + 1, scale=2 * K ** -0.5, dtype=dtype)
    b = _randn(N, seed=rows + 2, scale=0.5, dtype=dtype)
    with torch.no_grad():
        y = OF.linear(x, w, b)
    torch.cuda.synchronize()
    ref, terms = _gemm_ref(x, w, b)
    assert y.shape == (rows, N) and y.dtype == dtype
    _record("linear", dtype, R.assert_close(y, ref, dtype, scale=terms, n=K, approx=R.MMA_ACC, what=f"linear {rows} rows"))


@pytest.mark.parametrize("dtype", DTYPES)
def test_gemv_fused_at_eight_rows(dtype):
    x, w, b, lnp, r = _gemv_case(8, 1032, 4100, "gelu", True, True, True, dtype, seed=8)
    y = OF.gemv_fused(x, w, b, ln=lnp, residual=r, act="gelu")
    torch.cuda.synchronize()
    want, kw = D.gemv_ref(x, w, b, lnp, r, "gelu")
    _record("gemv gelu", dtype, R.assert_close(y, want, dtype, **kw, what="gemv_fused 8 rows"))
