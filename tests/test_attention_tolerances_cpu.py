"""The attention bounds in ``kernel_refs`` are neither too loose nor too tight (CPU only).

For the flash forward / backward, the decode step and the Evoformer attention, in bf16 and fp16 (Evoformer: bf16):
  * the float64 result rounded to the dtype passes, and so does an fp32 emulation of the kernel's algorithm (128-key tiles with an online
    maximum and rescale, P rounded to 16 bits before P V while l sums the fp32 p; 64 x 64 tiles for the backward with P and dS rounded to
    16 bits and dQ reduced per key tile).  ``-s`` prints the emulation's error / bound ratio;
  * a result with a plausible kernel mistake fails, on the inputs the GPU tests use (``R.attention_inputs``: peaked attention, so that a
    mistake moves O by about |O|).
"""
import math

import pytest
import torch

import kernel_refs as R

DTYPES = [torch.bfloat16, torch.float16]
LOG2E = 1.4426950408889634


def _inputs(dtype, B, Sq, Sk, H, D, Hkv=None, seed=0, rising=False):
    return tuple(t.to(dtype) for t in R.attention_inputs(B, Sq, Sk, H, D, Hkv, seed=seed, rising=rising))


def _rejects(got, ref, dtype, kw, what):
    with pytest.raises(AssertionError):
        R.assert_close(got, ref, dtype, what=what, **kw)


def _keep(B, H, Sq, Sk, p, seed=5):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, H, Sq, Sk, generator=g) >= p


def _attn_variant(q, k, v, scale, allowed=None, keep=None, kw=None, kv_map=None):
    """float64 attention with a given allowed-key mask [Sq, Sk], keep factors and K/V head map: the wrong versions are built with this."""
    qh = q.double().transpose(1, 2)
    H = qh.shape[1]
    idx = kv_map if kv_map is not None else torch.arange(H) // (H // k.shape[2])
    kh, vh = k.double()[:, :, idx].transpose(1, 2), v.double()[:, :, idx].transpose(1, 2)
    s = qh @ kh.transpose(-1, -2) * scale
    if allowed is not None:
        s = s.masked_fill(~allowed, -math.inf)
    pi = torch.softmax(s, -1)
    if kw is not None:
        pi = pi * kw
    return (pi @ vh).transpose(1, 2), torch.logsumexp(s, -1)


# ---------------------------------------------------------------------------------------------------------------- fp32 emulations
def _emulate_fwd(q, k, v, scale, dtype, bias=None, keep=None, p=0.0, rescale=True):
    """The flash forward's arithmetic in fp32: -> (out in dtype [B,Sq,H,D], lse fp32 [B,H,Sq]).  ``bias`` (natural units, -inf = masked)
    [.., Sq, Sk]; ``rescale=False`` forgets to rescale O when the row maximum moves (a mistake)."""
    qh = q.float().transpose(1, 2)
    H = qh.shape[1]
    kh = k.float().repeat_interleave(H // k.shape[2], 2).transpose(1, 2)
    vh = v.float().repeat_interleave(H // v.shape[2], 2).transpose(1, 2)
    c = torch.tensor(scale * LOG2E, dtype=torch.float32)
    z = (qh @ kh.transpose(-1, -2)) * c
    if bias is not None:
        z = z + (bias.float() * LOG2E if torch.is_tensor(bias) else bias)
    Sk = z.shape[-1]
    m = torch.full(z.shape[:-1] + (1,), -math.inf)
    l = torch.zeros_like(m)
    o = torch.zeros(qh.shape[:-1] + (vh.shape[-1],))
    for t0 in range(0, Sk, 128):
        zt = z[..., t0:t0 + 128]
        m_new = torch.maximum(m, zt.amax(-1, keepdim=True))
        f = torch.where(m == -math.inf, torch.zeros_like(m), torch.exp2(m - m_new))
        m_use = torch.where(m_new == -math.inf, torch.zeros_like(m_new), m_new)
        pt = torch.exp2(zt - m_use)
        l = l * f + pt.sum(-1, keepdim=True)
        if keep is not None:
            pt = pt * keep[..., t0:t0 + 128]
        o = (o * f if rescale else o) + pt.to(dtype).float() @ vh[:, :, t0:t0 + 128]
        m = m_new
    inv_keep = torch.tensor(1.0 / (1.0 - p), dtype=torch.float32)
    out = torch.where(l > 0, o * (inv_keep / l), torch.zeros_like(o))
    lse = torch.where(l > 0, (m + torch.log2(l)) * math.log(2.0), torch.full_like(l, -math.inf))
    return out.to(dtype).transpose(1, 2), lse.squeeze(-1)


def _emulate_bwd(q, k, v, out, dout, lse, scale, dtype, bias=None, keep=None, p=0.0):
    """The flash backward's arithmetic in fp32 over 64-key x 64-query tiles: -> (dq, dk, dv) in dtype (dk / dv summed over groups)."""
    qh = q.float().transpose(1, 2)
    H, Hkv = qh.shape[1], k.shape[2]
    kh = k.float().repeat_interleave(H // Hkv, 2).transpose(1, 2)
    vh = v.float().repeat_interleave(H // Hkv, 2).transpose(1, 2)
    doh, oh = dout.float().transpose(1, 2), out.float().transpose(1, 2)
    delta = (doh * oh).sum(-1, keepdim=True)
    lse2 = lse.unsqueeze(-1) * torch.tensor(LOG2E, dtype=torch.float32)
    c = torch.tensor(scale * LOG2E, dtype=torch.float32)
    z = (qh @ kh.transpose(-1, -2)) * c
    if bias is not None:
        z = z + bias.float() * LOG2E
    P = torch.exp2(z - lse2) * scale
    inv_keep = 1.0 / (1.0 - p)
    dP = doh @ vh.transpose(-1, -2)
    kf = torch.ones_like(P) if keep is None else keep.float()
    pd = (P * (inv_keep / scale) * kf).to(dtype).float()
    dsw = (P * (dP * inv_keep * kf - delta)).to(dtype).float()
    Sq, Sk = P.shape[-2], P.shape[-1]
    dq = torch.zeros_like(qh)
    for k0 in range(0, Sk, 64):
        dq = dq + dsw[..., k0:k0 + 64] @ kh[:, :, k0:k0 + 64]
    dk, dv = torch.zeros_like(kh), torch.zeros_like(vh)
    for q0 in range(0, Sq, 64):
        dk = dk + dsw[:, :, q0:q0 + 64].transpose(-1, -2) @ qh[:, :, q0:q0 + 64]
        dv = dv + pd[:, :, q0:q0 + 64].transpose(-1, -2) @ doh[:, :, q0:q0 + 64]
    B, _, _, D = dk.shape
    dk, dv = (t.reshape(B, Hkv, H // Hkv, Sk, D).sum(2) for t in (dk, dv))
    return tuple(t.transpose(1, 2).to(dtype) for t in (dq, dk, dv))


def _causal_bias(Sq, Sk):
    return torch.zeros(Sq, Sk).masked_fill(~R.causal_mask(Sq, Sk), -math.inf)


# ---------------------------------------------------------------------------------------------------------------- flash forward
FWD_SHAPES = [(2, 1, 300, 3, 64, True), (2, 63, 63, 3, 128, False), (2, 65, 65, 3, 64, True), (2, 127, 129, 3, 128, False),
              (2, 129, 257, 3, 64, True), (2, 200, 1000, 3, 128, True), (1, 1000, 1000, 2, 64, True)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", FWD_SHAPES, ids=lambda s: "B{}_Sq{}_Sk{}_H{}_D{}_{}".format(*s[:5], "causal" if s[5] else "full"))
def test_flash_forward_correct_results_pass(dtype, shape):
    B, Sq, Sk, H, D, causal = shape
    q, k, v, _ = _inputs(dtype, B, Sq, Sk, H, D, rising=Sq > 1000)
    scale = D ** -0.5
    ref, lse = R.attention(q, k, v, scale, causal)
    okw, lkw = R.attention_bounds(q, k, v, scale, causal, dtype)
    R.assert_close(ref.to(dtype), ref, dtype, **okw)
    out, lse_e = _emulate_fwd(q, k, v, scale, dtype, bias=_causal_bias(Sq, Sk) if causal else None)
    r = R.assert_close(out, ref, dtype, what="emulated out", **okw)
    rl = R.assert_close(lse_e, lse, torch.float32, what="emulated lse", **lkw)
    print(f"flash fwd emulation {dtype} {shape}: out {r:.3f}, lse {rl:.3f}")
    assert r < 0.5 and rl < 0.5


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_forward_rejects_key_tile_mistakes(dtype):
    B, Sq, Sk, H, D = 2, 200, 1000, 3, 64
    q, k, v, _ = _inputs(dtype, B, Sq, Sk, H, D)
    scale = D ** -0.5
    ref, _ = R.attention(q, k, v, scale, True)
    okw, _ = R.attention_bounds(q, k, v, scale, True, dtype)
    causal = R.causal_mask(Sq, Sk)
    cols = torch.arange(Sk)[None, :]
    rows = torch.arange(Sq)[:, None]
    wrong = {
        "skipped tile": causal & ~((cols >= 128) & (cols < 256)),
        "ragged last tile dropped": causal & (cols < (Sk // 128) * 128),
        "diagonal one key late": cols <= rows + (Sk - Sq) + 1,
        "diagonal one key early": cols <= rows + (Sk - Sq) - 1,
        "top-left causal": cols <= rows,
    }
    for what, allowed in wrong.items():
        allowed = allowed | (cols == 0)              # keep every row non-empty
        _rejects(_attn_variant(q, k, v, scale, allowed)[0].to(dtype), ref, dtype, okw, what)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Sq,Sk", [(63, 63), (129, 257)])
def test_flash_forward_rejects_an_off_by_one_diagonal_on_short_rows(dtype, Sq, Sk):
    q, k, v, _ = _inputs(dtype, 2, Sq, Sk, 3, 64)
    ref, _ = R.attention(q, k, v, 0.125, True)
    okw, _ = R.attention_bounds(q, k, v, 0.125, True, dtype)
    cols, rows = torch.arange(Sk)[None, :], torch.arange(Sq)[:, None]
    _rejects(_attn_variant(q, k, v, 0.125, cols <= rows + (Sk - Sq) + 1)[0].to(dtype), ref, dtype, okw, "diagonal late")
    _rejects(_attn_variant(q, k, v, 0.125, cols <= rows)[0].to(dtype) if Sq != Sk else
             _attn_variant(q, k, v, 0.125, (cols <= rows - 1) | (cols == 0))[0].to(dtype), ref, dtype, okw, "diagonal early")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Sq,Sk,causal", [(129, 257, True), (1000, 1000, True), (4096, 4096, True)])
def test_flash_forward_rejects_a_missing_rescale(dtype, Sq, Sk, causal):
    B, H = 1, 1
    q, k, v, _ = _inputs(dtype, B, Sq, Sk, H, 64, rising=True)
    ref, _ = R.attention(q, k, v, 0.125, causal)
    okw, _ = R.attention_bounds(q, k, v, 0.125, causal, dtype)
    bias = _causal_bias(Sq, Sk)
    good, _ = _emulate_fwd(q, k, v, 0.125, dtype, bias=bias)
    r = R.assert_close(good, ref, dtype, **okw)
    print(f"flash fwd emulation, rising rows {dtype} {Sq}x{Sk}: {r:.3f}")
    _rejects(_emulate_fwd(q, k, v, 0.125, dtype, bias=bias, rescale=False)[0], ref, dtype, okw, "no rescale")


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_lse_rejects_log2_units_and_a_missing_scale(dtype):
    q, k, v, _ = _inputs(dtype, 2, 127, 129, 3, 128)
    scale = 128 ** -0.5
    _, lse = R.attention(q, k, v, scale, False)
    _, lkw = R.attention_bounds(q, k, v, scale, False, dtype)
    R.assert_close(lse.float(), lse, torch.float32, **lkw)
    _rejects(lse * LOG2E, lse, torch.float32, lkw, "log2 lse")
    _rejects(_attn_variant(q, k, v, 1.0)[1], lse, torch.float32, lkw, "unscaled lse")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_flash_dropout_rejects_unscaled_or_foreign_masks(dtype, p):
    B, Sq, Sk, H, D = 2, 200, 1000, 3, 64
    q, k, v, do = _inputs(dtype, B, Sq, Sk, H, D)
    keep = _keep(B, H, Sq, Sk, p)
    ref, _ = R.attention(q, k, v, 0.125, True, keep, p)
    okw, _ = R.attention_bounds(q, k, v, 0.125, True, dtype, keep, p)
    R.assert_close(ref.to(dtype), ref, dtype, **okw)
    out, _ = _emulate_fwd(q, k, v, 0.125, dtype, bias=_causal_bias(Sq, Sk), keep=keep, p=p)
    print(f"flash fwd emulation, dropout {p} {dtype}: {R.assert_close(out, ref, dtype, **okw):.3f}")
    causal = R.causal_mask(Sq, Sk)
    _rejects(_attn_variant(q, k, v, 0.125, causal, kw=keep.double())[0].to(dtype), ref, dtype, okw, "no 1/(1-p)")
    foreign = keep.reshape(B * H, Sq, Sk).roll(1, 0).reshape(B, H, Sq, Sk)
    _rejects(_attn_variant(q, k, v, 0.125, causal, kw=foreign.double() / (1 - p))[0].to(dtype), ref, dtype, okw, "neighbouring mask")
    # the backward with the same two mistakes
    grads = R.attention_bwd(q, k, v, do, 0.125, True, keep, p)
    bkw = R.attention_bwd_bounds(q, k, v, do, 0.125, True, dtype, keep, p)
    for wrong_keep, wrong_p in ((keep, 0.0), (foreign, p)):
        wrong = R.attention_bwd(q, k, v, do, 0.125, True, wrong_keep, wrong_p)
        assert any(not R.error_ratio(w.to(dtype), g, dtype, **kw) <= 1 for w, g, kw in zip(wrong, grads, bkw))


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_gqa_rejects_modulo_head_mapping(dtype):
    B, Sq, Sk, H, Hkv, D = 2, 65, 65, 4, 2, 64
    q, k, v, do = _inputs(dtype, B, Sq, Sk, H, D, Hkv)
    ref, _ = R.attention(q, k, v, 0.125, True)
    okw, _ = R.attention_bounds(q, k, v, 0.125, True, dtype)
    out, _ = _emulate_fwd(q, k, v, 0.125, dtype, bias=_causal_bias(Sq, Sk))
    R.assert_close(out, ref, dtype, **okw)
    _rejects(_attn_variant(q, k, v, 0.125, R.causal_mask(Sq, Sk), kv_map=torch.arange(H) % Hkv)[0].to(dtype), ref, dtype, okw, "h % Hkv")


# ---------------------------------------------------------------------------------------------------------------- flash backward
BWD_SHAPES = [(2, 1, 1, 3, 64, False, 3), (2, 63, 63, 3, 128, True, 3), (2, 127, 129, 3, 64, False, 3), (2, 129, 257, 4, 64, True, 2),
              (1, 200, 1000, 2, 128, True, 2)]


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("shape", BWD_SHAPES, ids=lambda s: "B{}_Sq{}_Sk{}_H{}_D{}_{}_Hkv{}".format(*s[:5], "causal" if s[5] else "full", s[6]))
def test_flash_backward_correct_results_pass(dtype, shape):
    B, Sq, Sk, H, D, causal, Hkv = shape
    q, k, v, do = _inputs(dtype, B, Sq, Sk, H, D, Hkv)
    scale = D ** -0.5
    grads = R.attention_bwd(q, k, v, do, scale, causal)
    bkw = R.attention_bwd_bounds(q, k, v, do, scale, causal, dtype)
    bias = _causal_bias(Sq, Sk) if causal else None
    out, lse = _emulate_fwd(q, k, v, scale, dtype, bias=bias)
    emu = _emulate_bwd(q, k, v, out, do, lse, scale, dtype, bias=bias)
    ratios = []
    for name, g, e, kw in zip(("dq", "dk", "dv"), grads, emu, bkw):
        R.assert_close(g.to(dtype), g, dtype, what=name, **kw)
        ratios.append(R.assert_close(e, g, dtype, what="emulated " + name, **kw))
    print(f"flash bwd emulation {dtype} {shape}: dq {ratios[0]:.3f} dk {ratios[1]:.3f} dv {ratios[2]:.3f}")
    assert max(ratios) < 0.5


@pytest.mark.parametrize("dtype", DTYPES)
def test_flash_backward_rejects_key_tile_and_diagonal_mistakes(dtype):
    B, Sq, Sk, H, D = 1, 200, 1000, 2, 64
    q, k, v, do = _inputs(dtype, B, Sq, Sk, H, D)
    grads = R.attention_bwd(q, k, v, do, 0.125, True)
    bkw = R.attention_bwd_bounds(q, k, v, do, 0.125, True, dtype)
    cols, rows = torch.arange(Sk)[None, :], torch.arange(Sq)[:, None]
    causal = R.causal_mask(Sq, Sk)
    for what, allowed in {"skipped tile": causal & ~((cols >= 128) & (cols < 192)), "diagonal late": cols <= rows + (Sk - Sq) + 1,
                          "top-left": (cols <= rows) | (cols == 0)}.items():
        qd, kd, vd = (t.double().requires_grad_(True) for t in (q, k, v))
        out = _attn_variant(qd, kd, vd, 0.125, allowed)[0]
        wrong = torch.autograd.grad(out, (qd, kd, vd), do.double())
        assert any(not R.error_ratio(w.to(dtype), g, dtype, **kw) <= 1 for w, g, kw in zip(wrong, grads, bkw)), what


# ---------------------------------------------------------------------------------------------------------------- decode
def _decode_case(dtype, B, Lmax, H, Hkv, D, seed=0):
    q, k, v, _ = R.attention_inputs(B, 1, Lmax, H, D, Hkv, seed=seed)
    return q.to(dtype), k.to(dtype), v.to(dtype)


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("Lmax,L,D,G", [(1, 1, 64, 1), (9, 7, 128, 4), (136, 136, 64, 8), (1000, 977, 128, 1), (4097, 4097, 64, 4)])
def test_decode_correct_results_pass_and_padding_is_honoured(dtype, Lmax, L, D, G):
    B, Hkv = 2, 2
    q, k, v = _decode_case(dtype, B, Lmax, Hkv * G, Hkv, D)
    mask = torch.zeros(B, Lmax)
    mask[1, : Lmax // 3] = -math.inf                    # left padding of the second row
    mask = mask.to(dtype)
    ref = R.attention_decode(q, k, v, mask, L, D ** -0.5)
    kw = R.attention_decode_bound(q, k, v, mask, L, D ** -0.5)
    R.assert_close(ref.to(dtype), ref, dtype, **kw)
    if Lmax // 3:
        unpadded = R.attention_decode(q, k, v, None, L, D ** -0.5)
        _rejects(unpadded.to(dtype), ref, dtype, kw, "padding ignored")
    if L < Lmax:
        _rejects(R.attention_decode(q, k, v, mask, Lmax, D ** -0.5).to(dtype), ref, dtype, kw, "keys past L")


def test_decode_all_masked_row_returns_zero():
    q, k, v = _decode_case(torch.bfloat16, 1, 9, 2, 2, 64)
    out = R.attention_decode(q, k, v, torch.full((1, 9), -math.inf), 9, 0.125)
    assert torch.equal(out, torch.zeros_like(out))


def _append(cache, new, pos):
    c = cache.clone()
    c[:, pos] = new
    return c


@pytest.mark.parametrize("dtype", DTYPES)
def test_decode_packed_rejects_a_missing_or_misplaced_append(dtype):
    B, Lmax, Hkv, G, D, pos = 2, 136, 2, 4, 128, 70
    q, k, v = _decode_case(dtype, B, Lmax, Hkv * G, Hkv, D)
    k_new, v_new = R.decode_new_kv(q, Hkv, seed=3)
    k_new, v_new = k_new.to(dtype), v_new.to(dtype)
    mask = torch.zeros(B, Lmax)
    mask[:, pos + 1:] = -1e4                             # cache rows not written yet
    mask = mask.to(dtype)
    ref = R.attention_decode(q, _append(k, k_new, pos), _append(v, v_new, pos), mask, Lmax, D ** -0.5)
    kw = R.attention_decode_bound(q, _append(k, k_new, pos), _append(v, v_new, pos), mask, Lmax, D ** -0.5)
    R.assert_close(ref.to(dtype), ref, dtype, **kw)
    _rejects(R.attention_decode(q, k, v, mask, Lmax, D ** -0.5).to(dtype), ref, dtype, kw, "not appended")
    _rejects(R.attention_decode(q, _append(k, k_new, pos + 1), _append(v, v_new, pos + 1), mask, Lmax, D ** -0.5).to(dtype), ref, dtype, kw,
             "appended at write_idx + 1")


# ---------------------------------------------------------------------------------------------------------------- Evoformer
B16 = torch.bfloat16


def _evo_case(G, Sq, Sk, H, gpp, mask=True, pair=True, gate=True, seed=0):
    return [t if t is None else t.to(dt) for t, dt in zip(R.evoformer_inputs(G, Sq, Sk, H, gpp, mask, pair, gate, seed=seed),
                                                          (B16, B16, B16, torch.float32, B16, B16, B16))]


def _emulate_evo(q, k, v, mb, pb, gate, gpp, scale):
    G, Sq, H, _ = q.shape
    bias = torch.zeros(G, H, Sq, k.shape[1])
    if mb is not None:
        bias = bias + mb.float()[:, None, None, :]
    if pb is not None:
        bias = bias + pb.float().repeat_interleave(gpp, 0)
    out, _ = _emulate_fwd(q, k, v, scale, B16, bias=bias)
    if gate is None:
        return out
    # the kernel gates the fp32 O before its one rounding; the rounded ungated O is within the same budget
    return (out.float() * (1.0 / (1.0 + torch.exp(-gate.float())))).to(B16)


@pytest.mark.parametrize("shape", [(4, 1, 1, 2, 1), (6, 63, 65, 4, 3), (4, 129, 257, 8, 2), (2, 300, 77, 2, 1), (6, 96, 96, 4, 6)])
def test_evoformer_correct_results_pass(shape):
    G, Sq, Sk, H, gpp = shape
    q, k, v, mb, pb, gate, do = _evo_case(G, Sq, Sk, H, gpp)
    ref = R.evoformer(q, k, v, mb, pb, gate, gpp, 32 ** -0.5)
    grads = R.evoformer_bwd(q, k, v, mb, pb, gate, gpp, 32 ** -0.5, do)
    kws = R.evoformer_bounds(q, k, v, mb, pb, gate, gpp, 32 ** -0.5, do)
    R.assert_close(ref.to(B16), ref, B16, **kws[0])
    r = R.assert_close(_emulate_evo(q, k, v, mb, pb, gate, gpp, 32 ** -0.5), ref, B16, what="emulated evoformer", **kws[0])
    print(f"evoformer fwd emulation {shape}: {r:.3f}")
    for name, g, kw in zip(("dq", "dk", "dv", "dgate"), grads[:4], kws[1:5]):
        R.assert_close(g.to(B16), g, B16, what=name, **kw)
    R.assert_close(grads[4].float(), grads[4], torch.float32, what="dpair", **kws[5])


def test_evoformer_rejects_wrong_pair_bias_indexing():
    G, Sq, Sk, H, gpp = 4, 96, 96, 4, 2
    q, k, v, mb, pb, gate, _ = _evo_case(G, Sq, Sk, H, gpp)
    ref = R.evoformer(q, k, v, mb, pb, gate, gpp, 32 ** -0.5)
    kw = R.evoformer_bounds(q, k, v, mb, pb, gate, gpp, 32 ** -0.5)
    wrong = R.evoformer(q, k, v, mb, pb[torch.arange(G) % gpp], gate, 1, 32 ** -0.5)          # group g reads bias g % gpp
    _rejects(wrong.to(B16), ref, B16, kw, "pair bias g % gpp")
    _rejects(R.evoformer(q, k, v, mb, pb.transpose(-1, -2), gate, gpp, 32 ** -0.5).to(B16), ref, B16, kw, "pair bias [k, q]")


def test_evoformer_rejects_gate_gradient_mistakes():
    G, Sq, Sk, H, gpp = 2, 63, 65, 4, 1
    q, k, v, mb, pb, gate, do = _evo_case(G, Sq, Sk, H, gpp)
    scale = 32 ** -0.5
    grads = R.evoformer_bwd(q, k, v, mb, pb, gate, gpp, scale, do)
    kws = R.evoformer_bounds(q, k, v, mb, pb, gate, gpp, scale, do)
    sig = torch.sigmoid(gate.double())
    o = R.evoformer(q, k, v, mb, pb, None, gpp, scale)
    _rejects((do.double() * o * sig).to(B16), grads[3], B16, kws[4], "dgate with sig")
    # delta = rowsum(dOut o out) formed without the gate, rowsum(dOut o O), in dS = P (dP - delta) with dP = (dOut sig) V^T
    pi = torch.softmax(R._evo_logits(q, k, mb, pb, gpp, scale), -1)
    dop = (do.double() * sig).transpose(1, 2)
    dP = dop @ v.double().transpose(1, 2).transpose(-1, -2)
    delta_bad = (do.double() * o).sum(-1).transpose(1, 2).unsqueeze(-1)
    dq_bad = ((pi * (dP - delta_bad)) @ k.double().transpose(1, 2) * scale).transpose(1, 2)
    _rejects(dq_bad.to(B16), grads[0], B16, kws[1], "delta without the gate")


def test_evoformer_fully_masked_groups_follow_the_uniform_contract():
    G, Sq, Sk, H, gpp = 4, 63, 77, 2, 2
    q, k, v, mb, pb, gate, do = _evo_case(G, Sq, Sk, H, gpp)
    mb[1] = -1e9
    uni = torch.tensor([False, True, False, False])
    out = R.evoformer(q, k, v, mb, pb, gate, gpp, 32 ** -0.5, uniform=uni)
    mean = v.double()[1].mean(0) * torch.sigmoid(gate.double()[1])
    assert torch.allclose(out[1], mean.expand_as(out[1]), rtol=1e-12, atol=1e-12)
    kws = R.evoformer_bounds(q, k, v, mb, pb, gate, gpp, 32 ** -0.5, do, uniform=uni)
    R.assert_close(out.to(B16), out, B16, **kws[0])
    # the float64 result that keeps the scores is not the fp32 contract
    _rejects(R.evoformer(q, k, v, mb, pb, gate, gpp, 32 ** -0.5).to(B16), out, B16, kws[0], "scores kept")
    # a backward whose probabilities are Sk times too large on the masked group
    grads = R.evoformer_bwd(q, k, v, mb, pb, gate, gpp, 32 ** -0.5, do, uniform=uni)
    dv_bad = grads[2].clone()
    dv_bad[1] *= Sk
    _rejects(dv_bad.to(B16), grads[2], B16, kws[3], "dv Sk times")


class _Ctx:
    pass


@pytest.mark.parametrize("shape", [(6, 129, 77, 4, 3), (4, 63, 65, 2, 1)])
def test_evoformer_chunked_backward_within_the_kernel_bounds(shape):
    """The chunked PyTorch backward of ``evoformer_attention`` (CPU, the path also taken for a mask-bias gradient) meets the bounds the
    kernel meets.  Its logits must be fp32 products: a bf16 q.k moves every probability by about 1 % and dgate out of its bound."""
    from paddlefleetx_b200.ops import evoformer_attention as EA

    G, Sq, Sk, H, gpp = shape
    q, k, v, mb, pb, gate, do = _evo_case(G, Sq, Sk, H, gpp)
    scale = 32 ** -0.5
    ctx = _Ctx()
    e = q.new_empty(0)
    ctx.saved_tensors = (q, k, v, mb, pb, gate, e, EA.reference(q, k, v, mb, pb, gate, gpp, scale).to(B16))
    ctx.flags, ctx.gpp, ctx.scale = (True, True, True), gpp, scale
    ctx.bias_dtypes = (mb.dtype, pb.dtype)
    ctx.needs_input_grad = (True, True, True, False, True, True, False, False)
    dq, dk, dv, _, dpair, dgate, _, _ = EA._EvoAttnFn.backward(ctx, do)
    ref = R.evoformer_bwd(q, k, v, mb, pb, gate, gpp, scale, do)
    kws = R.evoformer_bounds(q, k, v, mb, pb, gate, gpp, scale, do)
    for name, got, want, kw in zip(("dq", "dk", "dv", "dgate", "dpair"), (dq, dk, dv, dgate, dpair), ref, kws[1:]):
        print(f"evoformer chunked backward {shape} {name}: {R.assert_close(got, want, B16, what=name, **kw):.3f}")
