"""The block schedule of parallel/ring_attention.py replayed inside ONE process (every "rank" is a zigzag slice of the same tensors, the ring
hop is a list rotation): checks the block plan, the online-softmax merge and the backward-from-final-statistics against attention over the whole
sequence.  On CPU it runs the PyTorch block; the ``gpu`` variant runs the same schedule through the wgmma flash kernels in bf16 — the block
shapes a ring produces (``q x k[:half]``, ``q[half:] x k``, unmasked, statistics of the FULL row) are shapes no other test feeds them."""
import pytest
import torch

from paddlefleetx_b200.parallel import ring_attention as R


def _replay(q, k, v, dout, c, causal, scale):
    """Returns (out, dq, dk, dv) over the full sequence, computed rank by rank with the ring's block functions."""
    loc = [[R.zigzag_slice(t, c, r) for t in (q, k, v, dout)] for r in range(c)]
    half = loc[0][0].shape[1] // 2
    outs, lses = [], []
    for r in range(c):
        out = lse = None
        for step in range(c):
            src = (r - step) % c
            qs, ks, bc = R._block_plan(causal, r, src, half)
            o_b, l_b = R._block_fwd(loc[r][0][:, qs], loc[src][1][:, ks], loc[src][2][:, ks], bc, scale, 0.0, 0)
            if qs == slice(None):
                out, lse = R._merge(out, lse, o_b, l_b)
            else:
                o2, l2 = R._merge(out[:, qs], lse[:, :, qs], o_b, l_b)
                out, lse = torch.cat([out[:, :half], o2], 1), torch.cat([lse[:, :, :half], l2], 2)
        outs.append(out.to(q.dtype))
        lses.append(lse)
    md = R._math_dtype(q)
    dqs = [torch.zeros(loc[r][0].shape, dtype=md, device=q.device) for r in range(c)]
    dks = [torch.zeros(loc[r][1].shape, dtype=md, device=q.device) for r in range(c)]
    dvs = [torch.zeros(loc[r][2].shape, dtype=md, device=q.device) for r in range(c)]
    for r in range(c):
        for step in range(c):
            src = (r - step) % c
            qs, ks, bc = R._block_plan(causal, r, src, half)
            gq, gk, gv = R._block_bwd(loc[r][0][:, qs], loc[src][1][:, ks], loc[src][2][:, ks], outs[r][:, qs], loc[r][3][:, qs], lses[r][:, :, qs], bc,
                                      scale, 0.0, 0)
            dqs[r][:, qs] += gq.to(md)
            dks[src][:, ks] += gk.to(md)
            dvs[src][:, ks] += gv.to(md)
    return tuple(R.zigzag_merge(x) for x in (outs, dqs, dks, dvs))


def _reference(q, k, v, dout, causal, scale):
    qf, kf, vf = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    o = torch.nn.functional.scaled_dot_product_attention(qf.transpose(1, 2), kf.transpose(1, 2), vf.transpose(1, 2), is_causal=causal, scale=scale).transpose(1, 2)
    (o * dout.double()).sum().backward()
    return o.detach(), qf.grad, kf.grad, vf.grad


@pytest.mark.parametrize("c", [2, 3])
@pytest.mark.parametrize("causal", [True, False])
def test_block_schedule_reproduces_full_attention_on_cpu(c, causal):
    torch.manual_seed(1)
    b, s, h, d = 2, 4 * 2 * c, 2, 8
    q, k, v, do = (torch.randn(b, s, h, d) for _ in range(4))
    got = _replay(q, k, v, do, c, causal, d ** -0.5)
    for a, r_ in zip(got, _reference(q, k, v, do, causal, d ** -0.5)):
        torch.testing.assert_close(a.double(), r_, atol=2e-5, rtol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("c,s,d", [(2, 1024, 128), (4, 2048, 64)])
def test_block_schedule_on_the_flash_kernels(c, s, d):
    torch.manual_seed(2)
    b, h = 2, 4
    q, k, v = (torch.randn(b, s, h, d, device="cuda").bfloat16() for _ in range(3))
    do = (torch.randn(b, s, h, d, device="cuda") * 0.5).bfloat16()
    loc = R.zigzag_slice(q, c, 1)
    assert R.ATT._native_ok(loc, loc, loc, None, True, True) and R.ATT._native_ok(loc[:, loc.shape[1] // 2:], loc, loc, None, False, True), \
        "the ring's block shapes must reach the native kernels on a GPU box"
    got = _replay(q, k, v, do, c, True, d ** -0.5)
    ref = _reference(q, k, v, do, True, d ** -0.5)
    for name, a, r_ in zip(("out", "dq", "dk", "dv"), got, ref):
        err = float((a.double() - r_).norm() / r_.norm())
        assert err < 2e-2, (name, err)
