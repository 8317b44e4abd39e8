"""Functions run on each rank of a gloo job by ``dist_utils.run_distributed`` for the SwiGLU MoE tests (``tests/test_moe_swiglu_cpu.py``)."""
import torch


def moe_ep_swiglu_matches_single(rank, world):
    """Expert-parallel MoELayer with SwiGLU experts (2 ranks x 2 experts) == single-process layer with 4 experts on the concatenated batch."""
    from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer, MoELayer
    from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

    hcg = HybridCommunicateGroup(dp=world)
    d, f, e_local, n_tok = 16, 24, 2, 24
    gate = {"type": "naive", "top_k": 2}
    torch.manual_seed(5)
    full = MoELayer(d, [ExpertLayer(d, f, activation="swiglu") for _ in range(e_local * world)], gate=gate, moe_group=None)
    x_all = torch.randn(world * n_tok, d)
    torch.manual_seed(99)
    ep = MoELayer(d, [ExpertLayer(d, f, activation="swiglu") for _ in range(e_local)], gate=gate, moe_group=hcg.get_moe_group())
    with torch.no_grad():
        for e, ex in enumerate(full.experts):      # non-zero gate / up biases, the same on every rank
            ex.htoh4.bias.normal_(0, 0.5, generator=torch.Generator().manual_seed(e))
        ep.gate.gate.weight.copy_(full.gate.gate.weight); ep.gate.gate.bias.copy_(full.gate.gate.bias)
        for i in range(e_local):
            ep.experts[i].load_state_dict(full.experts[rank * e_local + i].state_dict())
    assert ep.experts[0].htoh4.weight.shape == (2 * f, d) and ep.experts[0].h4toh.weight.shape == (d, f)
    mine = slice(rank * n_tok, (rank + 1) * n_tok)
    x = x_all[mine].clone().requires_grad_(True)
    xa = x_all.clone().requires_grad_(True)
    y, ya = ep(x), full(xa)
    assert torch.allclose(y, ya[mine], atol=1e-5), (y - ya[mine]).abs().max()
    g_all = torch.randn(world * n_tok, d, generator=torch.Generator().manual_seed(1))
    y.backward(g_all[mine])
    ya.backward(g_all)
    assert torch.allclose(x.grad, xa.grad[mine], atol=1e-5)
    for i in range(e_local):
        for (n1, p1), (n2, p2) in zip(ep.experts[i].named_parameters(), full.experts[rank * e_local + i].named_parameters()):
            assert n1 == n2 and torch.allclose(p1.grad, p2.grad, atol=1e-5), (i, n1)
