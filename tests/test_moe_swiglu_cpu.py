"""GPT-MoE with SwiGLU experts (``Model.ffn_activation: swiglu`` with ``moe_configs``) on the CPU path: config rules, the unchanged GELU
experts, the expert FFN against plain torch, the stacked expert parameters and their checkpoint keys, parameter counts, expert parallelism
under gloo and the recipe."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from dist_utils import run_distributed
from helpers import tiny_gpt_config

from paddlefleetx_b200.models.language_model.gpt import model as gpt
from paddlefleetx_b200.models.language_model.moe.grouped_experts import GroupedExperts, reference_grouped_ffn
from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer, MoELayer

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, FFN, E = 128, 128, 3
MOE = ["Model.moe_configs.expert_mode=True", "Model.moe_configs.num_experts=2"]


def _swiglu_ffn(x, w1, b1, w2, b2):
    """Plain-torch SwiGLU FFN from separate gate / up weights."""
    wg, wu, bg, bu = w1[0::2], w1[1::2], b1[0::2], b1[1::2]
    return F.linear(F.silu(F.linear(x, wg, bg)) * F.linear(x, wu, bu), w2, b2)


def _layer(fused, activation="swiglu", seed=3, dtype=None):
    torch.manual_seed(seed)
    ex = [ExpertLayer(H, FFN, activation=activation, dtype=dtype) for _ in range(E)]
    with torch.no_grad():
        for e in ex:
            e.htoh4.bias.normal_(0, 0.5); e.h4toh.bias.normal_(0, 0.5)
    return MoELayer(H, ex, gate={"type": "naive", "top_k": 2}, fused_p2p=fused)


# ---------------------------------------------------------------------------------------------------------------- configuration
def test_swiglu_moe_configs_are_accepted_and_the_other_rules_hold():
    from paddlefleetx_b200.utils import check

    one_expert = ["Model.moe_configs.expert_mode=True"]         # num_experts defaults to 1 and top_k to 2
    cases = [(one_expert, {}, "top_k"),
             (["Model.ffn_activation=swiglu", *one_expert], {}, "top_k"),
             (["Model.ffn_activation=swiglu", *MOE, "Model.moe_configs.top_k=3"], {}, "top_k"),
             (["Model.ffn_activation=relu"], {}, "gelu or swiglu"),
             (["Model.ffn_activation=swiglu", "Compress.Prune.enable=True"], {}, "Compress.Prune"),
             (["Model.ffn_activation=swiglu", *MOE, "Compress.Prune.enable=True"], {}, "Compress.Prune"),
             (["Model.ffn_activation=swiglu", "Model.ffn_hidden_size=100"], {"mp_degree": 8}, "divisible by mp_degree")]
    for ov, dist, msg in cases:
        cfg = tiny_gpt_config(ov, nranks=1)
        cfg.Distributed.update(dist)
        with pytest.raises(ValueError, match=msg):
            check.check_config(cfg)
    assert check.check_config(tiny_gpt_config(["Model.ffn_activation=swiglu"], nranks=1))
    assert check.check_config(tiny_gpt_config(["Model.ffn_activation=swiglu", *MOE], nranks=1))
    assert check.check_config(tiny_gpt_config(["Model.ffn_activation=swiglu", *one_expert, "Distributed.dp_degree=2"], nranks=2))
    with pytest.raises(ValueError, match="ffn_activation"):
        gpt.GPTModel(vocab_size=128, hidden_size=64, num_layers=1, num_attention_heads=4, max_position_embeddings=32, ffn_activation="geglu")
    with pytest.raises(ValueError, match="activation"):
        ExpertLayer(H, FFN, activation="geglu")


def test_swiglu_moe_model_builds_swiglu_experts_of_the_default_width():
    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=128, hidden_size=H, num_layers=2, num_attention_heads=4, max_position_embeddings=32, ffn_activation="swiglu",
                        moe_configs={"expert_mode": True, "num_experts": 2, "gate": "naive", "top_k": 2})
    f = gpt.swiglu_ffn_size(H)
    experts = [m for m in core.modules() if isinstance(m, ExpertLayer)]
    assert len(experts) == 4 and all(ex.activation == "swiglu" for ex in experts)
    assert all(ex.htoh4.weight.shape == (2 * f, H) and ex.h4toh.weight.shape == (H, f) for ex in experts)
    assert all(layer.ffn_activation == "swiglu" and layer.moe_mlp is not None for layer in core.decoder.layers)


# ---------------------------------------------------------------------------------------------------------------- GELU experts unchanged
def _gelu_moe_stats():
    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=128, hidden_size=64, num_layers=2, num_attention_heads=4, ffn_hidden_size=128, max_position_embeddings=32,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0,
                        moe_configs={"expert_mode": True, "num_experts": 2, "gate": "naive", "top_k": 2})
    ids = torch.randint(0, 128, (2, 12), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        out = core(ids)
    out = out[0] if isinstance(out, tuple) else out
    return {"params": {k: [list(v.shape), float(v.double().sum()), float(v.double().abs().sum())] for k, v in core.state_dict().items()},
            "out": [list(out.shape), float(out.double().sum()), float(out.double().abs().sum())] + out.flatten()[:32].double().tolist()}


def test_gelu_moe_model_keeps_its_parameters_keys_and_outputs():
    """A GELU GPT-MoE built from seeded initialisation matches the record taken before SwiGLU experts existed: the same state-dict keys and
    shapes, the same parameter values and the same outputs."""
    with open(os.path.join(ROOT, "tests", "golden", "moe_gelu_cpu.json")) as fh:
        want = json.load(fh)
    got = _gelu_moe_stats()
    assert list(got["params"]) == list(want["params"])
    for k, (shape, s, a) in want["params"].items():
        assert got["params"][k][0] == shape, k
        assert got["params"][k][1:] == pytest.approx([s, a], rel=1e-6, abs=1e-9), k
    assert got["out"][0] == want["out"][0]
    assert got["out"][1:] == pytest.approx(want["out"][1:], rel=1e-5, abs=1e-6)


def test_gelu_expert_default_is_the_gelu_ffn():
    torch.manual_seed(1)
    ex = ExpertLayer(H, FFN)
    assert ex.activation == "gelu" and ex.htoh4.weight.shape == (FFN, H)
    x = torch.randn(10, H)
    want = F.linear(F.gelu(F.linear(x, ex.htoh4.weight, ex.htoh4.bias), approximate="tanh"), ex.h4toh.weight, ex.h4toh.bias)
    torch.testing.assert_close(ex(x), want)


# ---------------------------------------------------------------------------------------------------------------- the SwiGLU expert
def test_swiglu_expert_equals_a_plain_torch_ffn_from_deinterleaved_weights():
    torch.manual_seed(2)
    ex = ExpertLayer(H, FFN, activation="swiglu", dtype=torch.float64)
    with torch.no_grad():
        ex.htoh4.bias.normal_(0, 0.5); ex.h4toh.bias.normal_(0, 0.5)
    assert ex.htoh4.weight.shape == (2 * FFN, H) and ex.h4toh.weight.shape == (H, FFN)
    x = torch.randn(20, H, dtype=torch.float64, requires_grad=True)
    y = ex(x)
    params = [ex.htoh4.weight, ex.htoh4.bias, ex.h4toh.weight, ex.h4toh.bias]
    ref_params = [p.detach().clone().requires_grad_(True) for p in params]
    xr = x.detach().clone().requires_grad_(True)
    want = _swiglu_ffn(xr, *ref_params)
    torch.testing.assert_close(y, want)
    g = torch.randn_like(y)
    y.backward(g)
    want.backward(g)
    torch.testing.assert_close(x.grad, xr.grad)
    for p, r in zip(params, ref_params):
        torch.testing.assert_close(p.grad, r.grad)


# ---------------------------------------------------------------------------------------------------------------- stacked experts
def test_grouped_swiglu_experts_stack_and_round_trip_per_expert_keys():
    plain, grouped = _layer(False), _layer(True, seed=4)
    ge = grouped.grouped
    assert ge is not None and plain.grouped is None and ge.activation == "swiglu"
    assert ge.w1.shape == (E, 2 * FFN, H) and ge.b1.shape == (E, 2 * FFN) and ge.w2.shape == (E, H, FFN) and ge.b2.shape == (E, H)
    assert sorted(plain.state_dict()) == sorted(grouped.state_dict())
    assert "experts.0.htoh4.weight" in grouped.state_dict() and not any(k.startswith("grouped.") for k in grouped.state_dict())
    grouped.load_state_dict(plain.state_dict())
    for k, v in plain.state_dict().items():
        assert torch.equal(v, grouped.state_dict()[k]), k
    assert torch.equal(ge.w1[1], plain.experts[1].htoh4.weight) and torch.equal(ge.w2[2], plain.experts[2].h4toh.weight)
    plain2 = _layer(False, seed=5)
    plain2.load_state_dict(grouped.state_dict())
    assert torch.equal(plain2.experts[2].htoh4.bias, ge.b1[2])
    # the loop path runs on the stacks and lands its gradients in them
    x = torch.randn(40, H)
    y0, y1 = plain(x), grouped(x)
    torch.testing.assert_close(y1, y0)
    y0.square().sum().backward(); y1.square().sum().backward()
    for e in range(E):
        torch.testing.assert_close(ge.w1.grad[e], plain.experts[e].htoh4.weight.grad)
        torch.testing.assert_close(ge.b1.grad[e], plain.experts[e].htoh4.bias.grad)


def test_reference_grouped_ffn_swiglu_form():
    layer = _layer(True, seed=6, dtype=torch.float64)
    ge = layer.grouped
    xs = torch.randn(12, H, dtype=torch.float64)
    seg2 = [0, 5, 5, 0, 8, 4]
    out = reference_grouped_ffn(xs, seg2, ge)
    assert out.dtype == torch.float64
    for e in range(E):
        s, n = seg2[2 * e], seg2[2 * e + 1]
        if n:
            torch.testing.assert_close(out[s:s + n], _swiglu_ffn(xs[s:s + n], ge.w1[e], ge.b1[e], ge.w2[e], ge.b2[e]))
    assert bool((out[5:8] == 0).all())


def test_grouped_path_needs_whole_tiles_of_swiglu_channels_and_one_activation():
    assert GroupedExperts.supported([ExpertLayer(H, 128, activation="swiglu") for _ in range(2)])
    assert not GroupedExperts.supported([ExpertLayer(H, 96, activation="swiglu") for _ in range(2)])      # F % 128 != 0
    assert not GroupedExperts.supported([ExpertLayer(H, 128, activation="swiglu"), ExpertLayer(H, 256)])  # 2F = 256 rows either way
    assert GroupedExperts.supported([ExpertLayer(H, 128) for _ in range(2)])


# ---------------------------------------------------------------------------------------------------------------- parameter counts
def test_parameter_counts():
    from paddlefleetx_b200.models.language_model.language_module import get_model_size
    from paddlefleetx_b200.utils import config as C
    from paddlefleetx_b200.utils.layout_planner import ModelShape

    h, f, layers = 64, 128, 2
    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=128, hidden_size=h, num_layers=layers, num_attention_heads=4, ffn_hidden_size=f, max_position_embeddings=32,
                        ffn_activation="swiglu", moe_configs={"expert_mode": True, "num_experts": 2, "gate": "naive", "top_k": 2})
    per_expert = 3 * h * f + 2 * f + h
    assert all(sum(p.numel() for p in ex.parameters()) == per_expert for ex in core.modules() if isinstance(ex, ExpertLayer))
    n_exp = sum(p.numel() for p in core.parameters() if getattr(p, "is_expert", False))
    assert n_exp == layers * 2 * per_expert
    gelu_core = gpt.GPTModel(vocab_size=128, hidden_size=h, num_layers=layers, num_attention_heads=4, ffn_hidden_size=f, max_position_embeddings=32,
                             moe_configs={"expert_mode": True, "num_experts": 2, "gate": "naive", "top_k": 2})
    assert sum(p.numel() for p in gelu_core.parameters() if getattr(p, "is_expert", False)) == layers * 2 * (2 * h * f + f + h)
    # get_model_size counts one expert FFN per layer, of the model's activation
    v, s = 128, 32
    assert get_model_size(layers, h, v, s, ffn=f, ffn_activation="swiglu") - get_model_size(layers, h, v, s, ffn=f) == layers * (h * f + f)
    cfg = C.get_config(os.path.join(ROOT, "paddlefleetx_b200/configs/nlp/moe/pretrain_moe_345M_swiglu_single_card.yaml"), [], show=False, nranks=1)
    shape = ModelShape.from_config(cfg)
    assert shape.ffn_activation == "swiglu" and shape.ffn1_width == 2 * shape.ffn


# ---------------------------------------------------------------------------------------------------------------- expert parallelism
def test_expert_parallel_swiglu_matches_single():
    run_distributed("moe_swiglu_dist_fns:moe_ep_swiglu_matches_single", 2)


# ---------------------------------------------------------------------------------------------------------------- recipe
def test_recipe_trains_through_the_cli():
    import re
    import subprocess
    import sys

    cfg = os.path.join(ROOT, "paddlefleetx_b200", "configs", "nlp", "moe", "pretrain_moe_345M_swiglu_single_card.yaml")
    ov = ["Global.device=cpu", "Engine.mix_precision.enable=False", "Model.num_layers=2", "Model.hidden_size=64", "Model.num_attention_heads=4",
          "Model.max_position_embeddings=32", "Model.hidden_dropout_prob=0.0", "Model.attention_probs_dropout_prob=0.0", "Model.use_recompute=False",
          "Data.Train.dataset.name=SyntheticGPTDataset", "Data.Train.dataset.max_seq_len=32", "Data.Train.loader.num_workers=0",
          "Global.local_batch_size=2", "Global.micro_batch_size=2", "Engine.max_steps=3", "Engine.logging_freq=1", "Engine.eval_freq=-1",
          "Engine.save_load.save_steps=-1"]
    args = [sys.executable, "tools/train.py", "-c", cfg]
    for item in ov:
        args += ["-o", item]
    p = subprocess.run(args, capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES=""))
    log = p.stdout + p.stderr
    assert p.returncode == 0, log[-3000:]
    losses = [float(x) for x in re.findall(r"loss: ([0-9.]+)", log)]
    assert log.count("[train]") >= 3 and losses and all(l == l for l in losses), log[-1500:]
    # F defaults to 8h/3 rounded up to 256 (256 at h = 64): 2 layers x 2 experts x (3 h F + 2 F + h) expert parameters
    n = re.search(r"MoE: 2 gated layers, ([0-9.]+) M expert parameters", log)
    assert n and float(n.group(1)) == pytest.approx(round(4 * (3 * 64 * 256 + 2 * 256 + 64) / 1e6, 1)), log[-1500:]
