"""SwiGLU feed-forward for GPT (``Model.ffn_activation: swiglu``) on the CPU path: the float64 references and their bounds, the
pair-interleaved layout, parameter counts, config validation, tensor / sequence / pipeline parallelism, checkpoint resharding, decoding and
the recipe."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import kernel_refs as R
import swiglu_refs as S
from dist_utils import run_distributed
from helpers import synthetic_batches, tiny_gpt_config

from paddlefleetx_b200.models.language_model.gpt import model as gpt
from paddlefleetx_b200.ops import functional as OF

HIDDEN, FFN = 64, 96


def _core(seed=0, **kw):
    torch.manual_seed(seed)
    return gpt.GPTModel(vocab_size=128, hidden_size=HIDDEN, num_layers=2, num_attention_heads=4, max_position_embeddings=64,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, **kw)


def _ids(b=2, s=12, seed=1):
    return torch.randint(0, 128, (b, s), generator=torch.Generator().manual_seed(seed))


# ---------------------------------------------------------------------------------------------------------------- references and bounds
def _inputs(dtype, rows=64, f=72, seed=0):
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(rows, 2 * f, generator=g) * 2.0).to(dtype)
    z[0, 0:8:2] = torch.tensor([30.0, -30.0, 90.0, -90.0])           # saturated gates
    bias = (torch.randn(2 * f, generator=g) * 0.5).to(dtype)
    dh = torch.randn(rows, f, generator=g).to(dtype)
    return z, bias, dh


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_rounded_reference_passes_and_each_mistake_fails(dtype):
    z, bias, dh = _inputs(dtype)
    f = z.shape[-1] // 2
    ref, kw = S.swiglu(z, bias), S.swiglu_bound(z, bias)
    R.assert_close(ref.to(dtype), ref, dtype, **kw)
    zb = R._d(z) + R._d(bias)
    wrong = {
        "gate and up swapped": F.silu(zb[:, 1::2]) * zb[:, 0::2],
        "[gate; up] halves instead of pairs": F.silu(zb[:, :f]) * zb[:, f:],
        "bias missing on the up half": S.swiglu(z, torch.stack([bias[0::2], torch.zeros_like(bias[1::2])], -1).reshape(-1)),
        "sigmoid in place of silu": torch.sigmoid(zb[:, 0::2]) * zb[:, 1::2],
    }
    for what, got in wrong.items():
        assert R.error_ratio(got.to(dtype), ref, dtype, **kw) > 1.0, what

    gref, gkw = S.swiglu_grad(dh, z, bias), S.swiglu_bound(z, bias, dh)
    R.assert_close(gref.to(dtype), gref, dtype, **gkw)
    a, b = S.split_pairs(z, bias)
    s = torch.sigmoid(a)
    no_term = gref.clone()
    no_term[:, 0::2] = R._d(dh) * b * s                               # d silu(a) / da without the a (1 - s) term
    assert R.error_ratio(no_term.to(dtype), gref, dtype, **gkw) > 1.0
    # float64 autograd of the plain expression agrees with the closed-form gradient
    zd = R._d(z).clone().requires_grad_(True)
    hd = S.swiglu(zd, bias)
    torch.testing.assert_close(torch.autograd.grad(hd, zd, R._d(dh))[0], gref)


def test_saturated_gates_stay_finite_in_the_torch_path():
    z = torch.tensor([[1e4, 2.0, -1e4, 2.0, 90.0, -1.0, -90.0, 3.0]] * 2, requires_grad=True)
    h = OF.bias_swiglu(z)
    h.sum().backward()
    assert torch.isfinite(h).all() and torch.isfinite(z.grad).all()
    torch.testing.assert_close(h.detach(), S.swiglu(z).float())


def test_cpu_paths_match_the_reference():
    z, bias, _ = _inputs(torch.float32, f=20)                       # F % 8 != 0 and CPU: the torch expression
    torch.testing.assert_close(OF.bias_swiglu(z, bias), S.swiglu(z, bias).float())
    x, w, b = torch.randn(3, 32), torch.randn(40, 32), torch.randn(40)
    ln = (torch.rand(32) + 0.5, torch.randn(32), 1e-5)
    res = torch.randn(3, 20)
    want = S.swiglu(F.linear(F.layer_norm(x, (32,), ln[0], ln[1], ln[2]), w, b)).float() + res
    torch.testing.assert_close(OF.gemv_fused(x, w, b, ln=ln, residual=res, act="swiglu"), want, rtol=1e-5, atol=1e-5)
    with pytest.raises(ValueError, match="act"):
        OF.gemv_fused(x, w, b, act="relu")


# ---------------------------------------------------------------------------------------------------------------- model
def test_default_ffn_is_unchanged():
    base, m = _core(ffn_hidden_size=FFN), _core(ffn_hidden_size=FFN, ffn_activation="gelu")
    sa, sb = base.state_dict(), m.state_dict()
    assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa)
    assert sa["decoder.layers.0.linear1.weight"].shape == (FFN, HIDDEN) and sa["decoder.layers.0.linear2.weight"].shape == (HIDDEN, FFN)
    ids = _ids()
    assert torch.equal(base.eval()(ids), m.eval()(ids))
    assert _core().decoder.layers[0].linear1.weight.shape == (4 * HIDDEN, HIDDEN)


def test_swiglu_model_equals_plain_torch_with_deinterleaved_weights():
    m = _core(ffn_hidden_size=FFN, ffn_activation="swiglu")
    layer = m.decoder.layers[0]
    assert layer.linear1.weight.shape == (2 * FFN, HIDDEN) and layer.linear1.bias.shape == (2 * FFN,)
    assert layer.linear2.weight.shape == (HIDDEN, FFN)
    ids = _ids()
    y = m(ids)
    y.float().pow(2).mean().backward()
    want_grads = {n: p.grad.clone() for n, p in m.named_parameters()}

    # the same model with every FFN replaced by plain torch on separate gate / up weights (rows 0::2 and 1::2 of linear1)
    ref = _core(seed=3, ffn_hidden_size=FFN, ffn_activation="swiglu")
    ref.load_state_dict(m.state_dict())
    split = {}
    for i, l in enumerate(ref.decoder.layers):
        w1, b1 = l.linear1.weight.detach(), l.linear1.bias.detach()
        p = {k: torch.nn.Parameter(v.clone()) for k, v in
             dict(wg=w1[0::2], wu=w1[1::2], bg=b1[0::2], bu=b1[1::2], w2=l.linear2.weight.detach(), b2=l.linear2.bias.detach()).items()}
        split[i] = p
        l._ffn = (lambda p: lambda h: (F.linear(F.silu(F.linear(h, p["wg"], p["bg"])) * F.linear(h, p["wu"], p["bu"]), p["w2"]), p["b2"]))(p)
    y2 = ref(ids)
    torch.testing.assert_close(y2, y, rtol=1e-5, atol=1e-5)
    y2.float().pow(2).mean().backward()
    for i, p in split.items():
        g1 = torch.stack([p["wg"].grad, p["wu"].grad], 1).reshape(2 * FFN, HIDDEN)
        gb = torch.stack([p["bg"].grad, p["bu"].grad], 1).reshape(-1)
        torch.testing.assert_close(g1, want_grads[f"decoder.layers.{i}.linear1.weight"], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(gb, want_grads[f"decoder.layers.{i}.linear1.bias"], rtol=1e-4, atol=1e-6)
        torch.testing.assert_close(p["w2"].grad, want_grads[f"decoder.layers.{i}.linear2.weight"], rtol=1e-4, atol=1e-6)


def test_default_width_follows_the_llama_rule():
    from paddlefleetx_b200.models.language_model.language_module import process_model_configs

    assert gpt.swiglu_ffn_size(2048) == 5632 and gpt.swiglu_ffn_size(4096) == 11008 and gpt.swiglu_ffn_size(64) == 256
    for act, want in (("swiglu", 5632), ("gelu", 8192)):
        cfg = tiny_gpt_config(["Model.hidden_size=2048", "Model.num_attention_heads=16", "Model.ffn_hidden_size=None", f"Model.ffn_activation={act}"],
                              nranks=1)
        process_model_configs(cfg)
        assert cfg.Model.ffn_hidden_size == want, act
    assert _core(ffn_activation="swiglu").decoder.layers[0].linear2.weight.shape == (HIDDEN, 256)


@pytest.mark.parametrize("act", ["gelu", "swiglu"])
def test_parameter_counts_match_the_model(act):
    from paddlefleetx_b200.models.language_model.language_module import get_model_size
    from paddlefleetx_b200.utils.layout_planner import ModelShape

    l, v, s = 2, 128, 64
    m = _core(ffn_hidden_size=FFN, ffn_activation=act)
    assert get_model_size(l, HIDDEN, v, s, None, FFN, act) == sum(p.numel() for p in m.parameters())
    per_layer = sum(p.numel() for p in m.decoder.layers[0].parameters())
    assert ModelShape(layers=l, hidden=HIDDEN, heads=4, vocab=v, ffn=FFN, seq=s, ffn_activation=act).params_per_layer == per_layer
    # the GELU count with the default width is the count the function always gave
    assert get_model_size(l, HIDDEN, v, s) == get_model_size(l, HIDDEN, v, s, None, 4 * HIDDEN, "gelu") \
        == (v + s) * HIDDEN + (4 * HIDDEN ** 2 + 4 * HIDDEN) * l + 4 * HIDDEN * l + (8 * HIDDEN ** 2 + 5 * HIDDEN) * l + 2 * HIDDEN


def test_planner_counts_the_wider_ffn1():
    from paddlefleetx_b200.utils.layout_planner import Hardware, ModelShape, _layer_time

    gelu = ModelShape(layers=24, hidden=2048, heads=16, vocab=50304, ffn=8192, seq=1024)
    swiglu = ModelShape(layers=24, hidden=2048, heads=16, vocab=50304, ffn=5632, seq=1024, ffn_activation="swiglu")
    assert swiglu.ffn1_width == 2 * 5632 and gelu.ffn1_width == 8192
    assert swiglu.params_per_layer - gelu.params_per_layer == 2048 * (3 * 5632 - 2 * 8192) + (2 * 5632 - 8192)
    hw = Hardware()
    t = {k: _layer_time(hw, s, 8192, 1, False, "none")["gemm"] for k, s in (("gelu", gelu), ("swiglu", swiglu))}
    assert t["swiglu"] > 0 and math.isclose(t["swiglu"] / t["gelu"], 1.0, rel_tol=0.1)


def test_invalid_configurations_are_rejected():
    from paddlefleetx_b200.utils import check

    cases = [(["Model.ffn_activation=relu"], {}, "gelu or swiglu"),
             (["Model.ffn_activation=swiglu", "Model.moe_configs.expert_mode=True"], {}, "moe_configs"),
             (["Model.ffn_activation=swiglu", "Compress.Prune.enable=True"], {}, "Compress.Prune"),
             (["Model.ffn_activation=swiglu", "Model.ffn_hidden_size=100"], {"mp_degree": 8}, "divisible by mp_degree")]
    for ov, dist, msg in cases:
        cfg = tiny_gpt_config(ov, nranks=1)
        cfg.Distributed.update(dist)
        with pytest.raises(ValueError, match=msg):
            check.check_config(cfg)
    assert check.check_config(tiny_gpt_config(["Model.ffn_activation=swiglu"], nranks=1))
    with pytest.raises(ValueError, match="ffn_activation"):
        _core(ffn_activation="geglu")


def test_pruning_a_swiglu_model_is_refused():
    from paddlefleetx_b200.utils.compression_helper import prune_model

    with pytest.raises(ValueError, match="swiglu"):
        prune_model(_core(ffn_hidden_size=FFN, ffn_activation="swiglu"), {"enable": True, "ratio": 0.25})


def test_pipe_keys_round_trip():
    from paddlefleetx_b200.utils.ckpt_convert import gpt_pipe_to_plain, gpt_plain_to_pipe

    plain = {"gpt." + k: v for k, v in _core(ffn_hidden_size=FFN, ffn_activation="swiglu").state_dict().items()}
    pipe = gpt_plain_to_pipe(plain, 2)
    assert pipe["layers.1.linear1.weight"].shape == (2 * FFN, HIDDEN)
    back = gpt_pipe_to_plain(pipe, 2)
    assert list(back) == list(plain) and all(torch.equal(back[k], plain[k]) for k in plain)


# ---------------------------------------------------------------------------------------------------------------- decoding
def test_incremental_decoding_matches_full_forward():
    core = _core(ffn_hidden_size=FFN, ffn_activation="swiglu").eval()
    ids = _ids(s=10)
    with torch.no_grad():
        full = core(ids)
        caches = core.new_caches(ids.shape[0], ids.shape[1])
        steps = [core(ids[:, :4], caches=caches)]
        for t in range(4, 10):
            steps.append(core(ids[:, t:t + 1], caches=caches))
    torch.testing.assert_close(torch.cat(steps, 1), full, rtol=1e-4, atol=1e-4)


def test_fused_decode_step_matches_the_generic_step():
    from paddlefleetx_b200.models.language_model.gpt.generation import GPTForGeneration

    core = _core(ffn_hidden_size=FFN, ffn_activation="swiglu").eval()
    cfg = dict(max_dec_len=6, decode_strategy="greedy_search", eos_token_id=None, pad_token_id=0)
    ids = torch.randint(1, 120, (3, 7), generator=torch.Generator().manual_seed(3))
    a, _ = GPTForGeneration(core, dict(cfg, use_cuda_graph=False)).generate(ids)
    b, _ = GPTForGeneration(core, dict(cfg, use_cuda_graph=True, force_static_decode=True)).generate(ids)
    calls = []
    for layer in core.decoder.layers:
        layer._force_decode_fast = True              # the five-launch step through its CPU expressions (act="swiglu" GEMV)
        layer._decode_fast = (lambda f: lambda *x: calls.append(1) or f(*x))(layer._decode_fast)
    try:
        c, _ = GPTForGeneration(core, dict(cfg, use_cuda_graph=True, force_static_decode=True)).generate(ids)
    finally:
        for layer in core.decoder.layers:
            layer._force_decode_fast = False
            del layer._decode_fast
    assert calls and torch.equal(a, b) and torch.equal(a, c)


# ---------------------------------------------------------------------------------------------------------------- parallelism
def swiglu_tp_matches_single(rank, world, sp):
    """Two tensor-parallel ranks (each holding F / 2 gate / up pairs), with or without sequence parallelism, reproduce the single-process
    losses and weights."""
    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module
    from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

    gb = 2
    ov = ["Global.global_batch_size=None", f"Global.local_batch_size={gb}", f"Global.micro_batch_size={gb}", "Model.ffn_activation=swiglu",
          f"Model.ffn_hidden_size={FFN}"]
    cfg1 = tiny_gpt_config(ov, nranks=1)
    env.set_hcg(HybridCommunicateGroup(world_size=1, rank=0, build_groups=False))
    real_ws = env.world_size
    env.world_size = lambda: 1
    try:
        env.set_seed(cfg1.Global.seed)
        module1 = build_module(cfg1)
        init = {k: v.detach().clone() for k, v in module1.model.state_dict().items()}
        eng1 = EagerEngine(configs=cfg1, module=module1)
        batches = synthetic_batches(cfg1, 3, seed=21)
        ref_losses = [float(eng1.train_step(b)) for b in batches]
        ref_state = {k: v.detach().clone() for k, v in module1.model.state_dict().items()}
    finally:
        env.world_size = real_ws
        env.set_hcg(None)

    def shard(full, p, r):
        return full.chunk(world, dim=p.split_axis)[r].clone() if getattr(p, "tp_sharded", False) else full.clone()

    cfg = tiny_gpt_config(ov + [f"Distributed.mp_degree={world}", f"Model.sequence_parallel={sp}"], nranks=world)
    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    module = build_module(cfg)
    r = env.get_hcg().get_model_parallel_rank()
    layer = next(m for m in module.model.modules() if isinstance(m, gpt.TransformerDecoderLayer))
    assert layer.linear1.weight.shape == (2 * FFN // world, 64) and layer.linear2.weight.shape == (64, FFN // world)
    with torch.no_grad():
        for k, p in module.model.named_parameters():
            p.copy_(shard(init[k], p, r))
    eng = EagerEngine(configs=cfg, module=module)
    losses = [float(eng.train_step(b)) for b in batches]
    assert max(abs(a - b) for a, b in zip(losses, ref_losses)) < 3e-4, (losses, ref_losses)
    for k, p in module.model.named_parameters():
        want = shard(ref_state[k], p, r)
        assert torch.allclose(p.detach(), want, atol=1e-4, rtol=1e-3), (k, (p.detach() - want).abs().max())


@pytest.mark.parametrize("sp", [False, True])
def test_tensor_parallel_swiglu_matches_single_process(sp):
    run_distributed("test_swiglu_cpu:swiglu_tp_matches_single", 2, sp)


def swiglu_ckpt_mp2_to_mp1_and_back(rank, world, tmpdir):
    """An mp2 SwiGLU checkpoint merged to mp1 gives the mp2 model's outputs, and split back to mp2 it gives them again."""
    import torch.distributed as dist

    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module
    from paddlefleetx_b200.utils import ckpt_convert as cc

    out = os.path.join(tmpdir, "out")
    ov = ["Global.global_batch_size=None", "Global.local_batch_size=2", "Global.micro_batch_size=2", "Model.ffn_activation=swiglu",
          f"Model.ffn_hidden_size={FFN}", f"Engine.save_load.output_dir={out}"]
    cfg = tiny_gpt_config(ov + [f"Distributed.mp_degree={world}"], nranks=world)
    from helpers import build_engine

    eng = build_engine(cfg)
    batch = synthetic_batches(cfg, 1, seed=5)[0]
    eng.train_step(batch)
    eng.save(epoch=0, step=1)
    dist.barrier()
    model = eng._module.model.eval()
    with torch.no_grad():
        want = model(batch[0], batch[1]).detach().clone()                     # vocab-parallel logits of this rank
    src = os.path.join(out, "epoch_0_step_1")
    one, two = os.path.join(tmpdir, "mp1"), os.path.join(tmpdir, "mp2")
    if rank == 0:
        model, optim, meta = cc.merge_checkpoint(src)
        cc.split_checkpoint(model, optim, meta, one, mp=1)
        merged, _, meta1 = cc.merge_checkpoint(one)
        assert list(merged) == list(model) and all(torch.equal(merged[k], model[k]) for k in model)
        cc.split_checkpoint(merged, optim, meta1, two, mp=world)
    dist.barrier()
    full = cc.merge_checkpoint(one)[0]
    assert full["gpt.decoder.layers.0.linear1.weight"].shape == (2 * FFN, 64)
    cfg2 = tiny_gpt_config(ov + [f"Distributed.mp_degree={world}", f"Engine.save_load.ckpt_dir={two}"], nranks=world)
    env.set_seed(cfg2.Global.seed + 1)
    eng2 = build_engine(cfg2)
    eng2.load()
    with torch.no_grad():
        got = eng2._module.model.eval()(batch[0], batch[1])
    torch.testing.assert_close(got, want, rtol=0, atol=0)
    if rank == 0:                                                             # the merged mp1 checkpoint in a single-process model
        from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

        cfg1 = tiny_gpt_config(ov, nranks=1)
        env.set_hcg(HybridCommunicateGroup(world_size=1, rank=0, build_groups=False))
        real_ws = env.world_size
        env.world_size = lambda: 1
        try:
            m1 = build_module(cfg1).model.eval()
            m1.load_state_dict(full)
            with torch.no_grad():
                logits = m1(batch[0], batch[1])
        finally:
            env.world_size = real_ws
            env.set_hcg(None)
        v = want.shape[-1]
        torch.testing.assert_close(logits[..., :v], want, rtol=1e-5, atol=1e-5)


def test_checkpoint_mp2_to_mp1_and_back(tmp_path):
    run_distributed("test_swiglu_cpu:swiglu_ckpt_mp2_to_mp1_and_back", 2, str(tmp_path))


def test_pipeline_swiglu_matches_single():
    run_distributed("dist_fns:pipeline_matches_single", 2, 2, 1, 1, 4, False, 1, "ulysses", ["Model.ffn_activation=swiglu", f"Model.ffn_hidden_size={FFN}"])


# ---------------------------------------------------------------------------------------------------------------- recipe
def test_recipe_trains_through_the_cli():
    import re
    import subprocess
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = os.path.join(root, "paddlefleetx_b200", "configs", "nlp", "gpt", "pretrain_gpt_1.3B_swiglu_single_card.yaml")
    ov = ["Global.device=cpu", "Engine.mix_precision.enable=False", "Model.num_layers=2", "Model.hidden_size=64", "Model.num_attention_heads=4",
          "Model.max_position_embeddings=32", "Model.hidden_dropout_prob=0.0", "Model.attention_probs_dropout_prob=0.0", "Model.use_recompute=False",
          "Data.Train.dataset.name=SyntheticGPTDataset", "Data.Train.dataset.max_seq_len=32", "Data.Train.loader.num_workers=0",
          "Global.local_batch_size=2", "Global.micro_batch_size=2", "Engine.max_steps=3", "Engine.logging_freq=1", "Engine.eval_freq=-1",
          "Engine.save_load.save_steps=-1"]
    args = [sys.executable, "tools/train.py", "-c", cfg]
    for item in ov:
        args += ["-o", item]
    p = subprocess.run(args, capture_output=True, text=True, timeout=600, cwd=root, env=dict(os.environ, PYTHONPATH=root, CUDA_VISIBLE_DEVICES=""))
    log = p.stdout + p.stderr
    assert p.returncode == 0, log[-3000:]
    losses = [float(x) for x in re.findall(r"loss: ([0-9.]+)", log)]
    assert log.count("[train]") >= 3 and all(l == l for l in losses), log[-1500:]
