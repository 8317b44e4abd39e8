"""Grouped-query attention for GPT (``Model.num_key_value_heads``) on the CPU path: layout, equivalences, decoding, validation, planner
and tensor parallelism."""
import pytest
import torch

from dist_utils import run_distributed
from helpers import synthetic_batches, tiny_gpt_config

from paddlefleetx_b200.models.language_model.finetune_module import convert_qkv_layout
from paddlefleetx_b200.models.language_model.gpt import model as gpt

H, HIDDEN = 4, 64


def _core(seed=0, **kw):
    torch.manual_seed(seed)
    return gpt.GPTModel(vocab_size=128, hidden_size=HIDDEN, num_layers=2, num_attention_heads=H, ffn_hidden_size=128,
                        max_position_embeddings=64, hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, **kw)


def _ids(b=2, s=12, seed=1):
    return torch.randint(0, 128, (b, s), generator=torch.Generator().manual_seed(seed))


@pytest.mark.parametrize("fuse", [True, False])
def test_kv_heads_equal_to_heads_changes_nothing(fuse):
    ids = _ids()
    base = _core(fuse_attn_qkv=fuse).eval()
    for kv in (None, H):
        m = _core(fuse_attn_qkv=fuse, num_key_value_heads=kv).eval()
        sa, sb = base.state_dict(), m.state_dict()
        assert list(sa) == list(sb)
        assert all(sa[k].shape == sb[k].shape and torch.equal(sa[k], sb[k]) for k in sa)
        assert torch.equal(base(ids), m(ids))


def _repeat_kv_into_mha(gqa: gpt.GPTModel, mha: gpt.GPTModel, kv: int):
    """Copy split-QKV GQA weights into an MHA model whose K/V heads repeat each group's K/V head (``repeat_interleave``)."""
    g, d = H // kv, HIDDEN // H
    state = dict(gqa.state_dict())
    for k in list(state):
        if ".k_proj." in k or ".v_proj." in k:
            t = state[k]
            state[k] = t.reshape(kv, d, *t.shape[1:]).repeat_interleave(g, 0).reshape(H * d, *t.shape[1:])
    mha.load_state_dict(state)


@pytest.mark.parametrize("kv", [1, 2])
def test_grouped_layout_fused_split_and_repeated_kv_agree(kv):
    ids = _ids()
    fused = _core(num_key_value_heads=kv).eval()
    assert fused.decoder.layers[0].self_attn.qkv_proj.weight.shape == ((H + 2 * kv) * HIDDEN // H, HIDDEN)
    split = _core(seed=5, fuse_attn_qkv=False, num_key_value_heads=kv).eval()
    st = convert_qkv_layout(fused.state_dict(), False, H, kv)
    split.load_state_dict(st)
    want = fused(ids)
    torch.testing.assert_close(split(ids), want, rtol=1e-5, atol=1e-5)
    back = convert_qkv_layout(st, True, H, kv)
    assert all(torch.equal(back[k], v) for k, v in fused.state_dict().items())
    # query head h uses K/V head h // G: the model equals an MHA model with every group's K/V repeated
    mha = _core(seed=7, fuse_attn_qkv=False).eval()
    _repeat_kv_into_mha(split, mha, kv)
    torch.testing.assert_close(mha(ids), want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("kv", [1, 2])
def test_incremental_decoding_matches_full_forward(kv):
    core = _core(num_key_value_heads=kv).eval()
    ids = _ids(s=10)
    with torch.no_grad():
        full = core(ids)
        caches = core.new_caches(ids.shape[0], ids.shape[1])
        assert all(c.k.shape == (2, 10, kv, HIDDEN // H) and c.v.shape == c.k.shape for c in caches)
        steps = [core(ids[:, :4], caches=caches)]
        for t in range(4, 10):
            steps.append(core(ids[:, t:t + 1], caches=caches))
    torch.testing.assert_close(torch.cat(steps, 1), full, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("kv", [1, 2])
def test_generation_static_and_fused_decode_match_dynamic_cache(kv):
    from paddlefleetx_b200.models.language_model.gpt.generation import GPTForGeneration

    core = _core(num_key_value_heads=kv).eval()
    cfg = dict(max_dec_len=6, decode_strategy="greedy_search", eos_token_id=None, pad_token_id=0)
    ids = torch.randint(1, 120, (3, 7), generator=torch.Generator().manual_seed(3))
    ids[1, :3] = 0
    a, _ = GPTForGeneration(core, dict(cfg, use_cuda_graph=False)).generate(ids)
    b, _ = GPTForGeneration(core, dict(cfg, use_cuda_graph=True, force_static_decode=True)).generate(ids)
    for layer in core.decoder.layers:
        layer._force_decode_fast = True              # the packed [b, 1, Hkv, G + 2, d] decode step through its CPU expressions
    try:
        c, _ = GPTForGeneration(core, dict(cfg, use_cuda_graph=True, force_static_decode=True)).generate(ids)
    finally:
        for layer in core.decoder.layers:
            layer._force_decode_fast = False
    assert torch.equal(a, b) and torch.equal(a, c)
    # greedy tokens from the cache equal greedy tokens recomputed without one
    seq = ids[0:1]
    with torch.no_grad():
        for _ in range(a.shape[1]):
            seq = torch.cat([seq, _last_logits(core, seq).argmax(-1, keepdim=True)], 1)
    assert torch.equal(seq[0, ids.shape[1]:], a[0])


def _last_logits(core, seq):
    h = core(seq)
    return h[:, -1] @ core.embeddings.word_embeddings.weight.t()


def test_invalid_head_configurations_are_rejected():
    from paddlefleetx_b200.utils import check

    with pytest.raises(AssertionError):
        _core(num_key_value_heads=3)
    cases = [({"num_key_value_heads": 3}, {}, "multiple of num_key_value_heads"),
             ({"num_key_value_heads": 1}, {"mp_degree": 2}, "divisible by mp_degree"),
             ({"num_key_value_heads": 2}, {"cp_degree": 2}, "context parallelism"),
             ({"num_key_value_heads": 2, "prune": True}, {}, "head pruning")]
    for model, dist, msg in cases:
        cfg = tiny_gpt_config([f"Model.num_key_value_heads={model['num_key_value_heads']}"]
                              + (["Compress.Prune.enable=True"] if model.get("prune") else []), nranks=1)
        cfg.Distributed.update(dist)
        with pytest.raises(ValueError, match=msg):
            check.check_config(cfg)
    ok = tiny_gpt_config(["Model.num_key_value_heads=2"], nranks=1)
    assert check.check_config(ok)


def test_head_pruning_of_a_grouped_model_is_refused():
    from paddlefleetx_b200.utils.compression_helper import prune_model

    with pytest.raises(ValueError, match="grouped-query"):
        prune_model(_core(num_key_value_heads=2), {"enable": True, "ratio": 0.25})


def test_planner_respects_kv_heads():
    from paddlefleetx_b200.utils.layout_planner import ModelShape, enumerate_plans

    mha = ModelShape(layers=24, hidden=2048, heads=16, vocab=50304, ffn=8192, seq=8192)
    gqa = ModelShape(layers=24, hidden=2048, heads=16, vocab=50304, ffn=8192, seq=8192, kv_heads=2)
    d = 2048 // 16
    assert mha.params_per_layer - gqa.params_per_layer == 2048 * (16 - 2) * 2 * d + (16 - 2) * 2 * d
    plans = enumerate_plans(gqa, 16, 1)
    assert plans and all(2 % p.mp == 0 for p in plans) and all(p.cp == 1 for p in plans)
    assert {p.mp for p in enumerate_plans(mha, 16, 1)} >= {4, 8}


def test_model_size_counts_grouped_qkv():
    from paddlefleetx_b200.models.language_model.language_module import get_model_size

    l, h, v, s = 2, 64, 512, 32
    assert get_model_size(l, h, v, s) == get_model_size(l, h, v, s, h)
    m = _core(num_key_value_heads=1)
    n_attn = sum(p.numel() for n, p in m.named_parameters() if "self_attn" in n)
    n_attn_mha = sum(p.numel() for n, p in _core().named_parameters() if "self_attn" in n)
    assert get_model_size(l, h, v, s) - get_model_size(l, h, v, s, h // H) == n_attn_mha - n_attn


def gqa_tp_matches_single(rank, world):
    """Two tensor-parallel ranks (mp 2, 2 K/V heads: one group per rank) reproduce the single-process losses and weights."""
    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module
    from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

    gb = 2
    ov = ["Global.global_batch_size=None", f"Global.local_batch_size={gb}", f"Global.micro_batch_size={gb}", "Model.num_key_value_heads=2"]
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

    cfg = tiny_gpt_config(ov + [f"Distributed.mp_degree={world}"], nranks=world)
    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    module = build_module(cfg)
    r = env.get_hcg().get_model_parallel_rank()
    attn = next(m for m in module.model.modules() if isinstance(m, gpt.MultiHeadAttention))
    assert (attn.local_heads, attn.local_kv_heads) == (2, 1)
    with torch.no_grad():
        for k, p in module.model.named_parameters():
            p.copy_(shard(init[k], p, r))
    eng = EagerEngine(configs=cfg, module=module)
    losses = [float(eng.train_step(b)) for b in batches]
    assert max(abs(a - b) for a, b in zip(losses, ref_losses)) < 3e-4, (losses, ref_losses)
    for k, p in module.model.named_parameters():
        want = shard(ref_state[k], p, r)
        assert torch.allclose(p.detach(), want, atol=1e-4, rtol=1e-3), (k, (p.detach() - want).abs().max())


def test_tensor_parallel_grouped_attention_matches_single_process():
    run_distributed("test_gqa_cpu:gqa_tp_matches_single", 2)


def test_prefix_tuning_of_a_grouped_model():
    from paddlefleetx_b200.utils.peft import apply_prefix_tuning

    core = _core(num_key_value_heads=2)
    enc = apply_prefix_tuning(core, num_virtual_tokens=4, hidden=16)
    core(_ids()).float().pow(2).mean().backward()
    assert all(p.grad is not None for p in enc.parameters() if p.requires_grad)
