"""Intra-document attention for packed sequences, without a GPU: dataset position ids (``reset_position_ids``), the ``DocumentMask``
derivation and its dense form, GPT with ``reset_attention_mask`` (a packed row equals its documents run alone), tensor / sequence
parallelism under gloo, the config rejections, the recipe through ``tools/train.py`` and left-padded generation prefill."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from dist_utils import run_distributed
from paddlefleetx_b200.data.dataset.gpt_dataset import GPTDataset, SyntheticGPTDataset, TokenCorpus, document_positions
from paddlefleetx_b200.models.language_model.gpt import model as gpt
from paddlefleetx_b200.ops import attention as ATT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "paddlefleetx_b200", "configs", "nlp", "gpt")


# ---------------------------------------------------------------------------------------------------------------- dataset
LENS = [5, 3, 5, 2, 9]


def _dataset(tmp_path, sample_idx, reset=True, mask_eos=False, eos_id=-1):
    ids = np.concatenate([100 * d + np.arange(n) for d, n in enumerate(LENS)]).astype(np.int64)
    np.save(tmp_path / "c_ids.npy", ids)
    np.savez(tmp_path / "c_idx.npz", lens=np.array(LENS, dtype=np.int32))
    ds = GPTDataset.__new__(GPTDataset)
    ds.corpus = TokenCorpus(str(tmp_path / "c"))
    ds.doc_idx = np.arange(len(LENS), dtype=np.int32)
    ds.sample_idx = np.array(sample_idx, dtype=np.int64)
    ds.shuffle_idx = np.arange(len(sample_idx) - 1)
    ds.mode, ds.max_seq_len, ds.eos_id, ds.mask_eos, ds.reset_position_ids = "Train", 8, eos_id, mask_eos, reset
    return ds


@pytest.mark.parametrize("bounds,pieces", [
    ([(0, 3), (2, 3)], [2, 3, 4]),          # starts mid-document, spans three documents
    ([(4, 0), (4, 8)], [9]),                # one document
    ([(1, 0), (3, 0)], [3, 5, 1]),          # the inputs end exactly on a document boundary (only the last label is the next document's)
    ([(1, 2), (4, 0)], [1, 5, 2, 1]),       # starts on a document's last token, spans four documents
])
def test_dataset_positions_restart_at_each_document(tmp_path, bounds, pieces):
    ds = _dataset(tmp_path, bounds)
    tokens, pos, labels, _ = ds[0]
    assert ds._piece_lengths(0) == pieces
    docs, offs = tokens // 100, tokens % 100
    first = docs == docs[0]
    np.testing.assert_array_equal(pos[~first], offs[~first])                  # whole documents: the offset inside the document
    np.testing.assert_array_equal(pos[first], np.arange(first.sum()))          # the first piece counts from 0, even mid-document
    np.testing.assert_array_equal(pos, document_positions(pieces, 8))
    np.testing.assert_array_equal(_dataset(tmp_path, bounds, reset=False)[0][1], np.arange(8))


def test_dataset_reset_positions_compose_with_mask_eos(tmp_path):
    ds = _dataset(tmp_path, [(0, 3), (2, 3)], mask_eos=True, eos_id=200)
    tokens, pos, _, loss_mask = ds[0]
    np.testing.assert_array_equal(pos, [0, 1, 0, 1, 2, 0, 1, 2])
    np.testing.assert_array_equal(loss_mask, (tokens != 200).astype(np.float32))


def test_synthetic_dataset_documents_are_seeded():
    ds = SyntheticGPTDataset(max_seq_len=300, vocab_size=100, reset_position_ids=True, document_length=40, seed=3)
    lens = ds.document_lengths(5)
    assert sum(lens) == 301 and all(1 <= n <= 60 for n in lens) and len(lens) > 3
    assert lens == SyntheticGPTDataset(max_seq_len=300, vocab_size=100, document_length=40, seed=3).document_lengths(5)
    np.testing.assert_array_equal(ds[5][1], document_positions(lens, 300))
    np.testing.assert_array_equal(SyntheticGPTDataset(max_seq_len=300, vocab_size=100)[5][1], np.arange(300))


# ---------------------------------------------------------------------------------------------------------------- the mask
def test_key_start_and_tile_bounds_from_positions():
    pos = torch.tensor([[0, 1, 2, 0, 1, 9, 0, -3] + list(range(122))])       # 9 > i and -3 < 0 are clamped into [0, i]
    doc = ATT.DocumentMask.from_positions(pos)
    ks = doc.key_start[0].tolist()
    assert doc.key_start.dtype == torch.int32 and ks[:8] == [0, 0, 0, 3, 3, 0, 6, 7] and ks[8:] == [8] * 122
    assert doc.tile_min.tolist() == [[0, 8, 8]] and doc.tile_max.tolist() == [[8, 8, 8]]
    expl = ATT.DocumentMask.from_key_start(torch.tensor([[0, 5, -1, 2, 100]]))
    assert expl.key_start.tolist() == [[0, 1, 0, 2, 4]] and expl.tile_min.tolist() == [[0]] and expl.tile_max.tolist() == [[4]]


def test_dense_mask_matches_a_hand_built_one():
    pos = torch.tensor(np.stack([document_positions([3, 1, 4], 8), document_positions([8], 8)]))
    want = torch.zeros(2, 8, 8, dtype=torch.bool)
    for b, lens in enumerate(([3, 1, 4], [8])):
        s = 0
        for n in lens:
            for i in range(s, s + n):
                want[b, i, s:i + 1] = True
            s += n
    doc = ATT.DocumentMask.from_positions(pos)
    assert torch.equal(doc.dense()[:, 0], want)
    add = doc.additive()
    assert torch.equal(add[:, 0] == 0, want) and torch.isinf(add[:, 0][~want]).all()


def test_attention_fallback_takes_a_document_mask():
    torch.manual_seed(0)
    q, k, v = (torch.randn(2, 8, 4, 16) for _ in range(3))
    doc = ATT.DocumentMask.from_positions(torch.tensor(np.stack([document_positions([3, 5], 8)] * 2)))
    want = ATT.attention(q, k, v, causal=False, attn_mask=doc.dense())
    torch.testing.assert_close(ATT.attention(q, k, v, attn_mask=doc), want)
    torch.testing.assert_close(ATT.core_attention(q, k, v, 16 ** -0.5, 0.0, False, attn_mask=doc), want, rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------------------------------------------------------- GPT
def _model(use_rope, kv, flash=True, **kw):
    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=128, hidden_size=64, num_layers=2, num_attention_heads=4, ffn_hidden_size=128, max_position_embeddings=64,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, use_rope=use_rope, num_key_value_heads=kv,
                        use_flash_attn=flash, reset_attention_mask=True, **kw)
    return gpt.GPTForPretraining(core).eval()


@pytest.mark.parametrize("flash", [True, False])
@pytest.mark.parametrize("use_rope,kv", [(False, None), (True, None), (False, 2), (True, 1)])
def test_packed_row_equals_documents_run_alone(use_rope, kv, flash):
    model = _model(use_rope, kv, flash)
    lens = [5, 11, 1, 7]
    tokens = torch.randint(0, 128, (1, sum(lens)))
    pos = torch.tensor(document_positions(lens, sum(lens))).unsqueeze(0)
    with torch.no_grad():
        packed = model(tokens, pos)
        s = 0
        for n in lens:
            alone = model(tokens[:, s:s + n], torch.arange(n).unsqueeze(0))
            torch.testing.assert_close(packed[:, s:s + n], alone, rtol=1e-5, atol=1e-5)
            s += n
        model.gpt.reset_attention_mask = False                               # plain causal attention sees the earlier documents
        assert not torch.allclose(model(tokens, pos)[:, 5:], packed[:, 5:], atol=1e-3)


def test_recompute_granularities_keep_the_mask():
    lens = [6, 10]
    tokens = torch.randint(0, 128, (2, 16))
    pos = torch.tensor(np.stack([document_positions(lens, 16)] * 2))
    ref = _model(False, None)
    with torch.no_grad():
        want = ref(tokens, pos)
    for gran in ("full", "full_attn", "core_attn"):
        m = _model(False, None, use_recompute=True, recompute_granularity=gran).train()
        out = m(tokens, pos)
        out.sum().backward()
        torch.testing.assert_close(out.detach(), want, rtol=1e-5, atol=1e-5)


def tp_doc_matches_single(rank, world, sequence_parallel):
    """mp2 (with or without sequence parallelism) against mp1 with the document mask on: same losses and weights after three steps."""
    from dist_fns import _shard_like
    from helpers import synthetic_batches, tiny_gpt_config
    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module
    from paddlefleetx_b200.parallel.topology import HybridCommunicateGroup

    ov = ["Global.global_batch_size=None", "Global.local_batch_size=2", "Global.micro_batch_size=2", "Model.reset_attention_mask=True",
          "Data.Train.dataset.reset_position_ids=True", "Data.Eval.dataset.reset_position_ids=True"]
    cfg1 = tiny_gpt_config(ov, nranks=1)
    env.set_hcg(HybridCommunicateGroup(world_size=1, rank=0, build_groups=False))
    real_ws = env.world_size
    env.world_size = lambda: 1
    try:
        env.set_seed(cfg1.Global.seed)
        module1 = build_module(cfg1)
        assert module1.model.gpt.reset_attention_mask
        init = {k: v.detach().clone() for k, v in module1.model.state_dict().items()}
        eng1 = EagerEngine(configs=cfg1, module=module1)
        batches = synthetic_batches(cfg1, 3, seed=21)
        s = batches[0][0].shape[1]
        for i, b in enumerate(batches):
            b[1] = torch.tensor(np.stack([document_positions([5 + 3 * i, 9, s], s), document_positions([s // 2, s], s)]))
        ref_losses = [float(eng1.train_step(b)) for b in batches]
        ref_state = {k: v.detach().clone() for k, v in module1.model.state_dict().items()}
    finally:
        env.world_size = real_ws
        env.set_hcg(None)
    cfg = tiny_gpt_config(ov + [f"Distributed.mp_degree={world}", f"Model.sequence_parallel={sequence_parallel}"], nranks=world)
    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    module = build_module(cfg)
    hcg = env.get_hcg()
    with torch.no_grad():
        for k, p in module.model.named_parameters():
            p.copy_(_shard_like(init[k], p, hcg.get_model_parallel_rank(), world))
    eng = EagerEngine(configs=cfg, module=module)
    losses = [float(eng.train_step(b)) for b in batches]
    assert max(abs(a - b) for a, b in zip(losses, ref_losses)) < 3e-4, (losses, ref_losses)
    for k, p in module.model.named_parameters():
        want = _shard_like(ref_state[k], p, hcg.get_model_parallel_rank(), world)
        assert torch.allclose(p.detach(), want, atol=1e-4, rtol=1e-3), (k, (p.detach() - want).abs().max())


@pytest.mark.parametrize("sp", [False, True])
def test_tensor_parallel_document_mask_matches_single(sp):
    run_distributed("test_doc_attention_cpu:tp_doc_matches_single", 2, sp)


# ---------------------------------------------------------------------------------------------------------------- config
@pytest.mark.parametrize("extra,dist,needle", [
    (["Data.Train.dataset.reset_position_ids=False"], {}, "reset_position_ids"),
    ([], {"pp_degree": 2}, "pp_degree"),
    ([], {"cp_degree": 2}, "cp_degree"),
])
def test_config_rejections(extra, dist, needle):
    from helpers import tiny_gpt_config
    from paddlefleetx_b200.utils import check

    base = ["Model.reset_attention_mask=True", "Data.Train.dataset.reset_position_ids=True", "Data.Eval.dataset.reset_position_ids=True"]
    assert check.check_config(tiny_gpt_config(base, nranks=1))
    cfg = tiny_gpt_config(base + extra, nranks=1)
    cfg.Distributed.update(dist)
    with pytest.raises(ValueError, match=needle):
        check.check_config(cfg)


def test_recipe_trains_through_the_cli():
    cfg = os.path.join(CFG, "pretrain_gpt_1.3B_packed_docs_single_card.yaml")
    ov = ["Global.device=cpu", "Engine.mix_precision.enable=False", "Model.num_layers=2", "Model.hidden_size=64", "Model.num_attention_heads=4",
          "Model.max_position_embeddings=64", "Model.hidden_dropout_prob=0.0", "Model.attention_probs_dropout_prob=0.0", "Model.use_recompute=False",
          "Data.Train.dataset.name=SyntheticGPTDataset", "Data.Train.dataset.max_seq_len=64", "Data.Train.dataset.document_length=12",
          "Data.Train.loader.num_workers=0", "Global.local_batch_size=2", "Global.micro_batch_size=2", "Engine.max_steps=3",
          "Engine.logging_freq=1", "Engine.eval_freq=-1", "Engine.save_load.save_steps=-1"]
    args = [sys.executable, "tools/train.py", "-c", cfg]
    for item in ov:
        args += ["-o", item]
    p = subprocess.run(args, capture_output=True, text=True, timeout=600, cwd=ROOT, env=dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES=""))
    log = p.stdout + p.stderr
    assert p.returncode == 0, log[-3000:]
    losses = [float(x) for x in re.findall(r"loss: ([0-9.]+)", log)]
    assert log.count("[train]") >= 3 and all(l == l for l in losses), log[-1500:]


# ---------------------------------------------------------------------------------------------------------------- generation
def test_left_padded_prefill_mask_equals_the_additive_path():
    from paddlefleetx_b200.models.language_model.gpt.generation import GPTForGeneration, _left_padded_mask, _to_additive

    core = _model(False, 2).gpt
    core.reset_attention_mask = False
    b, s = 3, 12
    ids = torch.randint(1, 128, (b, s))
    valid = torch.ones(b, s, dtype=torch.bool)
    valid[1, :4] = False
    valid[2, :11] = False
    ids[~valid] = 0
    pos = (valid.long().cumsum(-1) - 1).clamp(min=0)
    causal = torch.ones(s, s, dtype=torch.bool).tril()
    dense = ((causal.unsqueeze(0) & valid.unsqueeze(1)).unsqueeze(1)) | torch.eye(s, dtype=torch.bool)
    doc = _left_padded_mask(valid)
    assert torch.equal(doc.dense(), dense)
    assert doc.key_start.tolist()[1] == [0, 1, 2, 3] + [4] * 8
    with torch.no_grad():
        torch.testing.assert_close(core(ids, pos, doc, core.new_caches(b, s + 2)), core(ids, pos, _to_additive(dense, torch.float32),
                                                                                         core.new_caches(b, s + 2)), rtol=1e-5, atol=1e-5)
    right = valid.flip(-1)
    assert _left_padded_mask(right) is None                                  # right padding keeps the additive path
    gen = GPTForGeneration(core, dict(max_dec_len=3, decode_strategy="greedy_search", eos_token_id=None, pad_token_id=0, use_cuda_graph=False))
    out, _ = gen.generate(ids)
    assert out.shape == (b, 3)
