"""ERNIE's padding mask as a ``KeyPaddingMask`` on CPU.

The bits, ``key_end`` and ``key_dense`` for hand-written patterns (empty rows included), ``additive()`` against the tensors ERNIE built
before (bit for bit), ``ErnieModel`` outputs against the 4-D additive-mask path (bit for bit, flash and unfused attention), and gloo
parity of a padded batch under tensor parallelism, with and without sequence parallelism and with recompute.
"""
import pytest
import torch

from dist_utils import run_distributed
from paddlefleetx_b200.ops import attention as ATT


def _words(bits):
    return [[w & 0xFFFFFFFF for w in row] for row in bits.tolist()]


def test_bounds_of_hand_written_patterns():
    s = 70
    valid = torch.zeros(4, s, dtype=torch.bool)
    valid[0, :33] = True                                  # right padding
    valid[1] = True                                       # no padding
    valid[2, [0, 5, 40, 64]] = True                       # interior holes
    # row 3: no valid key -> every key of the row
    m = ATT.KeyPaddingMask.from_valid(valid)
    assert m.key_end.tolist() == [33, 70, 65, 70]
    assert m.key_dense.tolist() == [33, 70, 1, 70]
    assert m.key_bits.dtype == torch.int32 and m.key_bits.shape == (4, 3)
    assert _words(m.key_bits) == [[0xFFFFFFFF, 0x1, 0x0],
                                  [0xFFFFFFFF, 0xFFFFFFFF, 0x3F],
                                  [0x21, 0x100, 0x1],
                                  [0xFFFFFFFF, 0xFFFFFFFF, 0x3F]]
    want = valid.clone()
    want[3] = True
    assert torch.equal(m.dense(), want[:, None, None, :])


@pytest.mark.parametrize("dtype", [torch.bool, torch.int32, torch.int64, torch.float32, torch.float16, torch.bfloat16])
def test_every_validity_dtype_gives_the_same_bits(dtype):
    g = torch.Generator().manual_seed(0)
    valid = torch.rand(3, 100, generator=g) > 0.3
    valid[1, 60:] = False
    ref = ATT.KeyPaddingMask.from_valid(valid)
    got = ATT.KeyPaddingMask.from_valid(valid.to(dtype))
    for a, b in zip(ref.bounds(), got.bounds()):
        assert torch.equal(a, b)


def test_from_ids_matches_from_valid():
    ids = torch.tensor([[5, 7, 0, 9, 0, 0], [0, 0, 0, 0, 0, 0], [1, 2, 3, 4, 5, 6]])
    a, b = ATT.KeyPaddingMask.from_ids(ids, 0), ATT.KeyPaddingMask.from_valid(ids != 0)
    for x, y in zip(a.bounds(), b.bounds()):
        assert torch.equal(x, y)
    assert a.key_end.tolist() == [4, 6, 6] and a.key_dense.tolist() == [2, 6, 6]
    with pytest.raises(ValueError):
        ATT.KeyPaddingMask.from_ids(ids.float(), 0)
    with pytest.raises(ValueError):
        ATT.KeyPaddingMask.from_valid(ids[0])


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
def test_additive_is_the_previous_tensor(dtype):
    g = torch.Generator().manual_seed(1)
    ids = torch.randint(0, 5, (3, 40), generator=g)
    ids[2] = 0
    want = (ids == 0)[:, None, None, :].to(dtype) * -1e4
    got = ATT.KeyPaddingMask.from_ids(ids, 0, dtype).additive()
    assert got.dtype == dtype and torch.equal(got.view(torch.int16 if dtype != torch.float32 else torch.int32),
                                              want.view(torch.int16 if dtype != torch.float32 else torch.int32))
    for m in ((ids != 0).long(), (ids != 0).float(), ids != 0):
        want = (1.0 - m[:, None, None, :].to(dtype)) * -1e4
        got = ATT.KeyPaddingMask.from_valid(m, dtype).additive()
        assert got.dtype == dtype and torch.equal(got, want)
        assert torch.equal(ATT.KeyPaddingMask.from_valid(m).additive(dtype), want)


def _ernie(use_flash_attn, **kw):
    from paddlefleetx_b200.models.language_model.ernie import model as E

    torch.manual_seed(3)
    return E.ErnieModel(vocab_size=128, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, ffn_hidden_size=128,
                        max_position_embeddings=64, use_flash_attn=use_flash_attn, **kw).eval()


@pytest.mark.parametrize("use_flash_attn", [True, False])
def test_ernie_outputs_are_bit_identical_to_the_additive_mask(use_flash_attn):
    model = _ernie(use_flash_attn)
    g = torch.Generator().manual_seed(2)
    ids = torch.randint(1, 128, (3, 48), generator=g)
    ids[0, 30:] = 0
    ids[1, [3, 17, 18]] = 0
    seg = torch.randint(0, 2, (3, 48), generator=g)
    valid = (ids != 0).float()
    with torch.no_grad():
        old_ids = model(ids, seg, None, (ids == 0)[:, None, None, :].float() * -1e4)
        old_2d = model(ids, seg, None, (1.0 - valid[:, None, None, :]) * -1e4)
        new_ids = model(ids, seg)
        new_2d = model(ids, seg, None, valid)
    for a, b in ((old_ids, new_ids), (old_2d, new_2d)):
        for x, y in zip(a, b):
            assert torch.equal(x, y)


def test_ernie_builds_one_mask_per_forward(monkeypatch):
    model = _ernie(True)
    built = []
    real = ATT.KeyPaddingMask._build.__func__

    def count(cls, *a):
        built.append(1)
        return real(cls, *a)
    monkeypatch.setattr(ATT.KeyPaddingMask, "_build", classmethod(count))
    seen = []
    real_attention = ATT.attention

    def spy(q, k, v, *a, attn_mask=None, **kw):
        seen.append(attn_mask)
        return real_attention(q, k, v, *a, attn_mask=attn_mask, **kw)
    monkeypatch.setattr(ATT, "attention", spy)
    ids = torch.randint(1, 128, (2, 16))
    ids[:, 12:] = 0
    with torch.no_grad():
        model(ids)
    assert len(built) == 1 and len(seen) == 2
    assert all(isinstance(m, ATT.KeyPaddingMask) for m in seen) and seen[0] is seen[1]
    # the inspection path keeps the additive tensor
    seen.clear()
    with torch.no_grad():
        model(ids, output_hidden_states=True)
    assert len(built) == 1 and len(seen) == 2 and all(isinstance(m, torch.Tensor) and m.dim() == 4 for m in seen)


def ernie_padded_tp_matches_single(rank, world, sequence_parallel, use_recompute, mask_kind):
    """A padded batch (right padding, interior holes and one all-padding row) under tensor parallelism: the same scores and gradients as
    the single-process model."""
    import torch.distributed as dist

    from dist_fns import _shard_like
    from helpers import tiny_gpt_config
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models.language_model.ernie import model as E
    from paddlefleetx_b200.parallel.tp_layers import allreduce_sequence_parallel_grads, register_sequence_parallel_allreduce_hooks

    cfg = tiny_gpt_config(["Global.global_batch_size=None", "Global.local_batch_size=3", "Global.micro_batch_size=3", f"Distributed.mp_degree={world}"],
                          nranks=world)
    env.init_dist_env(cfg)
    hcg = env.get_hcg()
    group = hcg.get_model_parallel_group()
    mp_rank = hcg.get_model_parallel_rank()
    kw = dict(vocab_size=256, hidden_size=32, num_hidden_layers=2, num_attention_heads=4, ffn_hidden_size=64, max_position_embeddings=32,
              hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, use_flash_attn=True, use_recompute=use_recompute, dtype=torch.float64)
    torch.manual_seed(5)
    single = E.ErnieForPretraining(E.ErnieModel(**kw), 256).double()
    init = {k: v.detach().clone() for k, v in single.state_dict().items()}
    par = E.ErnieForPretraining(E.ErnieModel(mp_group=group, sequence_parallel=sequence_parallel, **kw), 256).double()
    with torch.no_grad():
        for k, p in par.named_parameters():
            p.copy_(_shard_like(init[k], p, mp_rank, world))
    if sequence_parallel:
        register_sequence_parallel_allreduce_hooks(par, 1, False, group)
    g = torch.Generator().manual_seed(9)
    ids = torch.randint(1, 256, (3, 16), generator=g)
    ids[0, 11:] = 0
    ids[1, [2, 7]] = 0
    ids[2] = 0
    mask = None if mask_kind == "ids" else (ids != 0).float()
    seg = torch.randint(0, 2, (3, 16), generator=g)
    masked = torch.tensor([1, 5, 9, 17, 20, 30])
    labels = torch.randint(0, 256, (6,), generator=g)
    single.train(); par.train()

    s1, r1 = single(ids, seg, None, mask, masked)
    tgt = torch.nn.functional.one_hot(labels, s1.shape[-1]).to(s1.dtype)
    ((s1 - tgt) ** 2).sum().add((r1 ** 2).sum()).backward()
    s2, r2 = par(ids, seg, None, mask, masked)
    v = s2.shape[-1]
    ((s2 - tgt[:, mp_rank * v:(mp_rank + 1) * v]) ** 2).sum().add((r2 ** 2).sum()).backward()
    if sequence_parallel:
        allreduce_sequence_parallel_grads(par)
    torch.testing.assert_close(s2, s1[:, mp_rank * v:(mp_rank + 1) * v], rtol=1e-8, atol=1e-9)
    torch.testing.assert_close(r2, r1, rtol=1e-8, atol=1e-9)
    ref_grads = {k: p.grad for k, p in single.named_parameters()}
    for k, p in par.named_parameters():
        torch.testing.assert_close(p.grad, _shard_like(ref_grads[k], p, mp_rank, world), rtol=1e-6, atol=1e-8, msg=lambda m, k=k: f"{k}: {m}")
    dist.barrier()


@pytest.mark.parametrize("sp,recompute,mask_kind", [(False, False, "ids"), (True, False, "valid"), (False, True, "valid"), (True, True, "ids")])
def test_padded_ernie_tensor_parallel_matches_single(sp, recompute, mask_kind):
    run_distributed("test_ernie_key_padding_cpu:ernie_padded_tp_matches_single", 2, sp, recompute, mask_kind)
