"""The references of ``decode_refs`` on the CPU: the Philox port against Random123's published known-answer vectors, and the top-p law
against the sort-based PyTorch sampler and on the rows generation hands it (zeros after top-k filtering, top_p = 1, a single token)."""
import numpy as np
import pytest
import torch

import decode_refs as D
from paddlefleetx_b200.models.language_model.gpt.generation import top_k_filter
from paddlefleetx_b200.ops import functional as OF

# Random123 kat_vectors, philox4x32 with 10 rounds: counter words 0..3, key words 0..1, result words 0..3
PHILOX_KAT = [
    ((0x00000000, 0x00000000, 0x00000000, 0x00000000), (0x00000000, 0x00000000), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF, 0xFFFFFFFF), (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
]


@pytest.mark.parametrize("ctr,key,want", PHILOX_KAT)
def test_philox_known_answers(ctr, key, want):
    got = D.philox4x32(np.array(ctr, dtype=np.uint32), np.array(key, dtype=np.uint32))
    assert [int(v) for v in got] == list(want)


def test_philox_of_seed_and_counter_is_the_four_word_generator():
    seed, counters = 0x0123456789ABCDEF, np.array([0, 1, 2 ** 32 + 7, 2 ** 64 - 1], dtype=np.uint64)
    got = D.philox(seed, counters)
    for c, row in zip(counters, got):
        c = int(c)
        want = D.philox4x32(np.array([c & 0xFFFFFFFF, c >> 32, 0x243F6A88, 0x85A308D3], dtype=np.uint32),
                            np.array([seed & 0xFFFFFFFF, seed >> 32], dtype=np.uint32))
        assert (row == want).all()
    uni = D.uniform(seed, counters)
    assert uni.dtype == np.float32 and ((uni >= 0) & (uni < 1)).all()
    assert (uni * np.float32(2 ** 24) == (got[:, 0] >> 8).astype(np.float64)).all()


def test_keep8_reads_both_halves_of_each_word():
    k = D.keep8(5, 9, 3, 0x8000)
    r = D.philox(5, np.arange(9, 12, dtype=np.uint64))
    assert k.shape == (24,)
    for v in range(3):
        for i in range(4):
            assert k[8 * v + 2 * i] == ((int(r[v, i]) & 0xFFFF) >= 0x8000)
            assert k[8 * v + 2 * i + 1] == ((int(r[v, i]) >> 16) >= 0x8000)


def _tie_free(rows, V, seed):
    """fp32 rows of V distinct probabilities: a random order of the weights 1 .. V, each moved by less than half a step."""
    g = torch.Generator().manual_seed(seed)
    wts = torch.argsort(torch.rand(rows, V, generator=g), -1).double() + 1 + 0.4 * torch.rand(rows, V, generator=g, dtype=torch.float64)
    p = (wts / wts.sum(-1, keepdim=True)).float()
    assert all(len(torch.unique(r)) == V for r in p)
    return p


def test_topp_law_matches_the_sorting_sampler_without_ties():
    rows, V, seed, offset = 256, 500, 11, 3
    p = _tie_free(rows, V, 1)
    tp = torch.full((rows,), 0.9)
    tp[::3] = 0.5
    _, ids = OF.topp_sampling(p, tp, seed, offset)            # CPU: the sort-based PyTorch path
    u = torch.rand(rows, 1, generator=torch.Generator().manual_seed(seed + offset)).reshape(-1).numpy()
    want, margin = D.topp_expected(p, tp.numpy(), u)
    # the fallback sums in fp32: a threshold closer to a boundary than its rounding may land on the neighbour
    clear = margin > V * 2.0 ** -24
    assert clear.float().mean() > 0.95
    assert torch.equal(ids.reshape(-1)[clear], want[clear])


def test_topp_law_on_rows_with_zeros_top_p_one_and_a_single_token():
    p = top_k_filter(_tie_free(64, 300, 2), 20)
    assert ((p > 0).sum(-1) == 20).all()
    p = p / p.sum(-1, keepdim=True)
    u = D.uniform(7, np.arange(64, dtype=np.uint64))
    ids, margin = D.topp_expected(p, np.ones(64, dtype=np.float32), u)
    assert (p.gather(-1, ids[:, None]) > 0).all()              # zeros are never chosen, even with top_p = 1
    order, cum = D.sorted_mass(p)
    for r in range(64):
        k = int((order[r] == ids[r]).nonzero())
        lo = float(cum[r, k - 1]) if k else 0.0
        assert lo < float(u[r]) <= float(cum[r, k]) and margin[r] >= 0
    # a threshold above the row's mass (rounding) takes the last token of positive probability
    short = torch.tensor([[0.25, 0.0, 0.5, 0.125]], dtype=torch.float64)
    assert int(D.topp_expected(short, [1.0], [0.9375])[0][0]) == 3
    # V = 1: the only token, whatever the draw
    ids, _ = D.topp_expected(torch.ones(5, 1), np.ones(5, np.float32), D.uniform(3, np.arange(5, dtype=np.uint64)))
    assert (ids == 0).all()


def test_topp_law_takes_ties_in_index_order_and_the_arg_max_early_out_agrees():
    p = torch.tensor([[0.125, 0.25, 0.125, 0.25, 0.25]], dtype=torch.float64)
    # sorted: 1, 3, 4 (0.25 each), then 0, 2 (0.125 each); boundaries at 0.25, 0.5, 0.75, 0.875, 1
    for u, want in ((0.1, 1), (0.25, 1), (0.2500001, 3), (0.5, 3), (0.74, 4), (0.8, 0), (0.99, 2)):
        assert int(D.topp_expected(p, [1.0], [u])[0][0]) == want, u
    # p_max >= u: the lowest index among the tokens tied at the maximum
    assert int(D.topp_expected(p, [0.25], [0.5])[0][0]) == int(torch.argmax(p))
