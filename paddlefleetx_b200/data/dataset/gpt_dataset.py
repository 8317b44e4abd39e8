"""GPT pre-training / evaluation datasets.

File formats and cache names are those of the reference (ppfleetx/data/dataset/gpt_dataset.py:42-217,274-393):
``<prefix>_ids.npy`` (flat token ids, memory-mapped) + ``<prefix>_idx.npz`` (``lens`` per document) and the
derived ``<prefix>_gpt_<mode>_indexmap_<N>ns_<S>sl_{doc,sample,shuffle}_idx.npy`` caches, so existing
pre-processed corpora and caches are reusable.  Differences:

  * no tokenizer is needed to *train* (the reference instantiates one only to read ``eos_token_id`` and it
    downloads the vocab): ``eos_id`` defaults to 50256 and is configurable,
  * EOS loss-masking is an explicit switch ``mask_eos`` (default False = the reference's *actual* behaviour:
    its mask expression compares a python list with an int and masks nothing — SURVEY F8),
  * ``SyntheticGPTDataset`` produces uniform random tokens of the same 4-tuple shape for benchmarking,
  * ``reset_position_ids`` restarts the position ids at 0 at each document start inside a sample (Megatron's switch of that name; the
    boundaries come from the sample's own document pieces, not from EOS tokens), so that ``Model.reset_attention_mask`` keeps attention
    inside each document.  A sample that starts in the middle of a document counts its first piece from 0.
"""
from __future__ import annotations

import os
import time
from typing import List, Optional, Sequence

import numpy as np
import torch

from ...utils.log import logger

MODE_TO_SPLIT = {"Train": 0, "Eval": 1, "Test": 2}


def _helpers():
    """The native index builder; compiled on first use by local rank 0."""
    try:
        from ..data_tools.cpp import fast_index_map_helpers as h
        return h
    except ImportError:
        from ...ops.build import build_data_helper

        if int(os.environ.get("LOCAL_RANK", "0")) == 0:
            build_data_helper(verbose=False)
        for _ in range(120):
            try:
                import importlib

                import paddlefleetx_b200.data.data_tools.cpp as pkg
                importlib.invalidate_caches()
                from ..data_tools.cpp import fast_index_map_helpers as h  # noqa: F811
                return h
            except ImportError:
                time.sleep(1)
        raise


def train_valid_test_split(split: Sequence[float], size: int) -> List[int]:
    w = [float(s) for s in split][:3]
    w += [0.0] * (3 - len(w))
    total = sum(w)
    assert total > 0
    bounds = [0]
    for x in w:
        bounds.append(bounds[-1] + int(round(x / total * float(size))))
    diff = bounds[-1] - size
    bounds = [bounds[0]] + [b - diff for b in bounds[1:]]
    assert bounds[-1] == size
    return bounds


def find_corpus_prefix(input_dir: str) -> str:
    names = sorted(f for f in os.listdir(input_dir) if f.endswith("_idx.npz"))
    if names:
        return os.path.join(input_dir, names[0][:-len("_idx.npz")])
    legacy = sorted(f for f in os.listdir(input_dir) if f.endswith("_ids.npz"))
    if legacy:
        return os.path.join(input_dir, legacy[0][:-len("_ids.npz")])
    raise RuntimeError(f"no xxx_ids.npy / xxx_idx.npz corpus found in {input_dir!r}")


def get_train_data_file(input_dir: str) -> List[str]:
    """Prefixes of every corpus in ``input_dir`` (``<prefix>_ids.npy`` + ``<prefix>_idx.npz``; falls back to the legacy single-file
    ``<prefix>_ids.npz``) — the reference's lookup (gpt_dataset.py:220-247); ``find_corpus_prefix`` is "the first of these"."""
    names = sorted(f for f in os.listdir(input_dir) if f.endswith("_idx.npz") and os.path.isfile(os.path.join(input_dir, f)))
    if names:
        return [os.path.join(input_dir, n[:-len("_idx.npz")]) for n in names]
    logger.warning("Not found dataset with name of xxx_ids.npy and xxx_idx.npz! Try to found old compatible xxx_ids.npz file.")
    legacy = sorted(f for f in os.listdir(input_dir) if f.endswith("_ids.npz") and os.path.isfile(os.path.join(input_dir, f)))
    if not legacy:
        raise RuntimeError(f"Not found dataset with name of xxx_ids.npz in given input_dir '{input_dir}'! ")
    return [os.path.join(input_dir, n[:-len("_ids.npz")]) for n in legacy]


get_train_valid_test_split_ = train_valid_test_split          # reference name (gpt_dataset.py:250-271)


class TokenCorpus:
    """Flat token stream + per-document lengths."""

    def __init__(self, prefix: str):
        if os.path.isfile(prefix + "_ids.npz"):
            blob = np.load(prefix + "_ids.npz", mmap_mode="r+", allow_pickle=True)
            self.ids, self.lens = blob["ids"], blob["lens"].astype("int32")
        else:
            for suffix in ("_ids.npy", "_idx.npz"):
                if not os.path.isfile(prefix + suffix):
                    raise ValueError(f"File Not found, {prefix + suffix}")
            self.ids = np.load(prefix + "_ids.npy", mmap_mode="r", allow_pickle=True)
            self.lens = np.load(prefix + "_idx.npz")["lens"].astype("int32")
        self.starts = np.concatenate([[0], np.cumsum(self.lens, dtype=np.int64)])

    def doc_tokens(self, doc: int, lo: int = 0, hi: Optional[int] = None) -> np.ndarray:
        s = self.starts[doc]
        e = self.starts[doc + 1] if hi is None else s + hi
        return np.asarray(self.ids[s + lo:e])


def _num_epochs(tokens_per_epoch: int, seq_len: int, num_samples: int) -> int:
    n = 1
    while (n * tokens_per_epoch - 1) // seq_len < num_samples:
        n += 1
    return n


def _doc_order(documents: np.ndarray, num_epochs: int, rng: np.random.RandomState, separate_last: bool) -> np.ndarray:
    if not separate_last or num_epochs == 1:
        order = np.tile(documents.astype(np.int32), num_epochs)
        rng.shuffle(order)
        return order
    return np.concatenate([_doc_order(documents, num_epochs - 1, rng, False), _doc_order(documents, 1, rng, False)])


def _shuffle_order(n_first: int, total: int, rng: np.random.RandomState) -> np.ndarray:
    dtype = np.uint32 if total < np.iinfo(np.uint32).max - 1 else np.int64
    first = np.arange(n_first, dtype=dtype)
    rng.shuffle(first)
    if n_first == total:
        return first
    last = np.arange(n_first, total, dtype=dtype)
    rng.shuffle(last)
    return np.concatenate([first, last])


def document_positions(piece_lengths: Sequence[int], n: int) -> np.ndarray:
    """Position ids of the first ``n`` tokens of a sample made of consecutive document pieces of the given lengths: 0, 1, ... restarting
    at every piece."""
    lens = np.asarray(piece_lengths, dtype=np.int64)
    starts = np.concatenate([[0], np.cumsum(lens)[:-1]])
    return (np.arange(int(lens.sum()), dtype=np.int64) - np.repeat(starts, lens))[:n]


def python_sample_idx(sizes: np.ndarray, doc_idx: np.ndarray, seq_len: int, num_epochs: int, tokens_per_epoch: int) -> np.ndarray:
    """Pure-python twin of the C++ ``build_sample_idx`` (used as its test oracle and as a fallback)."""
    n = (num_epochs * tokens_per_epoch - 1) // seq_len
    out = np.zeros((n + 1, 2), dtype=np.int64)
    d, off = 0, 0
    for s in range(1, n + 1):
        need = seq_len + 1
        while need > 0:
            avail = int(sizes[doc_idx[d]]) - off
            if avail >= need:
                off += need - 1
                need = 0
            else:
                need -= avail
                d, off = d + 1, 0
        out[s] = (d, off)
    return out


def build_index_files(name: str, prefix: str, documents: np.ndarray, sizes: np.ndarray, num_samples: int, seq_len: int, seed: int,
                      build: bool):
    tokens_per_epoch = int(np.sum(sizes[documents]))
    num_epochs = _num_epochs(tokens_per_epoch, seq_len, num_samples)
    base = f"{prefix}_{name}_indexmap_{num_samples}ns_{seq_len}sl"
    paths = [base + s for s in ("_doc_idx.npy", "_sample_idx.npy", "_shuffle_idx.npy")]
    if build and not all(os.path.isfile(p) for p in paths):
        rng = np.random.RandomState(seed=seed)
        separate_last = False
        n_before_last = 0
        if num_epochs > 1:
            n_before_last = ((num_epochs - 1) * tokens_per_epoch - 1) // seq_len
            last = num_samples - n_before_last
            per_epoch = (tokens_per_epoch - 1) // seq_len
            assert 0 <= last < per_epoch + 1, "last epoch sample count out of range"
            separate_last = last < int(0.80 * per_epoch)
        t0 = time.time()
        doc_idx = _doc_order(documents, num_epochs, rng, separate_last)
        np.save(paths[0], doc_idx, allow_pickle=True)
        sample_idx = _helpers().build_sample_idx(sizes.astype(np.int32), doc_idx, seq_len, num_epochs, tokens_per_epoch)
        np.save(paths[1], sample_idx, allow_pickle=True)
        total = sample_idx.shape[0] - 1
        shuffle_idx = _shuffle_order(n_before_last if separate_last else total, total, rng)
        np.save(paths[2], shuffle_idx, allow_pickle=True)
        logger.info(f"built GPT index maps for {name} in {time.time() - t0:.2f}s ({total} samples, {num_epochs} epochs)")
    else:
        while not all(os.path.isfile(p) for p in paths):
            time.sleep(1)
        for _ in range(60):
            try:
                np.load(paths[2], allow_pickle=True, mmap_mode="r")
                break
            except (OSError, ValueError, EOFError):  # still being written
                time.sleep(1)
    import torch.distributed as dist

    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        dist.barrier()          # a failing barrier must surface: continuing would leave the ranks with different views of the cache
    return tuple(np.load(p, allow_pickle=True, mmap_mode="r") for p in paths)


def construct_samples_and_shuffle_data(name, data_prefix, documents, sizes, num_samples, seq_length, seed, build_data_file):
    """``(doc_idx, sample_idx, shuffle_idx)`` for one split, built (or awaited) and cached next to the corpus as
    ``<prefix>_<name>_indexmap_<ns>ns_<sl>sl_{doc,sample,shuffle}_idx.npy`` — the reference entry point (gpt_dataset.py:274-393)."""
    return build_index_files(name, data_prefix, np.asarray(documents), np.asarray(sizes), num_samples, seq_length, seed, build_data_file)


class GPTDataset(torch.utils.data.Dataset):
    def __init__(self, input_dir: str, split: Sequence[float], max_seq_len: int, num_samples: int, mode: str, model_type: str = "GPT",
                 seed: int = 1234, eos_id: int = 50256, mask_eos: bool = False, reset_position_ids: bool = False, **unused):
        if mode not in MODE_TO_SPLIT:
            raise ValueError("valid str value for 'mode'")
        prefix = find_corpus_prefix(input_dir)
        self.corpus = TokenCorpus(prefix)
        bounds = train_valid_test_split(split, len(self.corpus.lens))
        k = MODE_TO_SPLIT[mode]
        documents = np.arange(bounds[k], bounds[k + 1])
        self.mode, self.max_seq_len, self.eos_id, self.mask_eos = mode, max_seq_len, eos_id, mask_eos
        self.reset_position_ids = reset_position_ids
        self.name = "gpt_" + mode
        local_rank = int(os.environ.get("LOCAL_RANK", os.environ.get("PADDLE_RANK_IN_NODE", 0)))
        self.doc_idx, self.sample_idx, self.shuffle_idx = build_index_files(
            self.name, prefix, documents, self.corpus.lens, num_samples, max_seq_len, seed, build=(local_rank == 0))

    def __len__(self) -> int:
        return self.sample_idx.shape[0] - 1

    def _tokens(self, idx: int) -> np.ndarray:
        d0, o0 = self.sample_idx[idx]
        d1, o1 = self.sample_idx[idx + 1]
        if d0 == d1:
            return self.corpus.doc_tokens(int(self.doc_idx[d0]), int(o0), int(o1) + 1)
        parts = [self.corpus.doc_tokens(int(self.doc_idx[d0]), int(o0))]
        parts += [self.corpus.doc_tokens(int(self.doc_idx[d])) for d in range(int(d0) + 1, int(d1))]
        parts.append(self.corpus.doc_tokens(int(self.doc_idx[d1]), 0, int(o1) + 1))
        return np.concatenate(parts)

    def _piece_lengths(self, idx: int) -> List[int]:
        """Lengths of the document pieces that ``_tokens(idx)`` concatenates."""
        d0, o0 = (int(x) for x in self.sample_idx[idx])
        d1, o1 = (int(x) for x in self.sample_idx[idx + 1])
        if d0 == d1:
            return [o1 + 1 - o0]
        lens = self.corpus.lens
        return [int(lens[self.doc_idx[d0]]) - o0] + [int(lens[self.doc_idx[d]]) for d in range(d0 + 1, d1)] + [o1 + 1]

    def __getitem__(self, index: int):
        idx = int(self.shuffle_idx[index])
        seq = self._tokens(idx).astype(np.int64)
        tokens, labels = seq[:-1], seq[1:]
        if self.reset_position_ids:
            position_ids = document_positions(self._piece_lengths(idx), len(tokens))
        else:
            position_ids = np.arange(len(tokens), dtype=np.int64)
        if self.mode == "Test":
            return [tokens, position_ids]
        loss_mask = np.ones(len(tokens), dtype=np.float32)
        if self.mask_eos:
            loss_mask[tokens == self.eos_id] = 0.0
        return [tokens, position_ids, labels, loss_mask]


class SyntheticGPTDataset(torch.utils.data.Dataset):
    """Uniform-random token ids with the GPTDataset sample contract; deterministic per index.  ``document_length`` > 0 packs each sample
    from documents of seeded random lengths in ``[ceil(L / 2), L + L // 2]``; with ``reset_position_ids`` their position ids restart at
    every document (see ``GPTDataset``)."""

    def __init__(self, max_seq_len: int = 1024, vocab_size: int = 50304, num_samples: int = 1 << 20, mode: str = "Train", seed: int = 1234,
                 eos_id: int = 50256, reset_position_ids: bool = False, document_length: int = 0, **unused):
        self.max_seq_len, self.vocab_size, self.num_samples, self.mode, self.seed = max_seq_len, vocab_size, int(num_samples), mode, seed
        self.reset_position_ids, self.document_length = reset_position_ids, int(document_length or 0)

    def document_lengths(self, index: int) -> List[int]:
        """The lengths of the documents packed into sample ``index`` (one document when ``document_length`` is 0)."""
        n, L = self.max_seq_len + 1, self.document_length
        if L <= 0:
            return [n]
        rng = np.random.default_rng([self.seed, index, 1])
        lens = rng.integers(-(-L // 2), L + L // 2 + 1, size=n // max(1, -(-L // 2)) + 1)
        cut = int(np.searchsorted(np.cumsum(lens), n))
        lens = lens[:cut + 1].tolist()
        lens[-1] = n - sum(lens[:-1])
        return lens

    def __len__(self) -> int:
        return self.num_samples

    def __getitem__(self, index: int):
        rng = np.random.default_rng(self.seed * 1000003 + index)
        seq = rng.integers(0, self.vocab_size, size=self.max_seq_len + 1, dtype=np.int64)
        tokens, labels = seq[:-1], seq[1:]
        if self.reset_position_ids:
            position_ids = document_positions(self.document_lengths(index), self.max_seq_len)
        else:
            position_ids = np.arange(self.max_seq_len, dtype=np.int64)
        if self.mode == "Test":
            return [tokens, position_ids]
        return [tokens, position_ids, labels, np.ones(self.max_seq_len, dtype=np.float32)]


# ------------------------------------------------------------------------------------ offline evaluation sets
def wikitext_detokenize(text: str) -> str:
    """Undo the WikiText tokenisation artefacts before BPE (reference ``_wikitext_detokenizer``)."""
    import re

    rules = [("s '", "s'"), (" @-@ ", "-"), (" @,@ ", ","), (" @.@ ", "."), (" : ", ": "), (" ; ", "; "), (" . ", ". "),
             (" ! ", "! "), (" ? ", "? "), (" , ", ", "), ("= = = =", "===="), ("= = =", "==="), ("= =", "=="),
             (" " + chr(176) + " ", chr(176)), (" \n", "\n"), ("\n ", "\n"), (" N ", " 1 "), (" 's", "'s")]
    out = text
    for a, b in rules[:1]:
        out = out.replace(a, b)
    out = re.sub(r"/' [0-9]/", r"/'[0-9]/", out)
    for a, b in rules[1:10]:
        out = out.replace(a, b)
    out = re.sub(r"\(\s*([^\)]*?)\s*\)", r"(\1)", out)
    out = re.sub(r"\[\s*([^\]]*?)\s*\]", r"[\1]", out)
    out = re.sub(r"{\s*([^}]*?)\s*}", r"{\1}", out)
    out = re.sub(r"\"\s*([^\"]*?)\s*\"", r'"\1"', out)
    out = re.sub(r"'\s*([^']*?)\s*'", r"'\1'", out)
    for a, b in rules[10:]:
        out = out.replace(a, b)
    return out


def _default_eval_tokenizer(vocab_dir=None):
    """The evaluation sets tokenise raw text themselves (reference gpt_dataset.py:484-655 builds ``GPTTokenizer.from_pretrained("gpt2")``);
    offline boxes without the GPT-2 vocabulary fall back to the byte-level vocabulary with a warning (scores are then not comparable)."""
    from ..tokenizers.gpt_tokenizer import GPTTokenizer
    from ...utils.log import logger

    try:
        return GPTTokenizer.from_pretrained(vocab_dir or "gpt2")
    except FileNotFoundError as exc:
        logger.warning(f"{exc}  Falling back to the byte-level tokenizer for evaluation.")
        return GPTTokenizer.byte_fallback()


class LM_Eval_Dataset(torch.utils.data.Dataset):
    """Sliding-window perplexity set: windows of ``max_seq_len`` advanced by ``overlapping_eval``; only the last
    ``overlapping_eval`` targets of every non-first window are scored (reference gpt_dataset.py:484-560)."""

    def __init__(self, input_dir: str, max_seq_len: int, overlapping_eval: Optional[int] = None, tokenizer=None, eos_id: Optional[int] = None,
                 tokens: Optional[Sequence[int]] = None, **unused):
        if tokens is None:
            with open(input_dir, "rb") as fh:
                raw = fh.read().decode("utf-8")
            self.num_original_tokens = len(raw.strip().split(" "))
            tokenizer = tokenizer or _default_eval_tokenizer(unused.get("vocab_dir"))
            tokens = tokenizer.encode(wikitext_detokenize(raw))
        else:
            self.num_original_tokens = len(tokens)
        self.tokens = list(tokens)
        self.seq_len = max_seq_len
        # pad id of the last (short) window: explicit > the tokenizer's end-of-text id > GPT-2's 50256
        self.pad_idx = eos_id if eos_id is not None else getattr(tokenizer, "eos_token_id", None) or 50256
        self.overlapping_eval = overlapping_eval or max_seq_len
        self.overlapping_eval = max(1, self.overlapping_eval)
        self.num_tokenized_tokens = len(self.tokens)
        targets = max(len(self.tokens) - 1 - self.overlapping_eval, 0)
        self.total_sequences = max((targets + self.overlapping_eval - 1) // self.overlapping_eval + 1, 1)

    def __len__(self) -> int:
        return self.total_sequences

    def __getitem__(self, idx: int):
        start = idx * self.overlapping_eval
        window = self.tokens[start:start + self.seq_len + 1]
        n = len(window)
        window = window + [self.pad_idx] * (self.seq_len + 1 - n)
        seq = np.asarray(window, dtype=np.int64)
        tokens, labels = seq[:-1], seq[1:]
        loss_mask = np.zeros(self.seq_len, dtype=np.float32)
        loss_mask[:max(n - 1, 0)] = 1.0
        if self.overlapping_eval != self.seq_len and idx != 0:
            loss_mask[:-self.overlapping_eval] = 0.0
        position_ids = np.arange(self.seq_len, dtype=np.int64)
        attention_mask = np.tril(np.ones((1, self.seq_len, self.seq_len), dtype=np.float32))
        return [tokens, loss_mask, attention_mask, position_ids, labels, np.array([self.num_original_tokens, self.num_tokenized_tokens])]


class Lambada_Eval_Dataset(torch.utils.data.Dataset):
    """LAMBADA last-word cloze (strict): context tokens + the BPE pieces of ``' ' + last_word``; a sample is
    correct iff every piece is the arg-max (reference gpt_dataset.py:563-655)."""

    def __init__(self, input_dir: str, max_seq_len: int, tokenizer=None, eos_id: Optional[int] = None, samples: Optional[list] = None, **unused):
        if samples is None:
            tokenizer = tokenizer or _default_eval_tokenizer(unused.get("vocab_dir"))
        self.seq_len = max_seq_len
        self.pad_idx = eos_id if eos_id is not None else getattr(tokenizer, "eos_token_id", None) or 50256
        self.tokens, self.labels = [], []
        if samples is not None:
            for ctx, tgt in samples:
                self.tokens.append(list(ctx)); self.labels.append(list(tgt))
        else:
            import json

            with open(input_dir, "r", encoding="utf-8") as fh:
                for line in fh:
                    text = json.loads(line)["text"]
                    last = text.split()[-1]
                    start = text.rfind(last)
                    self.tokens.append(tokenizer.encode(text[:start].strip()))
                    self.labels.append(tokenizer.encode(" " + last))

    def __len__(self) -> int:
        return len(self.tokens)

    def __getitem__(self, idx: int):
        ctx, tgt = self.tokens[idx], self.labels[idx]
        seq = (ctx + tgt)[: self.seq_len + 1]
        n = len(seq)
        seq = seq + [self.pad_idx] * (self.seq_len + 1 - n)
        arr = np.asarray(seq, dtype=np.int64)
        tokens, labels = arr[:-1], arr[1:]
        loss_mask = np.zeros(self.seq_len, dtype=np.float32)
        loss_mask[len(ctx) - 1:n - 1] = 1.0
        position_ids = np.arange(self.seq_len, dtype=np.int64)
        attention_mask = np.tril(np.ones((1, self.seq_len, self.seq_len), dtype=np.float32))
        return [tokens, loss_mask, attention_mask, position_ids, labels, np.array([len(self), len(self)])]
