"""Attention front-end.

``attention(q, k, v)`` takes ``[b, s, heads, d]`` tensors (views are fine: the slices of a packed QKV projection, sequence-major
storage).  k and v may have fewer heads than q (grouped-query attention: ``heads % kv_heads == 0``, query head ``h`` attends with K/V
head ``h // (heads // kv_heads)``, the convention of ``repeat_interleave``).  Path selection on CUDA / bf16 or fp16 (q, k and v of one
dtype):
  * training and inference at head_dim 128 or 64: our wgmma flash kernels — ``csrc/attention_fwd_sm90.cu`` and
    ``csrc/attention_bwd_sm90.cu`` — with in-kernel causal masking and counter-hash dropout (the backward regenerates the mask; nothing is
    stored).  ``flash_attention_packed`` is the same pair for the ``[b, s, heads, 3, d]`` output of a fused QKV projection (``[b, s,
    kv_heads, G + 2, d]`` with grouped K/V: the G query heads of a group, then its key and value): it reads q / k / v in place and writes
    ONE packed gradient, so no split / cat copies surround the kernels,
  * single-query decode steps over the static KV cache use ``csrc/attention_decode.cu`` (see models/.../gpt/model.py),
  * packed documents (``DocumentMask``: query ``i`` attends keys ``[key_start[b, i], i]``): the same kernels, in separate
    instantiations that skip the key tiles outside a query tile's documents; other head sizes, fp32 and CPU tensors run the dense
    boolean form of the mask through SDPA,
  * bidirectional key padding (``KeyPaddingMask``: every query of row ``b`` attends the valid keys of row ``b``, as ERNIE's padding mask):
    separate non-causal multi-head instantiations that never load the key tiles past the last valid key; grouped K/V heads, other head
    sizes, fp32 and CPU tensors run the mask's additive ``[b, 1, 1, s]`` form through SDPA,
  * explicit masks, other head sizes, mixed dtypes, fp32 and CPU tensors: PyTorch SDPA — a *library* call, reported as such by the launch
    accounting (it does not count towards ``gpu_launches``); ``PFX_NATIVE_ATTN=0`` forces it everywhere,
  * the unfused reference path (QK^T -> fused causal softmax -> PV) used when ``use_flash_attn=False`` — this mirrors reference
    ``core_attn`` (hybrid_model.py:303-346).
"""
from __future__ import annotations

from typing import Optional

import os

import torch
import torch.nn.functional as F

# 1 (default) = our kernels wherever they apply, 0 = library SDPA everywhere (A/B runs, debugging)
_NATIVE = int(os.environ.get("PFX_NATIVE_ATTN", "1"))
_MASK64 = (1 << 64) - 1


def _q_heads(q: torch.Tensor) -> int:
    """Query heads of ``[b, s, heads, d]`` or of the ``[b, s, kv_heads, G, d]`` query part of a grouped packed projection."""
    return q.shape[2] * q.shape[3] if q.dim() == 5 else q.shape[2]


class DocumentMask:
    """Causal attention that stays inside each document of a packed sequence: query ``i`` of batch row ``b`` attends the keys
    ``[key_start[b, i], i]`` (self-attention, ``sq == sk``).  No ``[s, s]`` tensor is built for the native kernels; they read

      * ``key_start`` int32 ``[b, s]``, clamped into ``[0, i]``,
      * ``tile_min`` / ``tile_max`` int32 ``[b, ceil(s / 64)]``: its minimum / maximum over each 64-query tile, from which the
        forward and backward kernels skip whole key tiles.

    Build it once per forward pass (``from_positions`` / ``from_key_start``) and hand the same object to every layer: on CUDA the
    derivation is one native launch.  ``dense()`` / ``additive()`` give the equivalent ``[b, 1, s, s]`` mask for the paths that take
    an explicit mask (SDPA, ``core_attention``)."""

    TILE = 64

    def __init__(self, key_start: torch.Tensor, tile_min: torch.Tensor, tile_max: torch.Tensor):
        self.key_start, self.tile_min, self.tile_max = key_start, tile_min, tile_max

    @classmethod
    def _build(cls, src: torch.Tensor, from_positions: bool) -> "DocumentMask":
        if src.dim() != 2:
            raise ValueError(f"DocumentMask expects [batch, seq] ids, got shape {tuple(src.shape)}")
        src = src.to(torch.int64).contiguous()
        b, s = src.shape
        if src.is_cuda:
            from . import _native
            from . import functional as OF

            ks, tmin, tmax = _native.require().attention_doc_bounds(src, bool(from_positions))
            OF._count()
            return cls(ks, tmin, tmax)
        i = torch.arange(s, dtype=torch.int64, device=src.device)
        ks = (i - src) if from_positions else src
        return cls.with_tile_bounds(torch.minimum(ks.clamp_min(0), i).to(torch.int32))

    @classmethod
    def with_tile_bounds(cls, key_start: torch.Tensor) -> "DocumentMask":
        """The mask of int32 ``key_start`` ``[b, sq]`` taken as it is, with its per-tile minimum / maximum computed in PyTorch."""
        b, s = key_start.shape
        t = -(-s // cls.TILE)
        pad = t * cls.TILE - s
        lo = torch.nn.functional.pad(key_start, (0, pad), value=torch.iinfo(torch.int32).max).view(b, t, cls.TILE).amin(-1)
        hi = torch.nn.functional.pad(key_start, (0, pad), value=0).view(b, t, cls.TILE).amax(-1)
        return cls(key_start, lo, hi)

    @classmethod
    def from_positions(cls, position_ids: torch.Tensor) -> "DocumentMask":
        """Position ids that restart at 0 at each document start: ``key_start = clamp(i - position_ids[b, i], 0, i)``."""
        return cls._build(position_ids, True)

    @classmethod
    def from_key_start(cls, key_start: torch.Tensor) -> "DocumentMask":
        """Explicit first attended key per query (clamped into ``[0, i]``)."""
        return cls._build(key_start, False)

    @property
    def shape(self):
        return tuple(self.key_start.shape)

    def dense(self) -> torch.Tensor:
        """bool ``[b, 1, s, s]``, True where query ``i`` may attend key ``j``: ``key_start[b, i] <= j <= i``."""
        s = self.key_start.shape[1]
        j = torch.arange(s, device=self.key_start.device)
        ks = self.key_start.to(torch.int64).unsqueeze(-1)
        return ((j.view(1, 1, s) >= ks) & (j.view(1, 1, s) <= j.view(1, s, 1))).unsqueeze(1)

    def additive(self, dtype=torch.float32) -> torch.Tensor:
        """``dense()`` as an additive mask: 0 where attended, ``-inf`` elsewhere (every row keeps its diagonal)."""
        m = self.dense()
        return torch.zeros(m.shape, dtype=dtype, device=m.device).masked_fill_(~m, float("-inf"))

    def bounds(self):
        return self.key_start, self.tile_min, self.tile_max


class KeyPaddingMask:
    """Bidirectional attention over the valid keys of each batch row: every query of row ``b`` attends key ``j`` iff ``valid[b, j]``.  A
    row without any valid key attends every key, which is what the additive ``-1e4`` mask gives (one constant added to every logit of a
    row leaves its softmax unchanged).  Any pattern is exact; the native kernels read

      * ``key_bits`` int32 ``[b, ceil(s / 32)]``: the validity bits, 32 keys per word (bit ``j % 32`` of word ``j // 32``),
      * ``key_end`` int32 ``[b]``: 1 + the last valid key; key tiles at or past it are never loaded,
      * ``key_dense`` int32 ``[b]``: the first invalid key; key tiles entirely below it need no per-element compare.

    Build it once per forward pass (``from_valid`` / ``from_ids``) and hand the same object to every layer: on CUDA the derivation is
    one native launch.  ``additive()`` gives the ``[b, 1, 1, s]`` tensor that the explicit-mask paths (SDPA, ``core_attention``) add to
    the logits, built by the same formula as ERNIE's padding mask, in ``dtype``."""

    WORD = 32
    _NATIVE_DTYPES = (torch.bool, torch.uint8, torch.int32, torch.int64, torch.float32, torch.float16, torch.bfloat16)   # read by the bounds kernel

    def __init__(self, key_bits: torch.Tensor, key_end: torch.Tensor, key_dense: torch.Tensor, src: torch.Tensor, from_ids: bool,
                 pad_id: int, dtype: torch.dtype):
        self.key_bits, self.key_end, self.key_dense = key_bits, key_end, key_dense
        self._src, self._from_ids, self._pad_id, self.dtype = src, from_ids, pad_id, dtype

    @classmethod
    def _build(cls, src: torch.Tensor, from_ids: bool, pad_id: int, dtype) -> "KeyPaddingMask":
        if src.dim() != 2 or src.shape[0] < 1 or src.shape[1] < 1:
            raise ValueError(f"KeyPaddingMask expects a [batch, seq] tensor, got shape {tuple(src.shape)}")
        if from_ids and src.dtype not in (torch.int32, torch.int64):
            raise ValueError(f"KeyPaddingMask.from_ids expects int32 / int64 ids, got {src.dtype}")
        if src.is_cuda:
            from . import _native
            from . import functional as OF

            native = src if from_ids or src.dtype in cls._NATIVE_DTYPES else src != 0
            bits, end, dense = _native.require().attention_key_pad_bounds(native.contiguous(), bool(from_ids), int(pad_id))
            OF._count()
            return cls(bits, end, dense, src, from_ids, pad_id, dtype)
        valid = (src != pad_id) if from_ids else (src != 0)
        b, s = valid.shape
        i = torch.arange(s, device=src.device)
        last = torch.where(valid, i, -1).amax(-1)
        first_bad = torch.where(valid, s, i).amin(-1)
        empty = last < 0
        valid = valid | empty.unsqueeze(-1)
        end = torch.where(empty, s, last + 1).to(torch.int32)
        dense = torch.where(empty, s, first_bad).to(torch.int32)
        w = -(-s // cls.WORD)
        padded = torch.nn.functional.pad(valid, (0, w * cls.WORD - s)).view(b, w, cls.WORD).to(torch.int64)
        words = (padded << torch.arange(cls.WORD, device=src.device)).sum(-1)
        bits = torch.where(words >= 1 << 31, words - (1 << 32), words).to(torch.int32)      # the uint32 words, stored as int32
        return cls(bits, end, dense, src, from_ids, pad_id, dtype)

    @classmethod
    def from_valid(cls, mask: torch.Tensor, dtype=torch.float32) -> "KeyPaddingMask":
        """``[b, s]`` validity (bool, integers or 0 / 1 floats; nonzero = a real token).  ``additive()`` is ``(1 - mask) * -1e4``."""
        return cls._build(mask, False, 0, dtype)

    @classmethod
    def from_ids(cls, input_ids: torch.Tensor, pad_id: int, dtype=torch.float32) -> "KeyPaddingMask":
        """``[b, s]`` token ids; keys equal to ``pad_id`` are padding.  ``additive()`` is ``(input_ids == pad_id) * -1e4``."""
        return cls._build(input_ids, True, int(pad_id), dtype)

    @property
    def shape(self):
        return tuple(self._src.shape)

    def dense(self) -> torch.Tensor:
        """bool ``[b, 1, 1, s]``, True where a key is attended (every key of a row without valid keys)."""
        s = self._src.shape[1]
        j = torch.arange(s, device=self.key_bits.device)
        words = self.key_bits.to(torch.int64)[:, j // self.WORD]
        return ((words >> (j % self.WORD)) & 1).bool()[:, None, None, :]

    def additive(self, dtype=None) -> torch.Tensor:
        """The ``[b, 1, 1, s]`` additive mask (0 for valid keys, -1e4 for padding) in ``dtype`` (default: the dtype the mask was built
        for), bit for bit the tensor ERNIE has always added to its logits."""
        dtype = self.dtype if dtype is None else dtype
        if self._from_ids:
            return (self._src == self._pad_id)[:, None, None, :].to(dtype) * -1e4
        return (1.0 - self._src[:, None, None, :].to(dtype)) * -1e4

    def bounds(self):
        return self.key_bits, self.key_end, self.key_dense


def _native_ok(q, k, v, attn_mask, causal, needs_grad: bool, doc: Optional[DocumentMask] = None,
               pad: Optional[KeyPaddingMask] = None) -> bool:
    from .functional import tensor_core_dtype

    if not _NATIVE or attn_mask is not None or not q.is_cuda or not tensor_core_dtype(q, k, v):
        return False
    d = q.shape[-1]
    if d not in (64, 128) or q.shape[1] < 1 or (causal and k.shape[1] < q.shape[1]):
        return False
    if doc is not None and ((causal and k.shape[1] != q.shape[1]) or doc.shape != (q.shape[0], q.shape[1]) or not doc.key_start.is_cuda):
        return False
    if pad is not None and (causal or q.dim() != 4 or k.shape[2] != q.shape[2] or pad.shape != (k.shape[0], k.shape[1])
                            or not pad.key_bits.is_cuda):
        return False
    if k.dim() != 4 or v.shape != k.shape or _q_heads(q) % k.shape[2] or (q.dim() == 5 and q.shape[2] != k.shape[2]):
        return False
    for t in (q, k, v):
        if t.dim() not in (4, 5) or t.stride(-1) != 1 or any(t.stride(i) % 8 for i in range(t.dim() - 1)) or t.data_ptr() % 16:
            return False
    from . import _native

    return _native.available()


def _dropout_seed(dropout_p: float, numel: int) -> int:
    if dropout_p <= 0.0:
        return 0
    from ..parallel.rng import get_rng_state_tracker

    seed, offset = get_rng_state_tracker().philox(numel)           # advances the active stream: recompute replays the same pair
    return ((int(seed) * 0x9E3779B97F4A7C15) ^ (int(offset) * 0xD1B54A32D192ED03 + 0x2545F4914F6CDD1D)) & 0x7FFFFFFFFFFFFFFF


def attn_keep_mask(seed: int, B: int, H: int, Sq: int, Sk: int, p: float, device) -> torch.Tensor:
    """The keep mask ``[B, H, Sq, Sk]`` (bool) our kernels generate for ``seed`` — a pure-PyTorch replica of csrc/pfx_attn.cuh used by
    the numerics tests (fp32 reference with the SAME dropout pattern)."""
    M = 0xFFFFFFFF

    def mix(x):
        x = x ^ (x >> 16); x = (x * 0x85EBCA6B) & M; x = x ^ (x >> 13); x = (x * 0xC2B2AE35) & M; x = x ^ (x >> 16)
        return x

    bh = torch.arange(B * H, device=device, dtype=torch.int64)
    key = mix(((seed & M) + 0x9E3779B9 * (bh + 1)) & M) ^ ((seed >> 32) & M)             # [BH]
    pairs = (Sk + 1) // 2
    q = torch.arange(Sq, device=device, dtype=torch.int64).view(1, Sq, 1)
    kp = torch.arange(pairs, device=device, dtype=torch.int64).view(1, 1, pairs)
    x = (q * pairs + kp) & M
    x = x ^ (x >> 16); x = (x * 0x85EBCA6B) & M
    x = x ^ key.view(-1, 1, 1)
    x = x ^ (x >> 13); x = (x * 0xC2B2AE35) & M; x = x ^ (x >> 16)
    thresh = int(p * 65536.0 + 0.5)
    even, odd = (x & 0xFFFF) >= thresh, (x >> 16) >= thresh
    keep = torch.stack([even, odd], dim=-1).reshape(B * H, Sq, 2 * pairs)[:, :, :Sk]
    return keep.view(B, H, Sq, Sk)


def _split_packed(mix: torch.Tensor):
    """q / k / v views of a ``[b, s, kv_heads, G + 2, d]`` projection output: q is ``[b, s, heads, d]`` for G = 1 (the ``[.., 3, d]``
    layout) and ``[b, s, kv_heads, G, d]`` otherwise (no uniform head stride; the kernels take it as it is)."""
    g = mix.shape[3] - 2
    if g == 1:
        return mix.unbind(3)
    return mix[:, :, :, :g], mix[:, :, :, g], mix[:, :, :, g + 1]


class _FlashAttnFn(torch.autograd.Function):
    """q / k / v ``[b, s, h, d]`` views (k / v may have fewer heads) -> ``[b, s, h, d]``.  ``packed`` = the three are slices of one
    ``[b, s, kv_heads, G + 2, d]`` tensor, which is then the single differentiable input (and the single gradient: dq / dk / dv are
    written straight into its slices)."""

    @staticmethod
    def forward(ctx, packed, q, k, v, causal, scale, dropout_p, seed, doc=None):
        from . import _native
        from . import functional as OF

        if packed is not None:
            q, k, v = _split_packed(packed)
        if isinstance(doc, KeyPaddingMask):
            out, lse = _native.require().attention_fwd_keypad(q, k, v, *doc.bounds(), float(scale), float(dropout_p), int(seed))
        elif doc is not None:
            out, lse = _native.require().attention_fwd_doc(q, k, v, *doc.bounds(), float(scale), float(dropout_p), int(seed), bool(causal))
        else:
            out, lse = _native.require().attention_fwd_v2(q, k, v, bool(causal), float(scale), float(dropout_p), int(seed))
        OF._count()
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.cfg = (packed is not None, bool(causal), float(scale), float(dropout_p), int(seed))
        ctx.doc = doc            # the tile (or key-padding) bounds of the forward serve the backward
        return out

    @staticmethod
    def backward(ctx, dout):
        from . import _native
        from . import functional as OF

        q, k, v, out, lse = ctx.saved_tensors
        is_packed, causal, scale, dropout_p, seed = ctx.cfg
        if dout.stride(3) != 1 or any(dout.stride(i) % 8 for i in range(3)):
            dout = dout.contiguous()
        dmix = None
        if is_packed:
            b, s, hkv, d = k.shape
            dmix = torch.empty(b, s, hkv, _q_heads(q) // hkv + 2, d, dtype=q.dtype, device=q.device)
            dq, dk, dv = _split_packed(dmix)
        else:
            dq, dk, dv = torch.empty_like(q, memory_format=torch.contiguous_format), torch.empty_like(k, memory_format=torch.contiguous_format), \
                torch.empty_like(v, memory_format=torch.contiguous_format)
        if isinstance(ctx.doc, KeyPaddingMask):
            _native.require().attention_bwd_keypad(q, k, v, out, dout, lse, dq, dk, dv, *ctx.doc.bounds(), scale, dropout_p, seed)
        elif ctx.doc is not None:
            _native.require().attention_bwd_doc(q, k, v, out, dout, lse, dq, dk, dv, *ctx.doc.bounds(), scale, dropout_p, seed, causal)
        else:
            _native.require().attention_bwd(q, k, v, out, dout, lse, dq, dk, dv, causal, scale, dropout_p, seed)
        OF._count(4)           # memset is a driver call; prep + main + dq convert (+ the tensor-core kernel counted once more for its size)
        if is_packed:
            return dmix, None, None, None, None, None, None, None, None
        return None, dq, dk, dv, None, None, None, None, None


def flash_attention_packed(mix: torch.Tensor, causal: bool = True, dropout_p: float = 0.0, scale: Optional[float] = None,
                           doc: Optional[DocumentMask] = None) -> Optional[torch.Tensor]:
    """Attention on the ``[b, s, heads, 3, d]`` view of a fused QKV projection output (any batch / sequence strides), or on its grouped form
    ``[b, s, kv_heads, G + 2, d]``.  ``doc`` keeps every query inside its document (causal only).  Returns ``None`` when the native
    kernels do not apply (caller falls back to ``attention`` on the slices)."""
    if mix.dim() != 5 or mix.shape[3] < 3:
        return None
    q, k, v = _split_packed(mix)
    needs_grad = torch.is_grad_enabled() and mix.requires_grad
    if not _native_ok(q, k, v, None, causal, needs_grad, doc):
        return None
    sc = float(scale if scale is not None else q.shape[-1] ** -0.5)
    seed = _dropout_seed(dropout_p, q.shape[0] * _q_heads(q) * q.shape[1] * k.shape[1])
    return _FlashAttnFn.apply(mix, None, None, None, causal, sc, dropout_p, seed, doc)


def attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, causal: bool = True, dropout_p: float = 0.0,
              scale: Optional[float] = None, attn_mask=None) -> torch.Tensor:
    """``attn_mask``: a boolean / additive tensor (SDPA), a ``DocumentMask`` (the native kernels where they apply; ``causal`` is
    implied) or a ``KeyPaddingMask`` (likewise; non-causal is implied)."""
    needs_grad = torch.is_grad_enabled() and (q.requires_grad or k.requires_grad or v.requires_grad)
    doc = attn_mask if isinstance(attn_mask, DocumentMask) else None
    pad = attn_mask if isinstance(attn_mask, KeyPaddingMask) else None
    if doc is not None:
        causal, attn_mask = True, None
    if pad is not None:
        causal, attn_mask = False, None
    if _native_ok(q, k, v, attn_mask, causal, needs_grad, doc, pad):
        sc = float(scale if scale is not None else q.shape[-1] ** -0.5)
        seed = _dropout_seed(dropout_p, q.shape[0] * q.shape[2] * q.shape[1] * k.shape[1])
        return _FlashAttnFn.apply(None, q, k, v, causal, sc, dropout_p, seed, doc if pad is None else pad)
    if doc is not None:
        attn_mask = doc.dense()
    if pad is not None:
        attn_mask = pad.additive().to(q.dtype)
    qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))           # [b, h, s, d]
    if attn_mask is not None:
        causal = False
    gqa = {"enable_gqa": True} if k.shape[2] != q.shape[2] else {}
    out = F.scaled_dot_product_attention(qt, kt, vt, attn_mask=attn_mask, dropout_p=dropout_p, is_causal=causal, scale=scale, **gqa)
    return out.transpose(1, 2)


def core_attention(q: torch.Tensor, k: torch.Tensor, v: torch.Tensor, scale: float, dropout_p: float, training: bool,
                   attn_mask: Optional[torch.Tensor] = None, causal: bool = True, rng_name: Optional[str] = "local_seed"
                   ) -> torch.Tensor:
    """Unfused attention: scores materialised as ``[b, heads, sq, sk]``.  Grouped K/V heads are repeated to the query heads."""
    from . import functional as OF

    if k.shape[2] != q.shape[2]:
        g = q.shape[2] // k.shape[2]
        k, v = k.repeat_interleave(g, dim=2), v.repeat_interleave(g, dim=2)
    if isinstance(attn_mask, (DocumentMask, KeyPaddingMask)):
        attn_mask = attn_mask.additive()
    qt, kt, vt = (t.transpose(1, 2) for t in (q, k, v))
    scores = torch.matmul(qt, kt.transpose(-1, -2))
    if attn_mask is None and causal:
        probs = OF.causal_softmax(scores.contiguous(), scale)
    else:
        scores = scores.float() * scale
        if attn_mask is not None:
            scores = scores + attn_mask.float()
        probs = torch.softmax(scores, -1).to(q.dtype)
    probs = OF.dropout(probs, dropout_p, training, rng_name)
    return torch.matmul(probs, vt).transpose(1, 2)
