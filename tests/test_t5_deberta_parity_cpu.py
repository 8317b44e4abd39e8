"""Text-tower parity (Imagen's encoders): ``T5EncoderModel`` built by the REFERENCE constructor (language_model/t5/modeling.py, executed
unmodified on a ``paddle.nn`` -> ``torch.nn`` shim, meta device) and by ours must have the same parameter count and the same multiset of tensor
sizes, for t5-11b and smaller shapes.  The original constructors are replayed from tests/golden (see golden_ref.py)."""
import contextlib
import importlib
import os
import sys
import types

import golden_ref
import pytest
import torch
import torch.nn as tnn

REF = os.path.join(golden_ref.REFERENCE_DIR, "ppfleetx/models/language_model")


def _shim():
    names = ["paddle", "paddle.nn", "paddle.nn.functional", "paddle.nn.initializer"]
    m = {n: types.ModuleType(n) for n in names}
    paddle, nn, init = m["paddle"], m["paddle.nn"], m["paddle.nn.initializer"]

    class Layer(tnn.Module):
        def create_parameter(self, shape, default_initializer=None, is_bias=False, **kw):
            return tnn.Parameter(torch.empty(*[int(s) for s in shape]))

        def add_parameter(self, name, p):
            self.register_parameter(name, p)

    class Linear(tnn.Linear):
        def __init__(self, i, o, weight_attr=None, bias_attr=None, **kw):
            super().__init__(int(i), int(o), bias=bias_attr is not False)

    class Embedding(tnn.Embedding):
        def __init__(self, n, d, padding_idx=None, weight_attr=None, **kw):
            super().__init__(int(n), int(d))

    class Dropout(tnn.Dropout):
        def __init__(self, p=0.5, **kw):
            super().__init__(p)

    class LayerNorm(tnn.LayerNorm):
        def __init__(self, shape, epsilon=1e-5, **kw):
            super().__init__(shape, eps=epsilon)

    nn.Layer, nn.Linear, nn.Embedding, nn.Dropout, nn.LayerNorm = Layer, Linear, Embedding, Dropout, LayerNorm
    nn.LayerList, nn.Tanh, nn.Sigmoid, nn.ReLU, nn.Sequential = tnn.ModuleList, tnn.Tanh, tnn.Sigmoid, tnn.ReLU, tnn.Sequential
    for name in ("Constant", "Normal", "Uniform", "TruncatedNormal", "XavierUniform"):
        setattr(init, name, lambda *a, **k: (lambda *a2, **k2: None))
    nn.initializer, nn.functional = init, m["paddle.nn.functional"]
    for fname in ("relu", "gelu", "sigmoid", "silu", "mish", "tanh", "softmax", "dropout"):
        setattr(m["paddle.nn.functional"], fname, getattr(torch.nn.functional, fname))
    paddle.nn = nn
    paddle.Tensor, paddle.no_grad = torch.Tensor, torch.no_grad
    paddle.int64, paddle.int32, paddle.float32, paddle.float16, paddle.bfloat16, paddle.bool = torch.int64, torch.int32, torch.float32, torch.float16, torch.bfloat16, torch.bool
    paddle.ones = lambda shape, dtype=None: torch.ones(*shape)
    pkg, sub = types.ModuleType("_ref_lm"), types.ModuleType("_ref_lm.t5")
    pkg.__path__, sub.__path__ = [REF], [os.path.join(REF, "t5")]
    m["_ref_lm"], m["_ref_lm.t5"] = pkg, sub
    return m


@contextlib.contextmanager
def _load_reference():
    import ppfleetx.data.tokenizers.t5_tokenizer  # noqa: F401  (imported by the reference module through the alias package)
    import ppfleetx.models.multimodal_model.imagen.utils  # noqa: F401

    mods = _shim()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        yield importlib.import_module("_ref_lm.t5.modeling")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k.startswith("_ref_lm")]:
            sys.modules.pop(k, None)


@pytest.fixture(scope="module")
def ref_t5():
    with golden_ref.namespaces("t5_parity", _load_reference, names=True) as (ns,):
        yield ns


def _sizes(m):
    seen, out = set(), []
    for p in m.parameters():
        if id(p) not in seen:
            seen.add(id(p))
            out.append(p.numel())
    return sorted(out)


@pytest.mark.parametrize("kw", [dict(vocab_size=32128, d_model=1024, d_kv=128, d_ff=65536, num_layers=24, num_heads=128, feed_forward_proj="relu"),      # t5-11b
                                dict(vocab_size=32128, d_model=512, d_kv=64, d_ff=2048, num_layers=6, num_heads=8, feed_forward_proj="relu"),             # t5-small
                                dict(vocab_size=1000, d_model=96, d_kv=16, d_ff=256, num_layers=3, num_heads=4, relative_attention_num_buckets=16, feed_forward_proj="relu")])
def test_t5_encoder_matches_reference_constructor(ref_t5, kw):
    from paddlefleetx_b200.models.multimodal_model.t5.modeling import T5EncoderModel

    with torch.device("meta"):
        ref = ref_t5.T5EncoderModel(num_decoder_layers=None, dropout_rate=0.0, **kw)
    mine = T5EncoderModel(device="meta", dropout_rate=0.0, **kw)
    assert sum(_sizes(ref)) == sum(_sizes(mine)), (sum(_sizes(ref)), sum(_sizes(mine)))
    assert _sizes(ref) == _sizes(mine)
    # same parameter names -> a converted reference checkpoint loads by key (the reference lists the embedding a second time under the encoder)
    ref_names = {n for n, _ in ref.named_parameters(remove_duplicate=False)} - {"encoder.embed_tokens.weight"}
    assert ref_names == {n for n, _ in mine.named_parameters()}
