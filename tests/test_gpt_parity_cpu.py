"""GPT parity: ``GPTModel`` / ``GPTForPretraining`` built by the REFERENCE constructor (gpt/dygraph/single_model.py, executed unmodified on a
``paddle.nn`` -> ``torch.nn`` shim, meta device) and by ours must have the same number of parameters and the same multiset of tensor sizes, for
the published model sizes (345M ... 175B) with and without the fused QKV projection.  The original constructors are replayed from tests/golden (see golden_ref.py)."""
import contextlib
import importlib
import os
import sys
import types

import golden_ref
import pytest
import torch
import torch.nn as tnn

REF_DIR = os.path.join(golden_ref.REFERENCE_DIR, "ppfleetx/models/language_model/gpt/dygraph")

SIZES = {"345M": (24, 1024, 16), "1.3B": (24, 2048, 16), "6.7B": (32, 4096, 32), "13B": (40, 5120, 40), "175B": (96, 12288, 96)}


def _shim():
    names = ["paddle", "paddle.nn", "paddle.nn.functional", "paddle.nn.initializer", "paddle.tensor", "paddle.fluid", "paddle.fluid.layers", "paddle.nn.layer",
             "paddle.nn.layer.transformer", "paddle.common_ops_import", "paddle.incubate", "paddle.incubate.nn", "paddle.distributed", "paddle.distributed.fleet",
             "paddle.distributed.fleet.utils", "paddle.nn.functional.flash_attention"]
    m = {n: types.ModuleType(n) for n in names}
    paddle, nn, init = m["paddle"], m["paddle.nn"], m["paddle.nn.initializer"]

    class Layer(tnn.Module):
        def create_parameter(self, shape, default_initializer=None, **kw):
            return tnn.Parameter(torch.empty(*[int(s) for s in shape]))

        def add_parameter(self, name, p):
            self.register_parameter(name, p)

    def has_bias(v):
        return v is not False

    class Linear(tnn.Linear):
        def __init__(self, i, o, weight_attr=None, bias_attr=None, **kw):
            super().__init__(int(i), int(o), bias=has_bias(bias_attr))

    class LayerNorm(tnn.LayerNorm):
        def __init__(self, shape, epsilon=1e-5, **kw):
            super().__init__(shape, eps=epsilon)

    class Embedding(tnn.Embedding):
        def __init__(self, n, d, weight_attr=None, **kw):
            super().__init__(int(n), int(d))

    class Dropout(tnn.Dropout):
        def __init__(self, p=0.5, mode=None, **kw):
            super().__init__(p)

    nn.Layer, nn.Linear, nn.LayerNorm, nn.Embedding, nn.Dropout = Layer, Linear, LayerNorm, Embedding, Dropout
    nn.LayerList, nn.Sequential, nn.CrossEntropyLoss = tnn.ModuleList, tnn.Sequential, (lambda **kw: tnn.CrossEntropyLoss())
    nn.GELU = lambda approximate=False, **kw: tnn.GELU(approximate="tanh" if approximate else "none")
    nn.ReLU, nn.Softmax = tnn.ReLU, (lambda axis=-1, **kw: tnn.Softmax(dim=axis))
    for name in ("Constant", "Normal", "KaimingUniform", "XavierUniform", "Uniform", "TruncatedNormal"):
        setattr(init, name, lambda *a, **k: (lambda *a2, **k2: None))
    nn.initializer, nn.functional, nn.layer = init, m["paddle.nn.functional"], m["paddle.nn.layer"]
    m["paddle.nn.layer"].transformer = m["paddle.nn.layer.transformer"]
    m["paddle.nn.layer.transformer"]._convert_param_attr_to_list = lambda attr, n: [attr] * n
    m["paddle.common_ops_import"].convert_dtype = lambda d: d
    m["paddle.incubate.nn"].FusedLinear = Linear
    m["paddle.incubate"].nn = m["paddle.incubate.nn"]
    m["paddle.fluid"].layers = m["paddle.fluid.layers"]
    m["paddle.distributed.fleet.utils"].recompute = lambda fn, *a, **k: fn(*a, **k)
    m["paddle.distributed.fleet"].utils = m["paddle.distributed.fleet.utils"]
    m["paddle.distributed"].fleet = m["paddle.distributed.fleet"]
    m["paddle.nn.functional.flash_attention"].flash_attention = None
    paddle.nn, paddle.tensor, paddle.incubate, paddle.distributed, paddle.fluid = nn, m["paddle.tensor"], m["paddle.incubate"], m["paddle.distributed"], m["paddle.fluid"]
    paddle.ParamAttr = lambda **kw: None
    paddle.no_grad = torch.no_grad
    paddle.get_default_dtype = lambda: "float32"
    paddle.float32, paddle.float16, paddle.bfloat16, paddle.int64, paddle.bool = torch.float32, torch.float16, torch.bfloat16, torch.int64, torch.bool
    paddle.Tensor = torch.Tensor
    pkg = types.ModuleType("_ref_gpt")
    pkg.__path__ = [REF_DIR]
    m["_ref_gpt"] = pkg
    return m


@contextlib.contextmanager
def _load_reference():
    import ppfleetx.models.language_model.moe  # noqa: F401  (imported by the reference file through the alias package; not constructed here)
    import ppfleetx.models.language_model.moe_exp.layer  # noqa: F401
    import ppfleetx.utils.log  # noqa: F401

    mods = _shim()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        yield importlib.import_module("_ref_gpt.single_model")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k.startswith("_ref_gpt")]:
            sys.modules.pop(k, None)


@pytest.fixture(scope="module")
def ref_gpt():
    with golden_ref.namespaces("gpt_parity", _load_reference) as (ns,):
        yield ns


def _sizes(m):
    return sorted(p.numel() for p in m.parameters())


@pytest.mark.parametrize("fuse_qkv", [True, False])
@pytest.mark.parametrize("size", list(SIZES))
def test_gpt_matches_reference_constructor(ref_gpt, size, fuse_qkv):
    from paddlefleetx_b200.models.language_model.gpt.model import GPTForPretraining, GPTModel

    L, h, a = SIZES[size]
    kw = dict(vocab_size=50304, hidden_size=h, num_layers=L, num_attention_heads=a, ffn_hidden_size=4 * h, max_position_embeddings=1024, fuse_attn_qkv=fuse_qkv)
    with torch.device("meta"):
        ref = ref_gpt.GPTForPretraining(ref_gpt.GPTModel(**kw))
    mine = GPTForPretraining(GPTModel(device="meta", **kw))
    n_ref, n_mine = sum(p.numel() for p in ref.parameters()), sum(p.numel() for p in mine.parameters())
    assert n_ref == n_mine, (size, n_ref, n_mine)
    if fuse_qkv:
        assert _sizes(ref) == _sizes(mine), size
