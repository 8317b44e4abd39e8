"""ERNIE parity: ``ErnieForPretraining(ErnieModel(..))`` and the sequence-classification head built by the REFERENCE constructors
(ernie/dygraph/single_model.py + ernie/layers/transformer.py, executed unmodified on a ``paddle.nn`` -> ``torch.nn`` shim, meta device) and by
ours have the same number of parameters and the same multiset of tensor sizes.  The original constructors are replayed from tests/golden (see golden_ref.py)."""
import contextlib
import importlib
import os
import sys
import types

import golden_ref
import pytest
import torch
import torch.nn as tnn

REF_DIR = os.path.join(golden_ref.REFERENCE_DIR, "ppfleetx/models/language_model/ernie")

CONFIGS = {"base": dict(vocab_size=40000, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072, max_position_embeddings=512, type_vocab_size=4),
           "large": dict(vocab_size=40000, hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096, max_position_embeddings=512, type_vocab_size=4),
           "10B-class": dict(vocab_size=40000, hidden_size=4096, num_hidden_layers=48, num_attention_heads=64, intermediate_size=16384, max_position_embeddings=512, type_vocab_size=4),
           "task-ids": dict(vocab_size=18000, hidden_size=384, num_hidden_layers=3, num_attention_heads=6, intermediate_size=1536, max_position_embeddings=128, type_vocab_size=2,
                            use_task_id=True, task_type_vocab_size=3)}


def _shim():
    names = ["paddle", "paddle.nn", "paddle.nn.functional", "paddle.nn.initializer", "paddle.tensor", "paddle.fluid", "paddle.fluid.layers", "paddle.fluid.data_feeder",
             "paddle.nn.layer", "paddle.nn.layer.transformer", "paddle.distributed", "paddle.distributed.fleet", "paddle.distributed.fleet.utils"]
    m = {n: types.ModuleType(n) for n in names}
    paddle, nn, init = m["paddle"], m["paddle.nn"], m["paddle.nn.initializer"]

    class Layer(tnn.Module):
        def create_parameter(self, shape, default_initializer=None, is_bias=False, **kw):
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
        def __init__(self, n, d, padding_idx=None, weight_attr=None, **kw):
            super().__init__(int(n), int(d))

    class Dropout(tnn.Dropout):
        def __init__(self, p=0.5, mode=None, **kw):
            super().__init__(p)

    nn.Layer, nn.Linear, nn.LayerNorm, nn.Embedding, nn.Dropout = Layer, Linear, LayerNorm, Embedding, Dropout
    nn.LayerList, nn.Sequential, nn.Tanh = tnn.ModuleList, tnn.Sequential, tnn.Tanh
    nn.CrossEntropyLoss = lambda **kw: tnn.CrossEntropyLoss()
    for name in ("Constant", "Normal", "KaimingUniform", "XavierUniform", "Uniform", "TruncatedNormal"):
        setattr(init, name, lambda *a, **k: (lambda *a2, **k2: None))
    F = m["paddle.nn.functional"]
    for act in ("gelu", "relu", "tanh", "softmax", "dropout"):
        setattr(F, act, getattr(torch.nn.functional, act))
    nn.initializer, nn.functional, nn.layer = init, F, m["paddle.nn.layer"]
    m["paddle.nn.layer"].transformer = m["paddle.nn.layer.transformer"]
    m["paddle.nn.layer.transformer"]._convert_param_attr_to_list = lambda attr, n: [attr] * n
    m["paddle.nn.layer.transformer"]._convert_attention_mask = lambda mask, dtype: mask
    m["paddle.nn.layer.transformer"].MultiHeadAttention = type("MultiHeadAttention", (tnn.Module,), {})
    m["paddle.fluid.data_feeder"].convert_dtype = lambda d: d
    m["paddle.fluid"].layers, m["paddle.fluid"].data_feeder = m["paddle.fluid.layers"], m["paddle.fluid.data_feeder"]
    m["paddle.distributed.fleet.utils"].recompute = lambda fn, *a, **k: fn(*a, **k)
    m["paddle.distributed.fleet"].utils = m["paddle.distributed.fleet.utils"]
    m["paddle.distributed"].fleet = m["paddle.distributed.fleet"]
    paddle.nn, paddle.tensor, paddle.distributed, paddle.fluid = nn, m["paddle.tensor"], m["paddle.distributed"], m["paddle.fluid"]
    class ParamAttr:                       # only what layers/transformer.py touches: a name slot and the _to_attr normaliser
        def __init__(self, name=None, **kw):
            self.name = name

        @staticmethod
        def _to_attr(a):
            return a if isinstance(a, ParamAttr) else ParamAttr()

    paddle.ParamAttr = ParamAttr
    paddle.no_grad = torch.no_grad
    paddle.get_default_dtype = lambda: "float32"
    paddle.float32, paddle.float16, paddle.int64, paddle.bool, paddle.Tensor = torch.float32, torch.float16, torch.int64, torch.bool, torch.Tensor
    for pkg, sub in (("_ref_ernie", ""), ("_ref_ernie.dygraph", "dygraph"), ("_ref_ernie.layers", "layers")):
        mod = types.ModuleType(pkg)
        mod.__path__ = [os.path.join(REF_DIR, sub)]
        m[pkg] = mod
    return m


@contextlib.contextmanager
def _load_reference():
    mods = _shim()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        mod = importlib.import_module("_ref_ernie.dygraph.single_model")
        for cls in (mod.ErnieModel, mod.ErnieForPretraining, mod.ErnieForSequenceClassification):
            cls.init_weights = lambda self, layer: None          # initialisation values are not what is compared
        yield mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k.startswith("_ref_ernie")]:
            sys.modules.pop(k, None)


@pytest.fixture(scope="module")
def ref_ernie():
    with golden_ref.namespaces("ernie_parity", _load_reference) as (ns,):
        yield ns


def _sizes(m):
    seen, out = set(), []
    for p in m.parameters():
        if id(p) not in seen:
            seen.add(id(p))
            out.append(p.numel())
    return sorted(out)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_ernie_pretraining_matches_reference_constructor(ref_ernie, name):
    from paddlefleetx_b200.models.language_model.ernie import model as ours

    kw = CONFIGS[name]
    with torch.device("meta"):
        ref = ref_ernie.ErnieForPretraining(ref_ernie.ErnieModel(**kw))
    mine = ours.ErnieForPretraining(ours.ErnieModel(device="meta", **kw))
    assert sum(_sizes(ref)) == sum(_sizes(mine)), (name, sum(_sizes(ref)), sum(_sizes(mine)))
    assert _sizes(ref) == _sizes(mine), name


def test_ernie_sequence_classification_matches_reference_constructor(ref_ernie):
    from paddlefleetx_b200.models.language_model.ernie import model as ours

    kw = CONFIGS["base"]
    with torch.device("meta"):
        ref = ref_ernie.ErnieForSequenceClassification(ref_ernie.ErnieModel(**kw), num_classes=3)
    mine = ours.ErnieForSequenceClassification(ours.ErnieModel(device="meta", **kw), num_classes=3)
    assert _sizes(ref) == _sizes(mine)
