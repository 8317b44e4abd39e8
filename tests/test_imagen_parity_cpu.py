"""Imagen U-Net parity: the four presets (and a sweep of constructor options) must build networks with exactly the parameter
count of the REFERENCE constructors.  The reference sources are executed unmodified for their ``__init__`` only, on top of a few-line
``paddle.nn`` -> ``torch.nn`` shim on the meta device (no Paddle needed, no memory allocated); the original constructors are replayed from tests/golden (see golden_ref.py)."""
import contextlib
import importlib
import os
import sys
import types

import golden_ref
import pytest
import torch
import torch.nn as tnn

REF_DIR = os.path.join(golden_ref.REFERENCE_DIR, "ppfleetx/models/multimodal_model/imagen")


def _install_shim():
    paddle, nn, F, init = (types.ModuleType(n) for n in ("paddle", "paddle.nn", "paddle.nn.functional", "paddle.nn.initializer"))

    class Layer(tnn.Module):
        def create_parameter(self, shape, default_initializer=None, **kw):
            return tnn.Parameter(torch.empty(*[int(s) for s in shape]))

    def nobias(v):
        return v is not False

    nn.Layer = Layer
    nn.Linear = lambda i, o, bias_attr=None, **kw: tnn.Linear(i, o, bias=nobias(bias_attr))
    nn.Conv2D = lambda i, o, k, stride=1, padding=0, groups=1, bias_attr=None, **kw: tnn.Conv2d(i, o, k, stride=stride, padding=padding, groups=groups,
                                                                                                bias=nobias(bias_attr))
    nn.LayerNorm, nn.GroupNorm, nn.Embedding, nn.Sequential, nn.LayerList = tnn.LayerNorm, tnn.GroupNorm, tnn.Embedding, tnn.Sequential, tnn.ModuleList
    nn.Silu, nn.GELU, nn.Sigmoid, nn.Dropout, nn.PixelShuffle = tnn.SiLU, tnn.GELU, tnn.Sigmoid, tnn.Dropout, tnn.PixelShuffle
    nn.Upsample = lambda scale_factor=None, mode="nearest", **kw: tnn.Upsample(scale_factor=scale_factor, mode=mode)
    for name in ("Normal", "Constant", "KaimingUniform"):
        setattr(init, name, lambda *a, **k: (lambda *a2, **k2: None))
    nn.initializer, nn.functional = init, F
    paddle.nn, paddle.einsum, paddle.expm1 = nn, torch.einsum, torch.expm1
    paddle.empty = lambda shape, **kw: torch.empty(*shape)
    fleet_utils = types.ModuleType("paddle.distributed.fleet.utils")
    fleet_utils.recompute = lambda fn, *a, **k: fn(*a, **k)
    mods = {"paddle": paddle, "paddle.nn": nn, "paddle.nn.functional": F, "paddle.nn.initializer": init, "paddle.distributed": types.ModuleType("paddle.distributed"),
            "paddle.distributed.fleet": types.ModuleType("paddle.distributed.fleet"), "paddle.distributed.fleet.utils": fleet_utils}
    t5 = types.ModuleType("ppfleetx.models.language_model.t5.modeling")
    t5.finfo = torch.finfo
    mods["ppfleetx.models.language_model.t5.modeling"] = t5
    pkg = types.ModuleType("_ref_imagen")
    pkg.__path__ = [REF_DIR]
    mods["_ref_imagen"] = pkg
    return mods


@contextlib.contextmanager
def _load_reference():
    import ppfleetx.models.language_model  # noqa: F401  (the alias package must be importable before its t5 leaf is stubbed)

    mods = _install_shim()
    saved = {k: sys.modules.get(k) for k in mods}
    sys.modules.update(mods)
    try:
        unet = importlib.import_module("_ref_imagen.unet")
        modeling_src = open(os.path.join(REF_DIR, "modeling.py")).read()
        # only the four preset classes of modeling.py are needed (the rest of that file imports the text towers)
        start, end = modeling_src.index("class Unet64_397M"), modeling_src.index("# main imagen ddpm class")
        ns = {"Unet": unet.Unet}
        exec(compile(modeling_src[start:end], "ref_presets", "exec"), ns)
        unet.PixelShuffleUpsample.init_conv_ = lambda self, conv: None       # initialisation detail, irrelevant for the structure
        unet.zero_init_ = lambda m: None
        yield unet, ns
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v
        for k in [k for k in sys.modules if k.startswith("_ref_imagen")]:
            sys.modules.pop(k, None)


@pytest.fixture(scope="module")
def ref_unet():
    with golden_ref.namespaces("imagen_parity", _load_reference, count=2) as nss:
        yield tuple(nss)


def _count(m):
    return sum(p.numel() for p in m.parameters())


def _shapes(m):
    return sorted(tuple(p.shape) for p in m.parameters())


@pytest.mark.parametrize("name,kw", [("Unet64_397M", {}), ("BaseUnet64", {}), ("BaseUnet64", {"dim": 360, "text_embed_dim": 1536}),
                                      ("SRUnet256", {"lowres_cond": True}), ("SRUnet1024", {"lowres_cond": True, "dim": 128})])
def test_presets_match_reference_parameter_counts(ref_unet, name, kw):
    from paddlefleetx_b200.models.multimodal_model.imagen import unet as U

    _, ns = ref_unet
    with torch.device("meta"):
        ours, ref = getattr(U, name)(**kw), ns[name](**kw)
    assert _count(ours) == _count(ref), (name, _count(ours), _count(ref))
    assert _shapes(ours) == _shapes(ref)


@pytest.mark.parametrize("kw", [
    dict(dim=32, dim_mults=(1, 2), layer_attns=(False, True), layer_cross_attns=(False, True), attn_heads=2, attn_dim_head=8),
    dict(dim=32, dim_mults=(1, 2, 4), memory_efficient=True, num_resnet_blocks=(1, 2, 2), layer_attns=False, layer_cross_attns=(False, False, True)),
    dict(dim=32, dim_mults=(1, 2), combine_upsample_fmaps=True, init_conv_to_final_conv_residual=True, pixel_shuffle_upsample=False),
    dict(dim=32, dim_mults=(1, 2), use_linear_attn=(True, False), use_linear_cross_attn=(True, False), layer_attns=(False, True), lowres_cond=True,
         self_cond=True, cond_images_channels=3, init_cross_embed=False, attn_pool_text=False, final_resnet_block=False, use_global_context_attn=False),
    dict(dim=32, dim_mults=(1, 2), cond_on_text=False, attend_at_middle=False, cosine_sim_attn=True, layer_attns_depth=2, layer_mid_attns_depth=2,
         resnet_groups=4, channels=4, channels_out=8, max_text_len=64, cond_dim=48, num_time_tokens=3, learned_sinu_pos_emb_dim=8),
])
def test_constructor_options_match_reference(ref_unet, kw):
    from paddlefleetx_b200.models.multimodal_model.imagen import unet as U

    unet, _ = ref_unet
    with torch.device("meta"):
        ours, ref = U.Unet(**kw), unet.Unet(**kw)
    assert _shapes(ours) == _shapes(ref), (_count(ours), _count(ref))


def test_unknown_option_raises():
    from paddlefleetx_b200.models.multimodal_model.imagen import modeling as I
    from paddlefleetx_b200.models.multimodal_model.imagen import unet as U

    with pytest.raises(TypeError):
        U.Unet(dim=32, pixel_shuffle_upsampling=True)
    with pytest.raises(TypeError):
        I.imagen_397M_text2im_64(no_such_option=1)


def test_every_variant_runs_forward_backward():
    from paddlefleetx_b200.models.multimodal_model.imagen import unet as U

    torch.manual_seed(0)
    common = dict(dim=16, text_embed_dim=12, attn_heads=2, attn_dim_head=8, max_text_len=8, attn_pool_num_latents=4, resnet_groups=4)
    variants = [
        dict(dim_mults=(1, 2), layer_attns=(False, True), layer_cross_attns=(False, True)),
        dict(dim_mults=(1, 2), memory_efficient=True, layer_attns=False, layer_cross_attns=(False, True), lowres_cond=True),
        dict(dim_mults=(1, 2), use_linear_attn=(True, False), use_linear_cross_attn=(True, False), layer_attns=(False, True), cross_embed_downsample=True,
             combine_upsample_fmaps=True, init_conv_to_final_conv_residual=True, pixel_shuffle_upsample=False, self_cond=True, use_recompute=True),
    ]
    for kw in variants:
        net = U.Unet(**common, **kw)
        net.train()
        x = torch.randn(2, 3, 16, 16)
        extra = {}
        if kw.get("lowres_cond"):
            extra = dict(lowres_cond_img=torch.randn(2, 3, 16, 16), lowres_noise_times=torch.rand(2))
        y = net(x, torch.rand(2), text_embeds=torch.randn(2, 5, 12), text_mask=torch.ones(2, 5, dtype=torch.bool), cond_drop_prob=0.5, **extra)
        assert y.shape == x.shape
        # the output convolution starts at zero: take a step so that gradients reach everything
        with torch.no_grad():
            net.final_conv.weight.normal_(0, 0.02)
        net(x, torch.rand(2), text_embeds=torch.randn(2, 5, 12), **extra).pow(2).mean().backward()
        missing = [n for n, p in net.named_parameters() if p.grad is None]
        assert not missing, missing[:5]
        g = net.forward_with_cond_scale(x, torch.rand(2), text_embeds=torch.randn(2, 5, 12), cond_scale=3.0, **extra)
        assert torch.isfinite(g).all()
