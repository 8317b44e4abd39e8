"""Model families on a real H100: every zoo member runs forward + backward + optimizer step in bf16 on CUDA through the native
op layer (the CPU suite only exercises the PyTorch expressions), and the serving / parallel-free engine paths work end to end."""
import os

import numpy as np
import pytest
import torch

from helpers import ROOT
from paddlefleetx_b200.utils import config as C

pytestmark = pytest.mark.gpu
CFG = os.path.join(ROOT, "paddlefleetx_b200", "configs")
SMALL_GPT = ["Model.num_layers=2", "Model.hidden_size=256", "Model.num_attention_heads=4", "Model.ffn_hidden_size=1024", "Model.vocab_size=1024",
             "Model.max_position_embeddings=128", "Data.Train.dataset.max_seq_len=128", "Data.Eval.dataset.max_seq_len=128",
             "Global.local_batch_size=4", "Global.micro_batch_size=2", "Engine.logging_freq=1", "Data.Train.dataset.name=SyntheticGPTDataset",
             "Data.Eval.dataset.name=SyntheticGPTDataset", "Data.Train.loader.num_workers=0", "Data.Eval.loader.num_workers=0",
             "Optimizer.lr.max_lr=2e-3", "Optimizer.lr.min_lr=2e-4", "Optimizer.lr.warmup_rate=0.0", "Model.hidden_dropout_prob=0.0",
             "Model.attention_probs_dropout_prob=0.0"]


def _engine(cfg):
    from paddlefleetx_b200.core import EagerEngine
    from paddlefleetx_b200.distributed.apis import env
    from paddlefleetx_b200.models import build_module

    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    return EagerEngine(configs=cfg, module=build_module(cfg))


def _gpt_batches(cfg, n):
    g = torch.Generator().manual_seed(0)
    b, s, v = cfg.Global.global_batch_size, cfg.Data.Train.dataset.max_seq_len, cfg.Model.vocab_size
    out = []
    for _ in range(n):
        t = torch.randint(0, v, (b, s + 1), generator=g)
        out.append([t[:, :-1].contiguous(), torch.arange(s).unsqueeze(0).expand(b, s).contiguous(), t[:, 1:].contiguous(), torch.ones(b, s)])
    return out


@pytest.mark.parametrize("extra", [[], ["Model.use_recompute=True", "Model.recompute_granularity=full"],
                                   ["Model.use_recompute=True", "Model.recompute_granularity=core_attn"], ["Model.use_rope=True"],
                                   ["Engine.mix_precision.use_main_grad=True"],
                                   ["Fused.fp8_tp_gemm=True"],                                   # MX block-scaled fp8 forward GEMMs (kind::mxf8f6f4.block_scale)
                                   ["Fused.fp8_tp_gemm=True", "Fused.fp8_recipe=rowwise"]])
def test_gpt_trains_on_gpu_with_native_kernels(extra):
    from paddlefleetx_b200.ops import functional as OF

    cfg = C.get_config(os.path.join(CFG, "nlp/gpt/pretrain_gpt_345M_single_card.yaml"), SMALL_GPT + extra, nranks=1)
    eng = _engine(cfg)
    assert next(eng._module.model.parameters()).dtype == torch.bfloat16 and eng.optimizer.direct_grad
    OF.reset_launch_count()
    batch = _gpt_batches(cfg, 1)[0]
    losses = [float(eng.train_step(batch)) for _ in range(12)]          # same batch: the loss must go down
    assert OF.native_launch_count() > 100, "native kernels were not used"
    assert np.isfinite(losses).all() and losses[-1] < losses[0] - 0.3, losses
    from paddlefleetx_b200.parallel import tp_layers as _tp
    _tp.configure({})                              # process-wide options: leave the defaults for the next test


@pytest.mark.parametrize("fused", [False, True])
def test_moe_gpt_trains_on_gpu(fused):
    """fused=True: device-side routing + dispatch kernel + grouped expert GEMMs from the device-side segment table + combine kernel — the
    sync-free MoE layer, here with an expert group of one rank (the multi-rank exchange is covered by tools/gpu_multi_selftest.py)."""
    cfg = C.get_config(os.path.join(CFG, "nlp/moe/pretrain_moe_345M_single_card.yaml"), SMALL_GPT + [f"Model.moe_configs.fused_p2p={fused}"], nranks=1)
    eng = _engine(cfg)
    if fused:
        from paddlefleetx_b200.models.language_model.moe.moe_layer import MoELayer

        layers = [m for m in eng._module.model.modules() if isinstance(m, MoELayer)]
        assert layers and all(m.grouped is not None for m in layers), "the grouped expert path was not built"
    batch = _gpt_batches(cfg, 1)[0]
    losses = [float(eng.train_step(batch)) for _ in range(6)]
    assert np.isfinite(losses).all() and losses[-1] < losses[0], losses


def test_moe_layer_sync_free_path_matches_the_expert_loop_on_one_gpu():
    from paddlefleetx_b200.models.language_model.moe.moe_layer import ExpertLayer, MoELayer

    def make(fused):
        torch.manual_seed(3)
        ex = [ExpertLayer(256, 1024, dtype=torch.bfloat16, device="cuda") for _ in range(4)]
        return MoELayer(256, ex, gate={"type": "naive", "top_k": 2}, dtype=torch.bfloat16, device="cuda", fused_p2p=fused)

    ref, fus = make(False), make(True)
    fus.load_state_dict(ref.state_dict())
    torch.manual_seed(5)
    x = (torch.randn(1000, 256, device="cuda") * 0.5).bfloat16()
    go = (torch.randn(1000, 256, device="cuda") * 0.1).bfloat16()
    outs = []
    for layer in (ref, fus):
        xi = x.clone().requires_grad_(True)
        y = layer(xi)
        y.backward(go)
        sd_grads = {n: p.grad.float() for n, p in layer.named_parameters() if p.grad is not None}
        outs.append((y.detach().float(), xi.grad.float(), sd_grads))
    rel = lambda a, b: float((a - b).norm() / (b.norm() + 1e-12))
    assert rel(outs[1][0], outs[0][0]) < 2e-2 and rel(outs[1][1], outs[0][1]) < 2e-2
    w1 = torch.stack([outs[0][2][f"experts.{e}.htoh4.weight"] for e in range(4)])
    assert rel(outs[1][2]["grouped.w1"], w1) < 2e-2
    b2 = torch.stack([outs[0][2][f"experts.{e}.h4toh.bias"] for e in range(4)])
    assert rel(outs[1][2]["grouped.b2"], b2) < 2e-2


def test_generation_cuda_graph_matches_eager_on_gpu():
    from paddlefleetx_b200.models.language_model.gpt import model as gpt
    from paddlefleetx_b200.models.language_model.gpt.generation import GPTForGeneration

    torch.manual_seed(0)
    core = gpt.GPTModel(vocab_size=1024, hidden_size=256, num_layers=2, num_attention_heads=4, ffn_hidden_size=1024, max_position_embeddings=128,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, dtype=torch.bfloat16, device="cuda")
    cfg = dict(max_dec_len=10, decode_strategy="greedy_search", eos_token_id=1023, pad_token_id=0)
    eager = GPTForGeneration(core, dict(cfg, use_cuda_graph=False))
    graph = GPTForGeneration(core, dict(cfg, use_cuda_graph=True))
    for bs in (1, 3, 12):
        ids = torch.randint(1, 1000, (bs, 9), device="cuda")
        a, _ = eager.generate(ids)
        b, _ = graph.generate(ids)
        c, _ = graph.generate(ids)              # replay of the captured graph
        assert torch.equal(b, c)
        assert (a == b).float().mean() > 0.9, (a, b)       # bf16 ties may flip an argmax; sequences must essentially agree
    sam = GPTForGeneration(core, dict(cfg, decode_strategy="sampling", top_p=0.8, use_cuda_graph=True))
    x, _ = sam.generate(ids, seed=3)
    y, _ = sam.generate(ids, seed=3)
    assert torch.equal(x, y)


def test_int8_serving_conversion_on_gpu():
    from paddlefleetx_b200.models.language_model.gpt import model as gpt
    from paddlefleetx_b200.ops.quant import quantize_tp_linears_int8

    def build():
        torch.manual_seed(0)
        return gpt.GPTModel(vocab_size=1024, hidden_size=256, num_layers=2, num_attention_heads=4, ffn_hidden_size=1024, max_position_embeddings=128,
                            hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0, dtype=torch.bfloat16, device="cuda")

    ref, q = build(), build()
    assert quantize_tp_linears_int8(q) == 8
    ids = torch.arange(1, 41, device="cuda").view(1, 40)
    with torch.no_grad():
        for n in (1, 3, 40):                    # W8A8 GEMV (<= 8 rows) and the wgmma int8 GEMM
            a, b = ref(ids[:, :n]).float(), q(ids[:, :n]).float()
            assert float((a - b).norm() / a.norm()) < 0.05, n


def test_vision_multimodal_and_text_towers_on_gpu():
    from paddlefleetx_b200.models.multimodal_model.debertav2.modeling import DebertaV2Model
    from paddlefleetx_b200.models.multimodal_model.imagen import modeling as I
    from paddlefleetx_b200.models.multimodal_model.imagen import unet as U
    from paddlefleetx_b200.models.multimodal_model.t5.modeling import T5EncoderModel
    from paddlefleetx_b200.models.protein_folding import EmbeddingsAndEvoformer
    from paddlefleetx_b200.models.vision_model.factory import build
    from paddlefleetx_b200.models.vision_model.moco import MoCo
    from paddlefleetx_b200.optims import FusedAdamW

    dev = "cuda"
    amp = lambda: torch.autocast("cuda", dtype=torch.bfloat16)     # forward only: autocast caches weight casts while a context is open
    vit = build(dict(name="ViT_tiny_patch16_224", img_size=64, patch_size=8, depth=2, class_num=10)).to(dev)
    opt = FusedAdamW(1e-3, named_parameters=list(vit.named_parameters()))
    x, y = torch.randn(8, 3, 64, 64, device=dev), torch.randint(0, 10, (8,), device=dev)
    crit = build(dict(name="CELoss", epsilon=0.1))
    losses = []
    for _ in range(5):
        with amp():
            loss = crit(vit(x), y)
        loss.backward()
        opt.step(); opt.clear_grad()
        losses.append(float(loss))
    assert losses[-1] < losses[0], losses
    moco = MoCo(dim=8, K=16, backbone="resnet18").to(dev)
    with amp():
        lg, _ = moco(torch.randn(4, 3, 32, 32, device=dev), torch.randn(4, 3, 32, 32, device=dev))
    lg.float().logsumexp(1).mean().backward()
    u = U.Unet(dim=16, text_embed_dim=12, dim_mults=(1, 2), layer_attns=(False, True), layer_cross_attns=(False, True), attn_heads=2,
               attn_dim_head=8, max_text_len=6, attn_pool_num_latents=2).to(dev)
    m = I.ImagenModel([u], image_sizes=[16], text_embed_dim=12, timesteps=2).to(dev)
    with amp():
        out = m(torch.rand(2, 3, 16, 16, device=dev), text_embeds=torch.randn(2, 4, 12, device=dev), text_masks=torch.ones(2, 4, device=dev))
        il = I.ImagenCriterion()(*out)
    il.backward()
    ids = torch.randint(0, 100, (2, 16), device=dev)
    mask = torch.ones(2, 16, dtype=torch.long, device=dev)
    t5 = T5EncoderModel(vocab_size=100, d_model=64, d_kv=16, d_ff=128, num_layers=2, num_heads=4, feed_forward_proj="gated-gelu").to(dev)
    with amp():
        o = t5(ids, mask).last_hidden_state
    o.float().sum().backward()
    deb = DebertaV2Model(vocab_size=100, hidden_size=64, num_hidden_layers=2, num_attention_heads=4, intermediate_size=128, position_buckets=8,
                         conv_kernel_size=3).to(dev)
    with amp():
        o = deb(ids, mask).last_hidden_state
    o.float().sum().backward()
    evo = EmbeddingsAndEvoformer(msa_feat_dim=9, target_feat_dim=6, c_m=16, c_z=8, c_s=12, num_blocks=2, max_relative_feature=4, msa_heads=2,
                                 pair_heads=2, extra_msa_channel=8, extra_msa_blocks=1,
                                 template=dict(enabled=True, c_t=8, num_block=1, num_head=2, attn_key_dim=8, embed_torsion_angles=True,
                                               use_template_unit_vector=True)).to(dev)
    R, T = 10, 2
    fold = dict(target_feat=torch.randn(1, R, 6, device=dev), msa_feat=torch.randn(1, 4, R, 9, device=dev), residue_index=torch.arange(R, device=dev)[None],
                aatype=torch.randint(0, 20, (1, R), device=dev), extra_msa=torch.randint(0, 23, (1, 6, R), device=dev),
                extra_has_deletion=torch.rand(1, 6, R, device=dev), extra_deletion_value=torch.rand(1, 6, R, device=dev),
                template_mask=torch.ones(1, T, device=dev), template_aatype=torch.randint(0, 20, (1, T, R), device=dev),
                template_pseudo_beta=torch.randn(1, T, R, 3, device=dev) * 5, template_pseudo_beta_mask=torch.ones(1, T, R, device=dev),
                template_all_atom_positions=torch.randn(1, T, R, 37, 3, device=dev) * 3, template_all_atom_masks=torch.ones(1, T, R, 37, device=dev))
    with amp():
        o = evo(fold, dict(prev_pos=torch.randn(1, R, 37, 3, device=dev)))
    assert o["msa"].shape == (1, 4, R, 16) and torch.isfinite(o["pair"].float()).all()
    (o["single"].float().sum() + o["pair"].float().sum()).backward()
    torch.cuda.synchronize()


def test_ernie_trains_on_gpu(tmp_path):
    rng = np.random.RandomState(0)
    sents = rng.randint(2, 6, size=40)
    lens = rng.randint(8, 24, size=int(sents.sum())).astype(np.int32)
    np.save(tmp_path / "c_ids.npy", rng.randint(4, 500, size=int(lens.sum())).astype(np.int32))
    np.savez(tmp_path / "c_idx.npz", lens=lens, docs=np.concatenate([[0], np.cumsum(sents)]))
    cfg = C.get_config(os.path.join(CFG, "nlp/ernie/pretrain_ernie_base.yaml"),
                       ["Model.hidden_size=128", "Model.num_hidden_layers=2", "Model.num_attention_heads=4", "Model.vocab_size=512",
                        "Model.max_position_embeddings=128", f"Data.Train.dataset.input_dir={tmp_path}", f"Data.Eval.dataset.input_dir={tmp_path}",
                        "Data.Train.dataset.max_seq_length=64", "Data.Train.dataset.vocab_size=500", "Global.local_batch_size=4",
                        "Global.micro_batch_size=4", "Engine.max_steps=4", "Data.Train.loader.num_workers=0", "Optimizer.lr.max_lr=1e-3"], nranks=1)
    from paddlefleetx_b200.data import build_dataloader

    eng = _engine(cfg)
    losses = [float(eng.train_step(b)) for _, b in zip(range(4), build_dataloader(cfg.Data, "Train"))]
    assert len(losses) >= 2 and np.isfinite(losses).all()


def test_native_flash_attention_serves_inference_and_training():
    """attention() routes unmasked bf16 calls (head dim 64 / 128) to the wgmma flash kernels: forward without grad, forward + backward with
    grad (no library kernel), a masked call falls back to SDPA; all three match fp32."""
    import torch.nn.functional as F

    from paddlefleetx_b200.ops import attention as A
    from paddlefleetx_b200.ops import functional as OF

    torch.manual_seed(0)
    q, k, v = (torch.randn(2, 200, 8, 64, device="cuda").bfloat16() for _ in range(3))
    OF.reset_launch_count()
    with torch.no_grad():
        y = A.attention(q, k, v, causal=True)
    assert OF.native_launch_count() == 1
    ref = F.scaled_dot_product_attention(q.transpose(1, 2).float(), k.transpose(1, 2).float(), v.transpose(1, 2).float(), is_causal=True).transpose(1, 2)
    assert float((y.float() - ref).norm() / ref.norm()) < 1e-2
    # training path: native forward and backward (64-wide heads included since round 2)
    OF.reset_launch_count()
    qg, kg, vg = (t.clone().requires_grad_(True) for t in (q, k, v))
    y2 = A.attention(qg, kg, vg, causal=True)
    assert OF.native_launch_count() >= 1 and y2.requires_grad
    go = torch.randn_like(y2)
    y2.backward(go)
    qf, kf, vf = (t.detach().float().requires_grad_(True) for t in (q, k, v))
    rf = F.scaled_dot_product_attention(qf.transpose(1, 2), kf.transpose(1, 2), vf.transpose(1, 2), is_causal=True).transpose(1, 2)
    rf.backward(go.float())
    for got, want in ((qg.grad, qf.grad), (kg.grad, kf.grad), (vg.grad, vf.grad)):
        assert float((got.float() - want).norm() / want.norm()) < 2e-2
    # an explicit mask is library territory
    OF.reset_launch_count()
    mask = torch.zeros(2, 1, 200, 200, device="cuda", dtype=torch.bfloat16)
    y3 = A.attention(q, k, v, attn_mask=mask, causal=False)
    assert OF.native_launch_count() == 0 and y3.shape == y.shape


def test_evoformer_block_runs_on_the_native_attention_kernels(monkeypatch):
    """One Evoformer iteration at the production head geometry (c_m 256 / 8 heads, c_z 128 / 4 heads: 32-wide heads) in bf16: every gated
    attention (MSA row with pair bias, MSA column, triangle start / end) goes through csrc/evoformer_attn_sm90.cu forward AND backward, and
    agrees with the plain PyTorch expression."""
    from paddlefleetx_b200.models.protein_folding.evoformer import EvoformerIteration
    from paddlefleetx_b200.ops import evoformer_attention as EA

    torch.manual_seed(0)
    dev = "cuda"
    blk = EvoformerIteration(c_m=256, c_z=128, msa_heads=8, pair_heads=4, dropout_msa=0.0, dropout_pair=0.0).to(dev)      # fp32 parameters + bf16 autocast, as the folding recipes run it
    with torch.no_grad():                           # the reference zero-initialises the output projections: give the attention a voice
        for n, p in blk.named_parameters():
            if n.endswith("o.weight") or n.endswith("g.weight"):
                p.normal_(0, 0.02)
    S, R = 6, 96
    msa = torch.randn(1, S, R, 256, device=dev) * 0.5
    pair = torch.randn(1, R, R, 128, device=dev) * 0.5
    msa_mask = (torch.rand(1, S, R, device=dev) > 0.1).float()
    pair_mask = (torch.rand(1, R, R, device=dev) > 0.1).float()
    calls = {"native": 0}
    real_apply = EA._EvoAttnFn.apply

    def counting_apply(*a):
        calls["native"] += 1
        return real_apply(*a)

    monkeypatch.setattr(EA._EvoAttnFn, "apply", staticmethod(counting_apply))

    def run():
        m, z = msa.clone().requires_grad_(True), pair.clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            mo, zo = blk(m, z, msa_mask, pair_mask)
        (mo.float().square().mean() + zo.float().square().mean()).backward()
        return mo.detach().float(), zo.detach().float(), m.grad.float(), z.grad.float()

    got = run()
    assert calls["native"] >= 4, calls                # row, column, triangle start, triangle end
    monkeypatch.setattr(EA, "supported", lambda q, k: False)
    blk.zero_grad(set_to_none=True)
    want = run()
    rel = lambda a, b: float((a - b).norm() / (b.norm() + 1e-12))
    errs = [rel(a, b) for a, b in zip(got, want)]
    assert all(torch.isfinite(t).all() for t in got) and max(errs) < 5e-2, errs
