"""The user-facing command line, end to end, as subprocesses: train (with checkpoint) -> resume -> generate -> export -> serve ->
latency tool.  Runs on CPU in the default suite and on the H100 with ``-m gpu`` (bf16, native kernels, CUDA-graph decode)."""
import os
import re
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = os.path.join(ROOT, "paddlefleetx_b200", "configs", "nlp", "gpt")
MODEL = ["Model.num_layers=2", "Model.hidden_size=128", "Model.num_attention_heads=2", "Model.ffn_hidden_size=512", "Model.vocab_size=50304",
         "Model.max_position_embeddings=128", "Model.hidden_dropout_prob=0.0", "Model.attention_probs_dropout_prob=0.0"]


def _run(args, device, timeout=600):
    env = dict(os.environ, PYTHONPATH=ROOT)
    if device == "cpu":
        env["CUDA_VISIBLE_DEVICES"] = ""
    p = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=timeout, cwd=ROOT, env=env)
    assert p.returncode == 0, (args, p.stdout[-1500:], p.stderr[-3000:])
    return p.stdout + p.stderr


def _workflow(tmp_path, device):
    out = str(tmp_path / "out")
    dev = ["Global.device=" + device] + (["Engine.mix_precision.enable=False"] if device == "cpu" else [])
    train = MODEL + dev + ["Data.Train.dataset.name=SyntheticGPTDataset", "Data.Eval.dataset.name=SyntheticGPTDataset", "Data.Train.dataset.max_seq_len=64",
                           "Data.Eval.dataset.max_seq_len=64", "Data.Train.loader.num_workers=0", "Data.Eval.loader.num_workers=0",
                           "Global.local_batch_size=4", "Global.micro_batch_size=2", "Engine.logging_freq=1", "Engine.eval_freq=3", "Engine.eval_iters=2",
                           f"Engine.save_load.output_dir={out}"]

    def o(lst):
        return [x for item in lst for x in ("-o", item)]

    log = _run(["tools/train.py", "-c", os.path.join(CFG, "pretrain_gpt_345M_single_card.yaml")] + o(train + ["Engine.max_steps=4", "Engine.save_load.save_steps=4"]), device)
    assert "ips_total:" in log and "[eval]" in log
    ckpt = os.path.join(out, "epoch_0_step_4")
    assert sorted(os.listdir(ckpt)) == ["meta_state.pdopt", "model.pdparams", "model_state.pdopt"]
    log = _run(["tools/train.py", "-c", os.path.join(CFG, "pretrain_gpt_345M_single_card.yaml")] + o(train + ["Engine.max_steps=6", "Engine.save_load.save_steps=-1",
                                                                                                            f"Engine.save_load.ckpt_dir={ckpt}"]), device)
    steps = [int(m) for m in re.findall(r"\[train\].*?batch: \[(\d+)/", log)]
    assert steps and min(steps) >= 4, (steps, log[-1500:])                     # resumed, did not start from scratch
    gen = MODEL + dev + ["Generation.max_dec_len=8", f"Engine.save_load.ckpt_dir={ckpt}", f"Engine.save_load.output_dir={out}"]
    log = _run(["tasks/gpt/generation.py", "-c", os.path.join(CFG, "generation_gpt_345M_single_card.yaml")] + o(gen), device)
    assert "Generation" in log or "generation" in log
    _run(["tools/export.py", "-c", os.path.join(CFG, "generation_gpt_345M_single_card.yaml")] + o(gen), device)
    assert sorted(os.listdir(os.path.join(out, "rank_0"))) == ["model.pdiparams", "model.pdmodel"]
    log = _run(["tasks/gpt/inference.py", "--model_dir", out, "--text", "hello b200"], device)
    assert "Generation:" in log
    conv = str(tmp_path / "conv")
    _run(["tools/reshard.py", "--src", ckpt, "--dst", conv, "--mp", "1"], device)
    assert os.path.isfile(os.path.join(conv, "model.pdparams"))


def test_cli_workflow_cpu(tmp_path):
    _workflow(tmp_path, "cpu")


@pytest.mark.gpu
def test_cli_workflow_gpu(tmp_path):
    _workflow(tmp_path, "gpu")


FAMILIES = {
    "vit": ("vis/vit/ViT_tiny_patch16_224_ci_cifar10_1n8c_dp_fp16o2.yaml",
            ["Data.Train.dataset.name=SyntheticImageDataset", "Data.Train.dataset.image_size=32", "Data.Train.dataset.class_num=10", "Data.Train.loader.num_workers=0",
             "Data.Train.sampler.batch_size=4", "Model.model.img_size=32", "Model.model.patch_size=8", "Model.model.depth=2", "Global.local_batch_size=4",
             "Global.micro_batch_size=4", "Distributed.dp_degree=1", "Engine.num_train_epochs=1", "Engine.run_mode=step"]),
    "moco": ("vis/moco/mocov2_pt_in1k_1n8c.yaml",
             ["Data.Train.dataset.name=SyntheticImageDataset", "Data.Train.dataset.image_size=32", "Data.Train.dataset.two_views=True", "Data.Train.loader.num_workers=0",
              "Data.Train.sampler.batch_size=4", "Global.local_batch_size=4", "Global.micro_batch_size=4", "Distributed.dp_degree=1", "Engine.run_mode=step",
              "Engine.num_train_epochs=1", "Model.model.backbone=resnet18", "Model.model.K=16", "Model.model.dim=8"]),
    "imagen": ("multimodal/imagen/imagen_397M_text2im_64x64.yaml",
               ["Data.Train.dataset.name=SyntheticImagenDataset", "Data.Train.loader.num_workers=0", "Global.local_batch_size=2", "Global.micro_batch_size=2",
                "Distributed.dp_degree=1", "Engine.run_mode=step", "Engine.num_train_epochs=1"]),
    "moe": ("nlp/moe/pretrain_moe_345M_single_card.yaml",
            ["Model.num_layers=2", "Model.hidden_size=64", "Model.num_attention_heads=4", "Model.ffn_hidden_size=128", "Model.max_position_embeddings=32",
             "Data.Train.dataset.name=SyntheticGPTDataset", "Data.Train.dataset.max_seq_len=32", "Data.Train.loader.num_workers=0", "Global.local_batch_size=2",
             "Global.micro_batch_size=2"]),
    "ernie": ("nlp/ernie/pretrain_ernie_base_345M_single_card.yaml",
              ["Model.hidden_size=64", "Model.num_hidden_layers=2", "Model.num_attention_heads=4", "Model.vocab_size=512", "Model.max_position_embeddings=64",
               "Global.local_batch_size=2", "Global.micro_batch_size=2", "Data.Train.loader.num_workers=0", "Data.Train.dataset.name=SyntheticErnieDataset",
               "Data.Train.dataset.max_seq_length=32", "Data.Train.dataset.vocab_size=512"]),
}


def _family(name, device):
    cfg, ov = FAMILIES[name]
    ov = ov + ["Global.device=" + device, "Engine.max_steps=3", "Engine.logging_freq=1", "Engine.eval_freq=-1", "Engine.save_load.save_steps=-1"]
    if device == "cpu":
        ov.append("Engine.mix_precision.enable=False")
    args = ["tools/train.py", "-c", os.path.join(ROOT, "paddlefleetx_b200", "configs", cfg)]
    for item in ov:
        args += ["-o", item]
    log = _run(args, device)
    assert log.count("[train]") >= 3, log[-1500:]
    losses = [float(x) for x in re.findall(r"loss: ([0-9.]+)", log)]
    assert losses and all(l == l and l < 1e4 for l in losses), losses


@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_train_cli_every_model_family_cpu(name):
    _family(name, "cpu")


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(FAMILIES))
def test_train_cli_every_model_family_gpu(name):
    _family(name, "gpu")


TINY_GPT = ["Global.device=cpu", "Engine.mix_precision.enable=False", "Model.num_layers=2", "Model.hidden_size=64", "Model.num_attention_heads=4",
            "Model.ffn_hidden_size=128", "Model.max_position_embeddings=64", "Model.hidden_dropout_prob=0.0", "Model.attention_probs_dropout_prob=0.0"]


def _cli(tool, cfg, ov, device="cpu"):
    args = [tool, "-c", os.path.join(CFG, cfg)]
    for item in ov:
        args += ["-o", item]
    return _run(args, device)


@pytest.mark.parametrize("cfg", ["qat_gpt_345M_single_card.yaml", "prune_gpt_345M_single_card.yaml"])
def test_compression_recipes_train_through_the_cli(cfg):
    log = _cli("tools/train.py", cfg, TINY_GPT + ["Data.Train.dataset.name=SyntheticGPTDataset", "Data.Train.dataset.max_seq_len=32", "Data.Train.loader.num_workers=0",
                                                  "Global.local_batch_size=2", "Global.micro_batch_size=2", "Engine.max_steps=3", "Engine.logging_freq=1",
                                                  "Engine.eval_freq=-1", "Engine.save_load.save_steps=-1"])
    assert log.count("[train]") >= 3


def test_offline_eval_cli_perplexity_and_lambada(tmp_path):
    import json

    wiki = tmp_path / "wiki.txt"
    wiki.write_text(("the quick brown fox jumps over the lazy dog . " * 40 + "\n") * 4)
    log = _cli("tools/eval.py", "eval_gpt_345M_single_card.yaml", TINY_GPT + [f"Offline_Eval.eval_path={wiki}", "Offline_Eval.cloze_eval=False",
                                                                             "Offline_Eval.overlapping_eval=16", "Offline_Eval.batch_size=2", "Offline_Eval.max_seq_len=32"])
    m = re.search(r"ppl: ([0-9.E+-]+) \| adjusted ppl: ([0-9.E+-]+) \| token ratio: ([0-9.]+)", log)
    assert m and float(m.group(1)) > 1.0 and float(m.group(3)) > 1.0, log[-800:]
    lam = tmp_path / "lambada.jsonl"
    lam.write_text("".join(json.dumps({"text": f"the quick brown fox jumps over the lazy dog number {i}"}) + "\n" for i in range(6)))
    log = _cli("tools/eval.py", "eval_gpt_345M_single_card.yaml", TINY_GPT + [f"Offline_Eval.eval_path={lam}", "Offline_Eval.cloze_eval=True", "Offline_Eval.batch_size=2",
                                                                             "Offline_Eval.max_seq_len=32"])
    assert "total examples: 6.0000E+00" in log, log[-800:]


def test_tipc_case_script_runs_and_reports_speed(tmp_path):
    """A benchmarks/test_tipc case script end to end on CPU: case variables -> family harness -> tipc.py -> log + speed json."""
    import json
    import subprocess

    case = os.path.join(ROOT, "benchmarks", "test_tipc", "gpt", "dygraph", "hybrid_parallel", "N1C1", "gpt_bs16_fp32_DP1-MP1-PP1.sh")
    tiny = ("Global.device=cpu Model.num_layers=2 Model.hidden_size=64 Model.num_attention_heads=4 Model.vocab_size=512 Model.max_position_embeddings=32 "
            "Data.Train.dataset.max_seq_len=32 Data.Train.dataset.vocab_size=512 Global.local_batch_size=2 Global.micro_batch_size=2")
    env = dict(os.environ, LOG_DIR=str(tmp_path), max_iter="6", skip_steps="2", TIPC_EXTRA_OPTS=tiny, DATA_DIR="")
    r = subprocess.run(["bash", case], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    with open(tmp_path / "gpt_bs16_fp32_DP1-MP1-PP1_N1C1_speed.json") as f:
        out = json.load(f)
    assert out["return_code"] == 0 and out["ips"] > 0 and out["unit"] == "tokens/s" and out["samples_used"] == 4 and out["final_loss"] > 0
    assert os.path.isfile(out["log"])
    # every case of the matrix resolves to a launchable command
    import glob

    sys.path.insert(0, os.path.join(ROOT, "benchmarks", "test_tipc"))
    cases = [c for c in glob.glob(os.path.join(ROOT, "benchmarks", "test_tipc", "*", "**", "N*C*", "*.sh"), recursive=True) if "/dygraph/" in c or "/static/" in c]
    assert len(cases) >= 60
    for c in cases:
        fam_sh = os.path.join(os.path.dirname(os.path.dirname(c)), "benchmark_common", "run_benchmark.sh")
        family = open(fam_sh).read().split("--family ")[1].split()[0]
        exports = [ln[len("export "):].split() for ln in open(c) if ln.startswith("export ")][0]
        e = dict(os.environ, **dict(kv.split("=", 1) for kv in exports), DATA_DIR="")
        d = subprocess.run([sys.executable, os.path.join(ROOT, "benchmarks", "test_tipc", "tipc.py"), "--family", family, "--dry-run"], env=e, capture_output=True, text=True)
        assert d.returncode == 0 and "-c paddlefleetx_b200/configs/" in d.stdout, (c, d.stderr[-500:])
        cfg = d.stdout.split("-c ")[1].split()[0]
        assert os.path.isfile(os.path.join(ROOT, cfg)), (c, cfg)
