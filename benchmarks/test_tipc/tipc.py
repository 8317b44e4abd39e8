"""Shared driver of the ``benchmarks/test_tipc`` matrix (the reference keeps one ~200-line bash harness per model family under
``benchmarks/test_tipc/<model>/<mode>/benchmark_common/run_benchmark.sh``; here every family's ``run_benchmark.sh`` calls this file).

A case script exports a handful of variables (``model_item fp_item dp_degree mp_degree pp_degree micro_bs bs_item run_mode device_num`` and
family-specific extras) and calls its family's ``run_benchmark.sh``.  This driver

1. turns them into a ``tools/train.py`` / ``tools/auto.py`` command line (recipe + ``-o`` overrides) launched with ``torch.distributed.run`` for
   the GPUs of this node (``NNODES`` / ``NODE_RANK`` / ``MASTER_ADDR`` for multi-node cases such as N4C32),
2. runs it for ``max_iter`` steps under a timeout, logging to ``<LOG_DIR>/<model_name>_<device_num>_log``,
3. parses the ``ips:`` (and ``loss:`` / metric) columns of the ``[train]`` / ``[eval]`` lines, skips the first ``skip_steps`` samples, and writes
   ``<LOG_DIR>/<model_name>_<device_num>_speed.json``.

Synthetic data of the recipe's shape is used unless ``DATA_DIR`` points at a prepared corpus.  ``fp_item=fp16`` means "16-bit mixed precision",
which on H100 is bf16 O2; ``fp32`` turns mixed precision off.  ``--dry-run`` prints the command without running it.
"""
import argparse
import json
import os
import re
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), "..", ".."))
CFG = "paddlefleetx_b200/configs"


def env(name, default=None, cast=str):
    v = os.environ.get(name)
    return default if v in (None, "") else cast(v)


def flag(name, default=False):
    return str(env(name, default)).lower() in ("1", "true", "yes")


def common(world, dp, sharding):
    bs, micro = env("bs_item", 16, int), env("micro_bs", None, int)
    local = max(bs // max(dp * sharding // env("cp_degree", 1, int), 1), 1)      # a context-parallel group consumes one batch
    amp = env("fp_item", "fp16") != "fp32"
    return local, micro or local, [
        "Global.seed=1234", f"Global.local_batch_size={local}", f"Global.micro_batch_size={micro or local}", "Global.global_batch_size=None",
        f"Engine.max_steps={env('max_iter', 50, int)}", f"Engine.eval_freq={env('eval_freq', -1, int)}", "Engine.logging_freq=1",
        f"Engine.mix_precision.enable={amp}", "Engine.save_load.save_steps=-1"]


def degrees():
    dp, mp, pp = env("dp_degree", 1, int), env("mp_degree", 1, int), env("pp_degree", 1, int)
    sh = env("sharding_degree", 1, int)
    return dp, mp, pp, sh, [f"Distributed.dp_degree={dp}", f"Distributed.mp_degree={mp}", f"Distributed.pp_degree={pp}",
                            f"Distributed.sharding.sharding_degree={sh}", f"Distributed.sharding.sharding_stage={env('sharding_stage', 1, int)}",
                            f"Distributed.sharding.sharding_offload={flag('sharding_offload')}",
                            f"Distributed.cp_degree={env('cp_degree', 1, int)}", f"Distributed.cp_mode={env('cp_mode', 'ulysses')}"]


def family_gpt(kind):
    dp, mp, pp, sh, dist = degrees()
    _, _, opts = common(dp * mp * pp * sh, dp, sh)
    big = mp >= 8 or pp >= 8 or flag("full_size")                # the 8-way cases need 16 heads / enough layers to split
    seq = env("seq_len", 1024, int)
    opts += dist + ["Model.hidden_size=1024", f"Model.num_layers={24 if big else 4}", f"Model.num_attention_heads={16 if big else 4}",
                    "Model.type_vocab_size=1", f"Model.use_recompute={flag('use_recompute')}", f"Model.sequence_parallel={flag('sequence_parallel')}",
                    f"Model.use_flash_attn={flag('use_flash_attn', True)}", f"Model.max_position_embeddings={seq}",
                    f"Data.Train.dataset.max_seq_len={seq}", "Optimizer.lr.max_lr=1e-4", "Optimizer.lr.min_lr=1e-5"]
    if env("DATA_DIR"):
        opts += [f"Data.Train.dataset.input_dir={env('DATA_DIR')}"]
    else:
        opts += ["Data.Train.dataset.name=SyntheticGPTDataset", "Data.Train.loader.num_workers=0"]
    if kind == "auto":
        return "tools/auto.py", f"{CFG}/nlp/gpt/auto/pretrain_gpt_345M_single_card.yaml", opts, dp * mp * pp * sh, "tokens/s"
    return "tools/train.py", f"{CFG}/nlp/gpt/pretrain_gpt_1.3B_dp8.yaml", opts, dp * mp * pp * sh, "tokens/s"


GLUE = {"CoLA": ("cola_public", 2, "Mcc", "mcc"), "SST2": ("SST-2", 2, "Accuracy", "acc"), "MRPC": ("MRPC", 2, "AccuracyAndF1", "acc"),
        "QNLI": ("QNLI", 2, "Accuracy", "acc"), "RTE": ("RTE", 2, "Accuracy", "acc"), "WNLI": ("WNLI", 2, "Accuracy", "acc"),
        "STSB": ("STS-B", 1, "PearsonAndSpearman", "pearson"), "QQP": ("QQP", 2, "AccuracyAndF1", "acc"), "MNLI": ("multinli_1.0", 3, "Accuracy", "acc")}


def family_gpt_finetune():
    task = env("task", "CoLA")
    root, classes, metric, _ = GLUE[task]
    data = os.path.join(env("DATA_DIR", "./dataset"), root)
    bs = env("bs_item", 32, int)
    opts = ["Global.seed=1234", f"Global.local_batch_size={bs}", f"Global.micro_batch_size={bs}", "Global.global_batch_size=None", "Engine.logging_freq=10",
            f"Engine.num_train_epochs={env('epochs', 5 if task in ('MRPC', 'WNLI') else 3, int)}", f"Engine.mix_precision.enable={env('fp_item', 'fp16') != 'fp32'}",
            f"Data.Train.dataset.name={task}", f"Data.Train.dataset.root={data}", f"Data.Eval.dataset.name={task}", f"Data.Eval.dataset.root={data}",
            f"Data.Eval.dataset.split={env('split', 'test' if task == 'MRPC' else 'dev')}", f"Model.num_classes={classes}",
            f"Model.metric.train.name={metric}", f"Model.metric.eval.name={metric}"]
    if task == "STSB":
        opts += ["Model.loss.train.name=MSELoss", "Model.loss.eval.name=MSELoss"]
    if env("PRETRAINED"):
        opts += [f"Model.pretrained={env('PRETRAINED')}"]
    return "tools/train.py", f"{CFG}/nlp/gpt/finetune_gpt_345M_single_card_glue.yaml", opts, 1, "sequences/s"


def family_ernie():
    dp, mp, pp, sh, dist = degrees()
    _, _, opts = common(dp * mp * pp * sh, dp, sh)
    opts += dist + [f"Model.use_recompute={flag('use_recompute')}"]
    if env("DATA_DIR"):
        opts += [f"Data.Train.dataset.input_dir={env('DATA_DIR')}"]
    else:
        opts += ["Data.Train.dataset.name=SyntheticErnieDataset", "Data.Train.loader.num_workers=0"]
    return "tools/train.py", f"{CFG}/nlp/ernie/pretrain_ernie_base.yaml", opts, dp * mp * pp * sh, "sequences/s"


IMAGEN = {"imagen_397M_text2im_64": "imagen_397M_text2im_64x64.yaml", "imagen_2B_text2im_64": "imagen_text2im_64x64_T5-11B.yaml",
          "imagen_text2im_64_debertav2": "imagen_text2im_64x64_DebertaV2.yaml", "imagen_SR256": "imagen_super_resolution_256.yaml",
          "imagen_SR1024": "imagen_super_resolution_1024.yaml"}


def family_imagen():
    dp, mp, pp, sh, dist = degrees()
    _, _, opts = common(dp * sh, dp, sh)
    opts += dist
    if not env("DATA_DIR"):
        opts += ["Data.Train.dataset.name=SyntheticImagenDataset", "Data.Train.loader.num_workers=0"]
    else:
        opts += [f"Data.Train.dataset.input_path={env('DATA_DIR')}/filelist.txt"]
    return "tools/train.py", f"{CFG}/multimodal/imagen/{IMAGEN[env('model_item', 'imagen_397M_text2im_64')]}", opts, dp * sh, "images/s"


def family_vit(kind):
    world = env("device_num", "N1C8")
    n = int(re.fullmatch(r"N(\d+)C(\d+)", world).group(2))
    bs = env("bs_item", 512, int)
    local = max(bs // n, 1)
    cfg = "ViT_large_patch16_384_ft_in1k_2n16c_dp_fp16o2.yaml" if kind == "finetune" else "ViT_base_patch16_224_pt_in1k_2n16c_dp_fp16o2.yaml"
    opts = ["Global.seed=1234", f"Global.local_batch_size={local}", f"Global.micro_batch_size={local}", "Global.global_batch_size=None",
            "Engine.run_mode=step", "Engine.num_train_epochs=1", f"Engine.max_steps={env('max_iter', 50, int)}", "Engine.eval_freq=-1", "Engine.logging_freq=1",
            "Engine.save_load.save_steps=-1", "Engine.save_load.save_epoch=-1",
            f"Engine.mix_precision.enable={env('fp_item', 'fp16') != 'fp32'}", f"Model.model.use_fused_attn={flag('use_fused_attn')}",
            f"Distributed.dp_degree={n}", f"Data.Train.sampler.batch_size={local}"]
    if kind == "pretrained":
        opts += ["Model.model.name=ViT_large_patch16_224"]
    if not env("DATA_DIR"):
        size = 384 if kind == "finetune" else 224
        opts += ["Data.Train.dataset.name=SyntheticImageDataset", f"Data.Train.dataset.image_size={size}", "Data.Train.loader.num_workers=0"]
    else:
        opts += [f"Data.Train.dataset.image_root={env('DATA_DIR')}", f"Data.Train.dataset.cls_label_path={env('DATA_DIR')}/train_list.txt"]
    return "tools/train.py", f"{CFG}/vis/vit/{cfg}", opts, n, "images/s"


FAMILIES = {"gpt": lambda: family_gpt("train"), "gpt_auto": lambda: family_gpt("auto"), "gpt_finetune": family_gpt_finetune, "ernie": family_ernie,
            "imagen": family_imagen, "vit_finetune": lambda: family_vit("finetune"), "vit_pretrained": lambda: family_vit("pretrained")}


def launch_prefix(world):
    if world == 1:
        return [sys.executable]
    per_node = min(world, env("GPUS_PER_NODE", 8, int))
    nnodes = max(world // per_node, 1)
    if nnodes > 1 and env("NNODES", 1, int) != nnodes:
        print(f"[tipc] this case spans {nnodes} nodes: run it on every node with NNODES={nnodes} NODE_RANK=<i> MASTER_ADDR=<node 0>", file=sys.stderr)
    return [sys.executable, "-m", "torch.distributed.run", f"--nnodes={env('NNODES', nnodes, int)}", f"--node-rank={env('NODE_RANK', 0, int)}",
            f"--nproc-per-node={per_node}", f"--master-addr={env('MASTER_ADDR', '127.0.0.1')}", f"--master-port={env('MASTER_PORT', 29533, int)}"]


def parse_log(path, skip, metric_key=None):
    ips, loss, metric, unit = [], None, None, None
    with open(path, errors="replace") as f:
        for line in f:
            if "[train]" in line:
                m = re.search(r"\bips: ([0-9.]+) ?([A-Za-z]+/s(?:ec)?)?", line)
                if m:
                    ips.append(float(m.group(1)))
                    unit = m.group(2) or unit
                m = re.search(r"\bloss: ([0-9.eE+-]+)", line)
                if m:
                    loss = float(m.group(1))
            elif metric_key and "[eval]" in line:
                m = re.search(rf"\b{re.escape(metric_key)}: ([0-9.eE+-]+)", line, re.I)
                if m:
                    metric = float(m.group(1))
    used = ips[skip:] if len(ips) > skip else ips
    return (sum(used) / len(used) if used else None), len(used), loss, metric, unit


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--family", required=True, choices=sorted(FAMILIES))
    p.add_argument("--dry-run", action="store_true")
    a = p.parse_args(argv)
    tool, cfg, opts, world, unit = FAMILIES[a.family]()
    opts += [o for o in env("TIPC_EXTRA_OPTS", "").split() if o]
    model_name = f"{env('model_item', a.family)}_bs{env('bs_item', 16)}_{env('fp_item', 'fp16')}_{env('run_mode', 'DP')}"
    device_num = env("device_num", "N1C1")
    cmd = launch_prefix(world) + [tool, "-c", cfg] + [x for o in opts for x in ("-o", o)]
    print("[tipc] " + " ".join(cmd), flush=True)
    if a.dry_run:
        return 0
    log_dir = env("LOG_DIR", os.path.join(ROOT, "tipc_logs"))
    os.makedirs(log_dir, exist_ok=True)
    log = os.path.join(log_dir, f"{model_name}_{device_num}_log")
    with open(log, "w") as f:
        try:
            rc = subprocess.run(cmd, cwd=ROOT, stdout=f, stderr=subprocess.STDOUT, timeout=env("timeout_s", 1800, int)).returncode
        except subprocess.TimeoutExpired:
            rc = 124
    metric_key = GLUE[env("task", "CoLA")][3] if a.family == "gpt_finetune" else None
    ips, n, loss, metric, logged_unit = parse_log(log, env("skip_steps", 5, int), env("metric_key", metric_key))
    out = {"model_name": model_name, "device_num": device_num, "n_gpus": world, "ips": ips, "unit": logged_unit or unit, "samples_used": n, "final_loss": loss, "return_code": rc, "log": log}
    if metric is not None:
        out["metric"] = metric
    with open(os.path.join(log_dir, f"{model_name}_{device_num}_speed.json"), "w") as f:
        json.dump(out, f)
    print("[tipc] " + json.dumps(out), flush=True)
    if rc != 0:
        with open(log, errors="replace") as f:
            sys.stderr.write("".join(f.readlines()[-25:]))
    return rc


if __name__ == "__main__":
    sys.exit(main())
