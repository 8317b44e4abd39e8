"""Training entry point:  python tools/train.py -c <yaml> [-o key.sub=value ...]

Flow (reference tools/train.py:44-73): parse -> config -> device -> init_dist_env -> set_seed -> build_module ->
dataloaders (Train/Eval) -> inject epochs/step_each_epoch/total_steps into Optimizer.lr -> EagerEngine ->
optional load() -> fit().  Launch multi-GPU with torchrun (one process per GPU).
"""
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

from paddlefleetx_b200.core import EagerEngine  # noqa: E402
from paddlefleetx_b200.data import build_dataloader  # noqa: E402
from paddlefleetx_b200.distributed.apis import env  # noqa: E402
from paddlefleetx_b200.models import build_module  # noqa: E402
from paddlefleetx_b200.utils import config  # noqa: E402


def main(argv=None):
    args = config.parse_args(argv)
    env.init_process_group("gpu")
    cfg = config.get_config(args.config, overrides=args.override, show=False)
    env.init_dist_env(cfg)
    env.set_seed(cfg.Global.seed)
    module = build_module(cfg)
    config.print_config(cfg)

    train_loader = build_dataloader(cfg.Data, "Train")
    eval_loader = build_dataloader(cfg.Data, "Eval") if cfg.Engine.eval_freq and cfg.Engine.eval_freq > 0 and "Eval" in cfg.Data else None
    if isinstance(cfg.Optimizer.get("lr"), dict):
        total = cfg.Engine.max_steps
        if cfg.Engine.get("run_mode", "step") == "epoch":
            # an epoch-mode run ends after num_train_epochs passes: schedules must span that, not a max_steps inherited from a pre-training base
            # recipe (the reference passes max_steps through unconditionally, tools/train.py:60-64, and the warm-up then never finishes)
            span = cfg.Engine.num_train_epochs * len(train_loader)
            total = min(total, span) if total and total > 0 else span
        cfg.Optimizer.lr.update({"epochs": cfg.Engine.num_train_epochs, "step_each_epoch": len(train_loader), "total_steps": total})
        known = {"CosineAnnealingWithWarmupDecay": ("epochs", "step_each_epoch", "total_steps")}
        for k in known.get(cfg.Optimizer.lr.get("name"), ()):
            cfg.Optimizer.lr.pop(k, None)

    engine = EagerEngine(configs=cfg, module=module)
    if cfg.Engine.save_load.ckpt_dir is not None:
        engine.load()
    engine.fit(train_data_loader=train_loader, valid_data_loader=eval_loader, epoch=cfg.Engine.num_train_epochs)
    return engine


if __name__ == "__main__":
    main()
    env.destroy_process_group()
