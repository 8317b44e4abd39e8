"""Convert a checkpoint between parallel layouts (see paddlefleetx_b200/utils/ckpt_convert.py).

    python tools/reshard.py --src output/epoch_0_step_1000 --dst output/tp2 --mp 2
    python tools/reshard.py --src ckpt_pp4 --dst ckpt_plain --to-plain --num-layers 32
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.abspath(os.path.join(os.path.dirname(__file__), "..")))

from paddlefleetx_b200.utils.ckpt_convert import convert  # noqa: E402


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--src", required=True)
    p.add_argument("--dst", required=True)
    p.add_argument("--mp", type=int, default=1, help="target tensor-parallel degree")
    p.add_argument("--to-plain", action="store_true", help="rename GPT pipeline keys to the non-pipeline model's names")
    p.add_argument("--num-layers", type=int, default=None)
    g = p.add_mutually_exclusive_group()
    g.add_argument("--fuse-qkv", action="store_true")
    g.add_argument("--split-qkv", action="store_true")
    p.add_argument("--num-heads", type=int, default=None)
    p.add_argument("--num-kv-heads", type=int, default=None, help="K/V heads of a grouped-query model (default: --num-heads)")
    a = p.parse_args()
    fuse = True if a.fuse_qkv else (False if a.split_qkv else None)
    if a.to_plain and a.num_layers is None:
        p.error("--to-plain needs --num-layers")
    out = convert(a.src, a.dst, a.mp, a.num_layers if a.to_plain else None, fuse, a.num_heads, a.num_kv_heads)
    print(f"wrote {out}")


if __name__ == "__main__":
    main()
