#!/bin/bash
# GPT: pretrain_gpt_6.7B_single_card on 1 GPU(s)
# 6.7B needs 106 GB for weights + AdamW state: it does not fit one 80 GB H100.  Add "-o Distributed.sharding.sharding_degree=2" on two GPUs
# (python -m torch.distributed.run --nproc-per-node 2 ...) or use pretrain_gpt_6.7B_sharding16.sh.
set -e
cd "$(dirname "$0")/../.."
python tools/train.py -c paddlefleetx_b200/configs/nlp/gpt/pretrain_gpt_6.7B_single_card.yaml "$@"
