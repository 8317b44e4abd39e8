# CUDA 12.9 + PyTorch image for H100 (sm_90a); the kernel library is compiled at image build time.
FROM nvcr.io/nvidia/pytorch:25.06-py3
WORKDIR /workspace/paddlefleetx_b200
COPY . .
RUN pip install --no-cache-dir -r requirements.txt && python -m paddlefleetx_b200.ops.build
ENV PYTHONPATH=/workspace/paddlefleetx_b200
CMD ["python", "tools/train.py", "-c", "paddlefleetx_b200/configs/nlp/gpt/pretrain_gpt_345M_single_card.yaml"]
