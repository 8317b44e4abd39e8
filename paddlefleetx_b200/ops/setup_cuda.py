"""``python -m paddlefleetx_b200.ops.setup_cuda`` — build the native library (reference ppfleetx/ops/setup_cuda.py builds the top-p sampling
op with ``paddle.utils.cpp_extension``; here one in-tree ``.so`` holds every kernel and ``ops/build.py`` drives nvcc for sm_90a)."""
from .build import build

if __name__ == "__main__":
    print(build(force=False))
