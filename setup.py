"""``pip install -e .`` builds the sm_90a kernel library and the C++ dataset helper in-tree (reference setup.py:17-38 runs the C++
``make`` at install time and ships ``fast_index_map_helpers.so`` as package data)."""
import os
import subprocess
import sys

from setuptools import find_packages, setup
from setuptools.command.build_py import build_py


class BuildNative(build_py):
    def run(self):
        here = os.path.dirname(os.path.abspath(__file__))
        subprocess.check_call([sys.executable, "-m", "paddlefleetx_b200.ops.build"], cwd=here)
        super().run()


setup(
    name="paddlefleetx_b200",
    version="0.1.0",
    description="H100 (sm_90a) large-model training and serving framework (GPT / ERNIE / MoE / ViT / MoCo / Imagen recipes)",
    packages=find_packages(include=["paddlefleetx_b200", "paddlefleetx_b200.*", "ppfleetx", "ppfleetx.*"]),
    package_data={"paddlefleetx_b200": ["configs/**/*.yaml", "ops/*.so", "ops/csrc/*", "data/data_tools/cpp/*"]},
    python_requires=">=3.10",
    install_requires=open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "requirements.txt")).read().split(),
    cmdclass={"build_py": BuildNative},
)
