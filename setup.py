"""Packaging.  The CUDA extension is built in-tree (``python __graft_entry__.py`` or on first
use through ``dfno_b200.ops.build``), so this is a plain source install."""
from setuptools import find_packages, setup

setup(
    name="dfno_b200",
    version="0.1.0",
    description="Hopper-native model-parallel Fourier Neural Operators (dfno-compatible API)",
    packages=find_packages(include=["dfno_b200*", "dfno"]),
    package_data={"dfno_b200": ["csrc/*"]},
    python_requires=">=3.10",
    install_requires=["torch>=2.6", "numpy"],
)
