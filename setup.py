#!/usr/bin/env python
"""Packaging for deepspeed_b200.

``pip install .`` installs the Python package and the ``bin/`` entry points.  The two native libraries
(``libdsb200_cuda.so`` for sm_90a, ``libdsb200_cpu.so`` for the host runtime) are built IN-TREE into ``deepspeed_b200/lib``:

* ``python setup.py build_ext --inplace`` (or ``DS_BUILD_OPS=1 pip install .``) compiles them ahead of time;
* otherwise they are compiled on first use by the op builders (``deepspeed_b200/op_builder``), like the reference's JIT path.

Environment knobs: ``DS_BUILD_OPS`` (0/1), ``DSB200_BUILD_JOBS``, ``DSB200_NVCC``, ``DSB200_CXX``.
"""
import os
import re
import sys

from setuptools import Command, find_packages, setup
from setuptools.command.build_py import build_py

ROOT = os.path.dirname(os.path.abspath(__file__))


def read_version():
    with open(os.path.join(ROOT, "version.txt")) as f:
        return f.read().strip()


def read_requirements(name):
    path = os.path.join(ROOT, "requirements", name)
    if not os.path.exists(path):
        return []
    with open(path) as f:
        return [l.strip() for l in f if l.strip() and not l.startswith("#")]


class BuildNative(Command):
    """Compile both native libraries into ``deepspeed_b200/lib``."""
    description = "build the sm_90a CUDA library and the host runtime library in-tree"
    user_options = [("inplace", "i", "accepted for compatibility (libraries are always built in-tree)"),
                    ("parallel=", "j", "number of parallel compile jobs")]

    def initialize_options(self):
        self.inplace, self.parallel = True, None

    def finalize_options(self):
        if self.parallel is not None:
            os.environ["DSB200_BUILD_JOBS"] = str(self.parallel)

    def run(self):
        sys.path.insert(0, ROOT)
        from deepspeed_b200.op_builder import build_all
        for lib in build_all(verbose=True):
            print(f"built {lib}")


class BuildPy(build_py):

    def run(self):
        if os.environ.get("DS_BUILD_OPS", "0") == "1":
            self.run_command("build_ext")
        super().run()


scripts = [os.path.join("bin", f) for f in sorted(os.listdir(os.path.join(ROOT, "bin")))]

setup(
    name="deepspeed_b200",
    version=read_version(),
    description="H100-native (sm_90a) large-model training and inference framework with the DeepSpeed feature set",
    long_description=open(os.path.join(ROOT, "README.md")).read(),
    long_description_content_type="text/markdown",
    packages=find_packages(include=["deepspeed_b200", "deepspeed_b200.*"]),
    package_data={"deepspeed_b200": ["csrc/**/*", "lib/*.so", "autotuning/config_templates/*.json"]},
    include_package_data=True,
    scripts=scripts,
    python_requires=">=3.9",
    install_requires=read_requirements("requirements.txt"),
    extras_require={
        "autotuning": read_requirements("requirements-autotuning.txt"),
        "inf": read_requirements("requirements-inf.txt"),
        "dev": read_requirements("requirements-dev.txt"),
    },
    cmdclass={"build_ext": BuildNative, "build_py": BuildPy},
    classifiers=["Programming Language :: Python :: 3", "Environment :: GPU :: NVIDIA CUDA :: 12"],
)
