#!/usr/bin/env python3
"""Packaging of tutel_b200.  The native runtime is built ahead of time for sm_90a by tutel_b200/_build.py
(`python setup.py build_ext --inplace` or `pip install -e .` trigger it; set NO_CUDA=1 to skip the CUDA kernels'
compilation check when nvcc is absent - the pure-PyTorch CPU paths keep working)."""
import os
import subprocess
import sys

from setuptools import Command, find_packages, setup
from setuptools.command.build_ext import build_ext as _build_ext
from setuptools.command.build_py import build_py as _build_py

ROOT = os.path.dirname(os.path.abspath(__file__))


def build_native():
    if int(os.environ.get('NO_CUDA', '0')):
        print('NO_CUDA=1: skipping the native sm_90a extension')
        return
    sys.path.insert(0, ROOT)
    from tutel_b200 import _build
    print('built', _build.build(verbose=bool(int(os.environ.get('VERBOSE', '0')))))


class BuildExt(_build_ext):
    def run(self):
        build_native()


class BuildPy(_build_py):
    def run(self):
        build_native()
        super().run()


class Tester(Command):
    description = 'run the CPU test-suite (GPU tests: pytest -m gpu)'
    user_options = []

    def initialize_options(self):
        pass

    def finalize_options(self):
        pass

    def run(self):
        raise SystemExit(subprocess.call([sys.executable, '-m', 'pytest', '-q', 'tests', '-m', 'not gpu'], cwd=ROOT))


setup(
    name='tutel_b200',
    version='0.1.0',
    description='H100-native Mixture-of-Experts framework with the capabilities of microsoft/tutel',
    packages=find_packages(include=['tutel_b200', 'tutel_b200.*']),
    package_data={'tutel_b200': ['_C*.so', 'examples/README.md', 'examples/fairseq_moe/*']},
    python_requires='>=3.9',
    install_requires=[],
    cmdclass={'build_ext': BuildExt, 'build_py': BuildPy, 'test': Tester},
)
