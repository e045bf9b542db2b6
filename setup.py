"""``pip install .`` / ``python setup.py build_ext --inplace``: compiles the two native libraries IN TREE
(``openembedding_b200/lib/libexb_core.so`` with g++, ``libexb_cuda.so`` with nvcc for sm_90a) and ships them as
package data -- the counterpart of the reference's sdist that compiles its pybind module and TF ops at install
time (the reference's setup.py:19-38). The libraries are also (re)built lazily on first import when stale."""
import os
import sys

from setuptools import setup
from setuptools.command.build_py import build_py

HERE = os.path.dirname(os.path.abspath(__file__))


class BuildNative(build_py):
    def run(self):
        sys.path.insert(0, HERE)
        from openembedding_b200 import _build
        _build.build_core(verbose=True)
        try:
            _build.build_cuda(verbose=True)
        except RuntimeError as e:           # no nvcc on this box: the CPU/gloo configuration still works
            print("warning: CUDA library not built:", e)
        super().run()


setup(cmdclass={"build_py": BuildNative})
