"""Builds the native core in-tree (nvcc -gencode arch=compute_90a,code=sm_90a) before packaging.
`pip install -e .` / `python setup.py build_ext --inplace` both end up in uccl_b200/_build.py, the same
entry point `__graft_entry__.build()` uses."""
import importlib.util
import pathlib

import sys

from setuptools import Distribution, setup
from setuptools.command.build_py import build_py

try:
    from setuptools.command.bdist_wheel import bdist_wheel
except ImportError:  # older setuptools: the command lives in the wheel package
    from wheel.bdist_wheel import bdist_wheel

ROOT = pathlib.Path(__file__).parent


def _native_build():
    spec = importlib.util.spec_from_file_location("_ub_build", ROOT / "uccl_b200" / "_build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build()


class BuildWithNative(build_py):
    def run(self):
        _native_build()
        super().run()


class PlatformWheel(bdist_wheel):
    """The package data holds a pybind11 module for THIS interpreter and platform: tag the wheel accordingly
    (the reference forces the tag with an empty C extension, uccl/_platform_tag_stub.c + setup.py:42-47)."""

    def finalize_options(self):
        super().finalize_options()
        self.root_is_pure = False

    def get_tag(self):
        _, _, plat = super().get_tag()
        py = f"cp{sys.version_info.major}{sys.version_info.minor}"
        return py, py, plat


class BinaryDistribution(Distribution):
    def has_ext_modules(self):
        return True


setup(cmdclass={"build_py": BuildWithNative, "bdist_wheel": PlatformWheel}, distclass=BinaryDistribution)
