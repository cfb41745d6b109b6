"""H100-native cost-volume hot path for OpenStereo (sm_90a CUDA kernels behind a C ABI).

Sub-modules are loaded on first access (``openstereo_b200.ops`` etc.) so that ``python -m openstereo_b200.build`` can
run before the shared library exists.  The first access to ``ops`` / ``_lib`` loads ``lib/libopenstereo_b200.so`` and
RAISES if it is missing or lacks a symbol -- there is no PyTorch/CPU fallback for the product path.
"""
import importlib

_SUBMODULES = ("_lib", "ops", "aggregation", "host_models", "patch", "distributed", "geo", "build")

__all__ = ["ops", "aggregation", "host_models", "patch", "distributed", "geo"]


def __getattr__(name):
    if name in _SUBMODULES:
        return importlib.import_module("." + name, __name__)
    raise AttributeError("module %r has no attribute %r" % (__name__, name))
