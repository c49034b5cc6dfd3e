"""ctypes front end of the robot reset's CPU emulation (tests only): tests/emu/_build/librg_emu_arm.so, compiled from
rg_emu_arm.cpp on first use with the flags of tests/emu/Makefile, and again whenever it or a kernel source is newer."""
import ctypes
import glob
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.abspath(os.path.join(_HERE, "..", ".."))
_SO = os.path.join(_HERE, "_build", "librg_emu_arm.so")
CXXFLAGS = ["-O2", "-g", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-function", "-Wno-unused-variable", "-ffp-contract=off"]
_lib = None


def _stale():
    deps = [os.path.join(_HERE, "rg_emu_arm.cpp")] + glob.glob(os.path.join(_ROOT, "robogym_b200", "csrc", "*")) + glob.glob(os.path.join(_ROOT, "include", "*.h"))
    return not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in deps)


def lib():
    global _lib
    if _lib is None:
        if _stale():
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(_SO))
            os.close(fd)
            try:
                subprocess.check_call([os.environ.get("CXX", "g++"), *CXXFLAGS, "-shared", "-o", tmp, os.path.join(_HERE, "rg_emu_arm.cpp")])
                os.replace(tmp, _SO)                         # whole, even when two processes build at once
            finally:
                if os.path.exists(tmp):
                    os.remove(tmp)
        L = ctypes.CDLL(_SO)
        L.rgea_sample.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p, ctypes.c_void_p]
        _lib = L
    return _lib


def sample(nenv, dim, seed, epoch, mask=None):
    """[nenv, dim] float32: the draws of the selected environments, zero elsewhere"""
    out = np.zeros((nenv, dim), dtype=np.float32)
    m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
    lib().rgea_sample(nenv, dim, seed & 0xFFFFFFFF, epoch & 0xFFFFFFFF, None if m is None else m.ctypes.data, out.ctypes.data)
    return out
