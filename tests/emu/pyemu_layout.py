"""ctypes front end of the layout goals' CPU emulation (tests only): tests/emu/_build/librg_emu_layout.so, compiled from
rg_emu_layout.cpp on first use with the flags of tests/emu/Makefile, and again whenever it or a kernel source is newer."""
import ctypes
import glob
import os
import subprocess
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.abspath(os.path.join(_HERE, "..", ".."))
_SO = os.path.join(_HERE, "_build", "librg_emu_layout.so")
CXXFLAGS = ["-O2", "-g", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-function", "-Wno-unused-variable", "-ffp-contract=off"]
_lib = None


def _stale():
    deps = [os.path.join(_HERE, "rg_emu_layout.cpp")] + glob.glob(os.path.join(_ROOT, "robogym_b200", "csrc", "*")) + \
        glob.glob(os.path.join(_ROOT, "include", "*.h"))
    return not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in deps)


def lib():
    """the layout goals' emulation library, with argtypes and restype of its entry points"""
    global _lib
    if _lib is None:
        if _stale():
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(_SO))
            os.close(fd)
            try:
                subprocess.check_call([os.environ.get("CXX", "g++"), *CXXFLAGS, "-shared", "-o", tmp, os.path.join(_HERE, "rg_emu_layout.cpp")])
                os.replace(tmp, _SO)                         # whole, even when two processes build at once
            finally:
                if os.path.exists(tmp):
                    os.remove(tmp)
        L = ctypes.CDLL(_SO)
        vp, ci, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32
        L.rge_layout_goals.argtypes = [ci, ci, ci, vp, vp, vp, vp, vp, vp, vp, ci, u32, u32, vp, vp, vp, vp, vp, vp]
        L.rge_layout_error.restype = ctypes.c_char_p
        _lib = L
    return _lib
