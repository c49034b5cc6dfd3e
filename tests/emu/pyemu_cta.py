"""ctypes front end of the CPU emulation of the one-environment-per-CTA step (tests only): tests/emu/rg_emu_cta.cpp compiled twice
with the flags of tests/emu/Makefile, as tests/emu/_build/librg_emu_cta.so (-DRG_COOP: the cooperative sections loop over 32 W
threads) and librg_emu_cta1.so (one warp per environment), on first use and again whenever a source is newer."""
import ctypes
import glob
import os
import subprocess
import tempfile

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.abspath(os.path.join(_HERE, "..", ".."))
CXXFLAGS = ["-O2", "-g", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-function", "-Wno-unused-variable", "-ffp-contract=off"]
_libs = {}


def _build(so, defines):
    src = os.path.join(_HERE, "rg_emu_cta.cpp")
    deps = [src] + glob.glob(os.path.join(_ROOT, "robogym_b200", "csrc", "*")) + glob.glob(os.path.join(_ROOT, "include", "*.h"))
    if os.path.exists(so) and os.path.getmtime(so) >= max(os.path.getmtime(d) for d in deps):
        return
    os.makedirs(os.path.dirname(so), exist_ok=True)
    fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(so))
    os.close(fd)
    try:
        subprocess.check_call([os.environ.get("CXX", "g++"), *CXXFLAGS, *defines, "-shared", "-o", tmp, src])
        os.replace(tmp, so)                                  # whole, even when two processes build at once
    finally:
        if os.path.exists(tmp):
            os.remove(tmp)


def lib(coop):
    """the cooperative (coop=True) or the one-warp build, with argtypes and restype of its entry points"""
    if coop not in _libs:
        so = os.path.join(_HERE, "_build", "librg_emu_cta.so" if coop else "librg_emu_cta1.so")
        _build(so, ["-DRG_COOP"] if coop else [])
        L = ctypes.CDLL(so)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.rgc_create.restype = vp
        L.rgc_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ci, ci, ci]
        L.rgc_destroy.argtypes = [vp]
        L.rgc_ncon.argtypes = [vp]
        L.rgc_ns.argtypes = [vp]
        L.rgc_set_warps.argtypes = [ci]
        L.rgc_step.argtypes = [vp, ci] + [vp] * 10 + [ci, ci]
        L.rgc_chol.argtypes = [ci] + [vp] * 6
        _libs[coop] = L
    return _libs[coop]
