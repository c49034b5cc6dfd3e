"""ctypes front end of the object groups' CPU emulation (tests only): tests/emu/_build/librg_emu_groups.so, compiled from
rg_emu_groups.cpp on first use with the flags of tests/emu/Makefile, and again whenever it or a kernel source is newer.

`object_groups(...)` takes the arguments of robogym_b200.rearrange_groups.object_groups as numpy values and returns the same
outputs as numpy arrays (a dict), from the kernel's own code."""
import ctypes
import glob
import os
import subprocess
import tempfile

import numpy as np

from robogym_b200 import engine, rearrange_groups as rgr

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.abspath(os.path.join(_HERE, "..", ".."))
_SO = os.path.join(_HERE, "_build", "librg_emu_groups.so")
CXXFLAGS = ["-O2", "-g", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-function", "-Wno-unused-variable", "-ffp-contract=off"]
_lib = None
OUTPUTS = ("group", "count", "material", "rgba", "scale", "mesh", "yaw", "quat", "ngroups")


def _stale():
    deps = [os.path.join(_HERE, "rg_emu_groups.cpp")] + glob.glob(os.path.join(_ROOT, "robogym_b200", "csrc", "*")) + \
        glob.glob(os.path.join(_ROOT, "include", "*.h"))
    return not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in deps)


def lib():
    """the object groups' emulation library, with argtypes and restype of its entry points"""
    global _lib
    if _lib is None:
        if _stale():
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(_SO))
            os.close(fd)
            try:
                subprocess.check_call([os.environ.get("CXX", "g++"), *CXXFLAGS, "-shared", "-o", tmp, os.path.join(_HERE, "rg_emu_groups.cpp")])
                os.replace(tmp, _SO)                         # whole, even when two processes build at once
            finally:
                if os.path.exists(tmp):
                    os.remove(tmp)
        L = ctypes.CDLL(_SO)
        L.rge_object_groups.argtypes = [ctypes.POINTER(engine.GroupsIn), ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(engine.GroupsOut)]
        L.rge_groups_error.restype = ctypes.c_char_p
        _lib = L
    return _lib


def empty_outputs(nenv, nobj, fill=None):
    """host output arrays; `fill` (a numpy RandomState) fills them with noise, to show what a call leaves untouched"""
    shapes = dict(group=(nenv, nobj), count=(nenv, nobj), material=(nenv, nobj), rgba=(nenv, nobj, 4), scale=(nenv, nobj), mesh=(nenv, nobj),
                  yaw=(nenv, nobj), quat=(nenv, nobj, 4), ngroups=(nenv,))
    out = {}
    for k, s in shapes.items():
        dt = np.float64 if k in ("rgba", "scale", "yaw", "quat") else np.int32
        out[k] = np.zeros(s, dt) if fill is None else (fill.uniform(-9, 9, s) if dt == np.float64 else fill.randint(-9, 9, s)).astype(dt)
    return out


def call(nenv, nobj, active, seed, epoch, mask=None, mask_len=None, out=None, group_mode="random", lam=(0.1, 5.0), n_materials=1,
         color_mode="random", palette=None, scale_range=(0.0, 0.0), n_candidates=0, replace=True, fixed_counts=None, mesh_mode=None):
    """rg_object_groups' code on the host: the outputs (dict of arrays); ValueError with the engine's message when refused"""
    keep = []

    def arr(x, dt):
        if x is None:
            return None
        a = np.ascontiguousarray(x, dtype=dt)
        keep.append(a)
        return a.ctypes.data

    c = engine.GroupsIn()
    c.nenv, c.nobj = nenv, nobj
    c.active = arr(np.broadcast_to(active, (nenv,)), np.int32)
    c.group_mode, c.lam_low, c.lam_high = rgr.GROUP_MODES[group_mode], float(lam[0]), float(lam[1])
    c.fixed_counts = arr(fixed_counts, np.int32)
    c.n_materials, c.color_mode = int(n_materials), rgr.COLOR_MODES[color_mode]
    c.palette = arr(palette, np.float64)
    c.n_palette = 0 if palette is None else len(palette)
    c.scale_low, c.scale_high = float(scale_range[0]), float(scale_range[1])
    c.mesh_mode = (0 if not n_candidates else 1 if replace else 2) if mesh_mode is None else mesh_mode
    c.n_candidates = int(n_candidates)
    c.seed, c.epoch = seed & 0xFFFFFFFF, epoch & 0xFFFFFFFF
    out = empty_outputs(nenv, nobj) if out is None else out
    o = engine.GroupsOut(**{k: out[k].ctypes.data for k in OUTPUTS})
    m = arr(mask, np.uint8)
    rc = lib().rge_object_groups(ctypes.byref(c), m, nenv if mask_len is None else mask_len, ctypes.byref(o))
    if rc != 0:
        raise ValueError(lib().rge_groups_error().decode())
    return out
