"""ctypes front end of the settle launch's CPU emulation (tests only): tests/emu/_build/librg_emu_settle.so, compiled from
rg_emu_settle.cpp on first use with the flags of tests/emu/Makefile, and again whenever it or a kernel source is newer.
SettleBatch has EmuBatch's state layout, backed by this library's own handles."""
import ctypes
import glob
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ROOT = os.path.abspath(os.path.join(_HERE, "..", ".."))
_SO = os.path.join(_HERE, "_build", "librg_emu_settle.so")
CXXFLAGS = ["-O2", "-g", "-fPIC", "-std=c++17", "-Wall", "-Wno-unused-function", "-Wno-unused-variable", "-ffp-contract=off"]
_lib = None


def _stale():
    deps = [os.path.join(_HERE, f) for f in ("rg_emu_settle.cpp", "rg_emu.cpp")] + glob.glob(os.path.join(_ROOT, "robogym_b200", "csrc", "*")) + \
        glob.glob(os.path.join(_ROOT, "include", "*.h"))
    return not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(d) for d in deps)


def lib():
    """the settle emulation library, with argtypes and restype of the entry points SettleBatch uses"""
    global _lib
    if _lib is None:
        if _stale():
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            fd, tmp = tempfile.mkstemp(suffix=".so", dir=os.path.dirname(_SO))
            os.close(fd)
            try:
                subprocess.check_call([os.environ.get("CXX", "g++"), *CXXFLAGS, "-shared", "-o", tmp, os.path.join(_HERE, "rg_emu_settle.cpp")])
                os.replace(tmp, _SO)                         # whole, even when two processes build at once
            finally:
                if os.path.exists(tmp):
                    os.remove(tmp)
        L = ctypes.CDLL(_SO)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.rge_create_ex.restype = vp
        L.rge_create_ex.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ci, ci, ci]
        L.rge_destroy.argtypes = [vp]
        for f in ("rge_dbg_size", "rge_ncon", "rge_pidw"):
            getattr(L, f).argtypes = [vp]
        L.rge_model_field.restype = vp
        L.rge_model_field.argtypes = [vp, ctypes.c_char_p, ctypes.POINTER(ci)]
        L.rge_set_sensordata.argtypes = [vp, vp]
        L.rge_set_mocap.argtypes = [vp, vp, vp]
        L.rges_step.argtypes = [vp, vp, ci] + [vp] * 18 + [ci, ci]
        L.rges_settle.argtypes = [vp, vp, ci] + [vp] * 18 + [vp, ci, ctypes.c_float, ci, ci, ci]
        _lib = L
    return _lib


def _p(a):
    return None if a is None else a.ctypes.data


class SettleBatch:
    """nenv environments of one model with EmuBatch's state and output arrays; step() and settle() take a mask"""

    def __init__(self, blob, dims, nenv, contact_capacity=0, row_capacity=0, dofs_per_contact=0):
        L = lib()
        self.h = L.rge_create_ex(bytes(blob), len(blob), contact_capacity, row_capacity, dofs_per_contact)
        if not self.h:
            raise RuntimeError("rge_create failed")
        self.nenv, self.d = nenv, dims
        f = np.float32
        self.qpos = np.zeros((nenv, dims["nq"]), f)
        self.qvel = np.zeros((nenv, dims["nv"]), f)
        self.ctrl = np.zeros((nenv, dims["nu"]), f)
        self.pid = np.zeros((nenv, L.rge_pidw(self.h) * dims["nu"]), f)
        self.warm = np.zeros((nenv, dims["nv"]), f)
        self.time = np.zeros(nenv, f)
        self.xfrc = self.timestep = None
        self.site_xpos = np.zeros((nenv, dims["nsite"], 3), f)
        self.body_xpos = np.zeros((nenv, dims["nbody"], 3), f)
        self.body_xquat = np.zeros((nenv, dims["nbody"], 4), f)
        self.geom_xpos = np.zeros((nenv, dims["ngeom"], 3), f)
        self.act_force = np.zeros((nenv, dims["nu"]), f)
        self.qacc = np.zeros((nenv, dims["nv"]), f)
        self.contact = np.zeros((nenv, L.rge_ncon(self.h), 4), f)
        self.ncon = np.zeros(nenv, np.int32)
        self.warn = np.zeros(nenv, np.int32)
        self.dbg = np.zeros((nenv, L.rge_dbg_size(self.h)), f)
        self.sensordata = np.zeros((nenv, dims.get("nsensordata", 0)), f)
        nm = dims.get("nmocap", 0)
        self.mocap_pos = np.zeros((nenv, nm, 3), f) if nm else None
        self.mocap_quat = np.zeros((nenv, nm, 4), f) if nm else None

    def model_field(self, name, dtype):
        n = ctypes.c_int()
        p = lib().rge_model_field(self.h, name.encode(), ctypes.byref(n))
        ct = ctypes.c_int32 if dtype == np.int32 else ctypes.c_float
        return np.frombuffer((ct * n.value).from_address(p), dtype=dtype)

    def _args(self, mask):
        L = lib()
        L.rge_set_mocap(self.h, _p(self.mocap_pos), _p(self.mocap_quat))
        L.rge_set_sensordata(self.h, _p(self.sensordata) if self.sensordata.size else None)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self._mask = m                                         # alive for the call
        return [self.h, _p(m), self.nenv] + [_p(a) for a in (self.qpos, self.qvel, self.ctrl, self.pid, self.warm, self.time, self.xfrc, self.timestep,
                                                                self.site_xpos, self.body_xpos, self.body_xquat, self.geom_xpos, self.act_force,
                                                                self.qacc, self.contact, self.ncon, self.warn, self.dbg)]

    def step(self, nsub, final_forward=1, mask=None):
        """rg_step_subset (mask None: rg_step)"""
        lib().rges_step(*self._args(mask), nsub, final_forward)

    def settle(self, dofs, damping, nsub, final_forward=1, mask=None, reads=3):
        """rg_step_settle; `reads` 3 = the kernel's settle, 1 / 2 = the override on one read of dof_damping only"""
        d = np.ascontiguousarray(dofs, dtype=np.int32)
        lib().rges_settle(*self._args(mask), _p(d), len(d), damping, nsub, final_forward, reads)

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.rge_destroy(self.h)
            self.h = None
