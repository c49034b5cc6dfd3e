"""ctypes front end of the CPU emulation build of the CUDA device code (tests only): tests/emu/_build/librg_emu.so, made on first
use.  RG_EMU_LIB names another build of tests/emu/rg_emu.cpp (e.g. tools/emu_stats.py's -DRG_STATS one), loaded as it is."""
import ctypes
import os
import subprocess

import numpy as np

from robogym_b200 import rearrange_goal as rg
from robogym_b200 import rearrange_obs as ro

_HERE = os.path.dirname(os.path.abspath(__file__))
_ENV_LIB = os.environ.get("RG_EMU_LIB")
NCON = 32
CON_STRIDE = 24
_lib = None


def lib():
    """the emulation library, with argtypes and restype of every entry point"""
    global _lib
    if _lib is None:
        if _ENV_LIB is None:
            subprocess.check_call(["make", "-C", _HERE, "-s", "_build/librg_emu.so"])
        L = ctypes.CDLL(_ENV_LIB or os.path.join(_HERE, "_build", "librg_emu.so"))
        vp, ci, cd, u32 = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_uint32
        pi = ctypes.POINTER(ctypes.c_int)
        # handles and the step
        L.rge_create_ex.restype = vp
        L.rge_create_ex.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ci, ci, ci]
        L.rge_destroy.argtypes = [vp]
        for f in ("rge_dbg_size", "rge_scratch_floats", "rge_small_bytes", "rge_ncon", "rge_pidw"):
            getattr(L, f).argtypes = [vp]
        L.rge_layout.argtypes = [vp, pi, ci]
        L.rge_name2id.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p]
        L.rge_model_field.restype = vp
        L.rge_model_field.argtypes = [vp, ctypes.c_char_p, pi]
        L.rge_set_const.argtypes = [vp] + [vp] * 6
        L.rge_set_sensordata.argtypes = [vp, vp]
        L.rge_set_mocap.argtypes = [vp, vp, vp]
        L.rge_step.argtypes = [vp, ci] + [vp] * 18 + [ci, ci]
        # a handle's model view: pair lists, geom scale
        L.rge_pairs.argtypes = [vp, vp, vp, ci, pi]
        L.rge_use_pairs.argtypes = [vp, vp, ci]
        L.rge_use_geom_scale.argtypes = [vp, vp]
        # hull support mapping
        L.rge_support_table.restype = vp
        L.rge_support_table.argtypes = [vp]
        L.rge_support_entries.restype = vp
        L.rge_support_entries.argtypes = [vp, pi]
        L.rge_support_cell.argtypes = [vp]
        L.rge_support_scan.argtypes = [vp, ci, vp, ci, vp]
        L.rge_support_set_vert.argtypes = [vp, vp]
        L.rge_support_build_seconds.restype = cd
        L.rge_support_build_seconds.argtypes = [vp]
        # placement
        L.rge_philox.argtypes = [ci, vp, u32, u32, vp]
        L.rge_body_aabb.argtypes = [vp, ci, vp, vp, vp, vp, vp, vp, vp, vp]
        L.rge_place.argtypes = [ci, ci, vp, vp, vp, vp, ci, ci, ci, cd, cd, vp, u32, u32, vp, vp, vp]
        # goal evaluation and goal orientations
        L.rge_goal.argtypes = [ctypes.POINTER(rg.GoalIn), vp, vp, ctypes.POINTER(rg.GoalOut)]
        L.rge_goal_error.restype = ctypes.c_char_p
        L.rge_goal_rot.argtypes = [ci, ci, vp, vp, ci, u32, u32, vp, vp]
        L.rge_parallel_quats.argtypes = [vp]
        # rearrange observations
        L.rge_obs.argtypes = [ctypes.POINTER(ro.ObsIn), vp, ctypes.POINTER(ro.ObsOut)]
        L.rge_obs_error.restype = ctypes.c_char_p
        _lib = L
    return _lib


def philox_check():
    """the sm_90a check of the device Philox against cuRAND's (needs a GPU): rg_philox_mismatches(n, k0, k1)"""
    subprocess.check_call(["make", "-C", _HERE, "-s", "_build/librg_philox_check.so"])
    L = ctypes.CDLL(os.path.join(_HERE, "_build", "librg_philox_check.so"))
    L.rg_philox_mismatches.restype = ctypes.c_longlong
    L.rg_philox_mismatches.argtypes = [ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32]
    return L


# RgLayout's members in declaration order (robogym_b200/csrc/rg_defs.h): float offsets into a warp's scratch, then the capacities
LAYOUT_FIELDS = ("qpos", "qvel", "ctrl", "pid", "warm", "lpos", "lquat", "xpos", "xquat", "gxpos", "sxpos", "S", "M", "H", "Sdot", "I10",
                 "crb", "bias", "smooth", "qacc", "Ma", "search", "Mv", "qfc", "tmp", "tlen", "tvel", "tJn", "tJi", "tJv", "alen", "aforce",
                 "con", "cu", "cw", "cF", "cprm", "el_i", "el_D", "el_jar", "el_jv", "el_f", "tileJ", "tileWJ", "tileDof", "cand", "cand2",
                 "scal", "eldof", "env", "cdof", "sep", "stage", "mocap", "ncon", "nel", "tile", "total")


def layout(blob, ncon=0, nel=0, tile=0):
    """the scratch layout rg_make_layout gives the model at these capacities (0 = engine default): {member: int}"""
    h = lib().rge_create_ex(bytes(blob), len(blob), ncon, nel, tile)
    if not h:
        raise RuntimeError("rge_create failed")
    try:
        out = (ctypes.c_int * len(LAYOUT_FIELDS))()
        n = lib().rge_layout(h, out, len(out))
    finally:
        lib().rge_destroy(h)
    if n != len(LAYOUT_FIELDS):
        raise RuntimeError(f"RgLayout has {n} members, LAYOUT_FIELDS names {len(LAYOUT_FIELDS)}")
    return dict(zip(LAYOUT_FIELDS, out))


def _p(a):
    return None if a is None else a.ctypes.data


class EmuBatch:
    """Same state layout as robogym_b200.engine.Batch, backed by the emulation library."""

    def __init__(self, blob, dims, nenv, contact_capacity=0, row_capacity=0, dofs_per_contact=0):
        self.h = lib().rge_create_ex(bytes(blob), len(blob), contact_capacity, row_capacity, dofs_per_contact)
        if not self.h:
            raise RuntimeError("rge_create failed")
        self.ncon_cap = lib().rge_ncon(self.h)
        self.nenv = nenv
        self.d = dims
        f = np.float32
        self.qpos = np.zeros((nenv, dims["nq"]), f)
        self.qvel = np.zeros((nenv, dims["nv"]), f)
        self.ctrl = np.zeros((nenv, dims["nu"]), f)
        self.pid = np.zeros((nenv, lib().rge_pidw(self.h) * dims["nu"]), f)
        self.warm = np.zeros((nenv, dims["nv"]), f)
        self.time = np.zeros(nenv, f)
        self.xfrc = None
        self.timestep = None
        self.site_xpos = np.zeros((nenv, dims["nsite"], 3), f)
        self.body_xpos = np.zeros((nenv, dims["nbody"], 3), f)
        self.body_xquat = np.zeros((nenv, dims["nbody"], 4), f)
        self.geom_xpos = np.zeros((nenv, dims["ngeom"], 3), f)
        self.act_force = np.zeros((nenv, dims["nu"]), f)
        self.qacc = np.zeros((nenv, dims["nv"]), f)
        self.contact = np.zeros((nenv, self.ncon_cap, 4), f)
        self.ncon = np.zeros(nenv, np.int32)
        self.warn = np.zeros(nenv, np.int32)
        self.dbg = np.zeros((nenv, lib().rge_dbg_size(self.h)), f)
        self.sensordata = np.zeros((nenv, dims.get("nsensordata", 0)), f)
        self.mocap_pos = np.zeros((nenv, dims.get("nmocap", 0), 3), f) if dims.get("nmocap", 0) else None
        self.mocap_quat = np.zeros((nenv, dims.get("nmocap", 0), 4), f) if dims.get("nmocap", 0) else None

    def model_field(self, name, dtype):
        n = ctypes.c_int()
        p = lib().rge_model_field(self.h, name.encode(), ctypes.byref(n))
        ct = ctypes.c_int32 if dtype == np.int32 else ctypes.c_float
        return np.frombuffer((ct * n.value).from_address(p), dtype=dtype)

    def use_pairs(self, pairs, n):
        """step the first n pairs of `pairs` (packed g1 | g2 << 16) instead of the model's static list, as the engine does for an
        environment with its own list; the batch keeps the array alive"""
        self._pairs = np.ascontiguousarray(pairs, dtype=np.uint32)
        lib().rge_use_pairs(self.h, _p(self._pairs), n)

    def use_geom_scale(self, row):
        """step with the [ngeom] geom_mesh_scale row (None: unbound, every factor 1), as the engine binds it per environment; the
        batch keeps the array alive.  Returns ngeom."""
        self._geom_scale = None if row is None else np.ascontiguousarray(row, dtype=np.float32)
        return lib().rge_use_geom_scale(self.h, _p(self._geom_scale))

    def step(self, nsub, final_forward=1):
        lib().rge_set_mocap(self.h, _p(self.mocap_pos), _p(self.mocap_quat))
        lib().rge_set_sensordata(self.h, _p(self.sensordata) if self.sensordata.size else None)
        lib().rge_step(self.h, self.nenv, _p(self.qpos), _p(self.qvel), _p(self.ctrl), _p(self.pid), _p(self.warm), _p(self.time),
                       _p(self.xfrc), _p(self.timestep), _p(self.site_xpos), _p(self.body_xpos), _p(self.body_xquat),
                       _p(self.geom_xpos), _p(self.act_force), _p(self.qacc), _p(self.contact), _p(self.ncon), _p(self.warn),
                       _p(self.dbg), nsub, final_forward)

    def forward(self):
        self.step(0, 1)

    def set_const(self):
        """mj_setConst of the (edited) model through the kernel code: dict of float32 arrays"""
        d = self.d
        out = dict(dof_invweight0=np.zeros(d["nv"], np.float32), body_invweight0=np.zeros(2 * d["nbody"], np.float32),
                   tendon_invweight0=np.zeros(d["ntendon"], np.float32), tendon_length0=np.zeros(d["ntendon"], np.float32),
                   body_subtreemass=np.zeros(d["nbody"], np.float32), opt_meaninertia=np.zeros(1, np.float32))
        lib().rge_set_const(self.h, *[_p(out[k]) if out[k].size else None for k in ("dof_invweight0", "body_invweight0", "tendon_invweight0", "tendon_length0", "body_subtreemass", "opt_meaninertia")])
        return out

    def dbg_view(self, env=0):
        d = self.d
        nv, nt, nu = d["nv"], d["ntendon"], d["nu"]
        g = self.dbg[env]
        o = 0
        out = {}
        out["M"] = g[o:o + nv * nv].reshape(nv, nv); o += nv * nv
        for k in ("bias", "passive", "qfa", "smooth", "qacc", "qfc"):
            out[k] = g[o:o + nv]; o += nv
        out["tlen"] = g[o:o + nt]; o += nt
        out["alen"] = g[o:o + nu]; o += nu
        out["aforce"] = g[o:o + nu]; o += nu
        out["ncon"], out["nel"], out["niter"], out["warn"] = [int(x) for x in g[o:o + 4]]; o += 4
        out["con"] = g[o:o + self.ncon_cap * CON_STRIDE].reshape(self.ncon_cap, CON_STRIDE); o += self.ncon_cap * CON_STRIDE
        out["tJ"] = g[o:o + nt * nv].reshape(nt, nv)
        return out

    def __del__(self):
        if getattr(self, "h", None) and _lib is not None:
            _lib.rge_destroy(self.h)
            self.h = None
