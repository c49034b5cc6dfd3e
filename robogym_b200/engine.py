"""Python binding of the C ABI (include/robogym_b200.h) + the batched simulation object.

`BatchedSim` is the batched counterpart of `robogym.mujoco.simulation_interface.SimulationInterface`
(robogym/mujoco/simulation_interface.py:25-250): `step()` = `sim.step()` (nsubsteps x mj_step)
+ `sim.forward()`, `forward()`, `reset()`, `qpos`/`qvel`/`ctrl` accessors -- for `nenv`
independent environments whose state lives in torch CUDA tensors ([nenv, n], float32).

There is NO CPU fallback: without the compiled CUDA library or without a GPU the constructors
raise.  (The fp64 CPU oracle under oracle/ is test infrastructure and is never imported here.)
"""
import ctypes
import os

import numpy as np

from . import modelblob

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("RG_LIB", os.path.join(_HERE, "librobogym_b200.so"))  # RG_LIB: e.g. the -DRG_PROFILE build

# enum rg_field (include/robogym_b200.h)
(QPOS, QVEL, CTRL, PID, WARMSTART, TIME, XFRC, TIMESTEP, SITE_XPOS, BODY_XPOS, BODY_XQUAT, GEOM_XPOS,
 ACT_FORCE, QACC, CONTACT, NCON, WARN, DBG, BODY_XVEL, MOCAP_POS, MOCAP_QUAT, SENSORDATA) = range(22)
MAX_CONTACTS = 32
CON_STRIDE = 24

_lib = None


class EngineError(RuntimeError):
    pass


def lib():
    """Load librobogym_b200.so (built in-tree by `python -m robogym_b200.build`)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineError(
                f"{LIB_PATH} is missing: build it with `python -m robogym_b200.build` "
                "(nvcc, sm_90a). There is no CPU fallback."
            )
        L = ctypes.CDLL(LIB_PATH)
        vp, ci = ctypes.c_void_p, ctypes.c_int
        L.rg_last_error.restype = ctypes.c_char_p
        L.rg_model_load.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ci, ctypes.POINTER(vp)]
        L.rg_model_destroy.argtypes = [vp]
        L.rg_model_dim.argtypes = [vp, ctypes.c_char_p]
        L.rg_model_set_field.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_size_t]
        L.rg_model_set_field_async.argtypes = [vp, ctypes.c_char_p, vp, ctypes.c_size_t, vp]
        L.rg_model_name2id.argtypes = [vp, ctypes.c_char_p, ctypes.c_char_p]
        L.rg_model_id2name.argtypes = [vp, ctypes.c_char_p, ci]
        L.rg_model_id2name.restype = ctypes.c_char_p
        L.rg_dbg_size.argtypes = [vp]
        L.rg_scratch_bytes.argtypes = [vp]
        L.rg_batch_create.argtypes = [vp, ci, ctypes.POINTER(vp)]
        L.rg_batch_create_ex.argtypes = [vp, ci, ci, ci, ci, ctypes.POINTER(vp)]
        L.rg_batch_capacity.argtypes = [vp, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)]
        L.rg_batch_dbg_size.argtypes = [vp]
        L.rg_batch_scratch_bytes.argtypes = [vp]
        L.rg_batch_destroy.argtypes = [vp]
        L.rg_batch_bind.argtypes = [vp, ci, vp]
        L.rg_batch_bind_param.argtypes = [vp, ctypes.c_char_p, vp]
        L.rg_model_origin.argtypes = [vp, ctypes.POINTER(ctypes.c_float)]
        L.rg_batch_launch_info.argtypes = [vp, ctypes.POINTER(ci), ctypes.POINTER(ci), ctypes.POINTER(ci)]
        L.rg_batch_set_balance.argtypes = [vp, ci]
        L.rg_step.argtypes = [vp, ci, ci, vp]
        L.rg_step_subset.argtypes = [vp, vp, ci, ci, vp]
        L.rg_forward.argtypes = [vp, vp]
        L.rg_reset.argtypes = [vp, vp, vp]
        L.rg_set_const.argtypes = [vp, vp, vp]
        L.rg_batch_update_pairs.argtypes = [vp, vp, vp]
        L.rg_batch_mark_pairs_stale.argtypes = [vp, vp, vp]
        L.rg_batch_set_pair_capacity.argtypes = [vp, ci]
        L.rg_batch_pair_info.argtypes = [vp, ctypes.POINTER(ci), ctypes.POINTER(vp)]
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise EngineError(lib().rg_last_error().decode())


def check_geom_dataid(v, m):
    """Per-environment geom_dataid rows ([rows, ngeom]) must hold -1 or a mesh id on mesh geoms and -1 on every other geom."""
    a = np.asarray(v.detach().cpu() if hasattr(v, "detach") else v).reshape(-1, m["ngeom"])
    mesh = np.asarray(m["geom_type"]) == 7
    ok = np.where(mesh[None, :], (a >= -1) & (a < m["nmesh"]), a == -1)
    if not ok.all():
        raise ValueError("geom_dataid: -1 or a mesh id on mesh geoms, -1 on every other geom")


def check_mesh_scale(v, name="mesh_scale"):
    """mesh_scale (and geom_mesh_scale) values must be finite and > 0: the narrow phase scales the arg-max vertex of the
    unscaled hull, which is the scaled hull's support point only for a positive scale."""
    a = np.asarray(v.detach().cpu() if hasattr(v, "detach") else v, dtype=np.float64)
    if not (np.isfinite(a).all() and (a > 0).all()):
        raise ValueError(f"{name} must be finite and positive")


class DeviceModel:
    """A compiled model uploaded to one GPU (rg_model)."""

    def __init__(self, blob, device=0):
        self.blob = bytes(blob)
        self.host = modelblob.unpack(self.blob)  # float64 host copy, source of truth for edits
        self.mesh_scale = np.ones(self.host["nmesh"])  # engine-derived parameter (not in the blob): uniform scale per hull
        self.device = int(device)
        h = ctypes.c_void_p()
        _check(lib().rg_model_load(self.blob, len(self.blob), self.device, ctypes.byref(h)))
        self.h = h

    def dim(self, name):
        return self.host[name]

    def set_field(self, name, values, stream=None):
        """Overwrite a model array (randomisers write e.g. geom_friction, dof_damping, opt_gravity).  The upload is ordered
        on `stream` (a raw cudaStream_t; default: torch's current stream on the model's device when torch is loaded).
        `mesh_scale` ([nmesh], finite and > 0) scales every hull uniformly without touching mesh_vert.  `geom_mesh_scale` exists
        per environment only (BatchedSim.set_param)."""
        if name == "geom_mesh_scale":
            raise ValueError("geom_mesh_scale is a per-environment array (BatchedSim.set_param); scale hulls model-wide with mesh_scale")
        if name == "mesh_scale":
            check_mesh_scale(values)
        arr = self.mesh_scale if name == "mesh_scale" else self.host[name]
        arr[...] = np.asarray(values, dtype=arr.dtype).reshape(arr.shape)
        buf = np.ascontiguousarray(arr)
        if stream is None:
            import sys

            t = sys.modules.get("torch")
            stream = t.cuda.current_stream(self.device).cuda_stream if t is not None and t.cuda.is_available() else 0
        _check(lib().rg_model_set_field_async(self.h, name.encode(), buf.ctypes.data, buf.size, ctypes.c_void_p(stream)))

    def name2id(self, objtype, name):
        """mjModel.<objtype>_name2id through the C ABI (the blob carries its name tables)."""
        i = lib().rg_model_name2id(self.h, objtype.encode(), name.encode())
        if i < 0:
            raise ValueError(f'No "{objtype}" with name {name} exists.')
        return i

    def id2name(self, objtype, i):
        """mjModel.<objtype>_id2name through the C ABI; None for an unnamed object"""
        n = lib().rg_model_id2name(self.h, objtype.encode(), int(i))
        if n is None:
            raise ValueError(f'No "{objtype}" with id {i} exists.')
        return n.decode() or None

    @property
    def dbg_size(self):
        return lib().rg_dbg_size(self.h)

    @property
    def scratch_bytes(self):
        return lib().rg_scratch_bytes(self.h)

    def __del__(self):
        if getattr(self, "h", None) is not None and _lib is not None:
            _lib.rg_model_destroy(self.h)
            self.h = None


def world_shift_rows(t, v, name, m, origin):
    """Subtract the engine's world origin, in place, from the rows of a per-environment body_pos / geom_pos / site_pos
    tensor `v` ([nenv, 3 * count], any device) that live in world coordinates: bodies whose parent is the world, geoms
    and sites attached to the world body itself."""
    if name == "body_pos":
        sel = np.asarray(m["body_parentid"]) == 0
        sel[0] = False
    else:
        sel = np.asarray(m["geom_bodyid" if name == "geom_pos" else "site_bodyid"]) == 0
    idx = t.as_tensor(np.nonzero(sel)[0], dtype=t.long, device=v.device)
    if idx.numel():
        rows = v.view(v.shape[0], -1, 3)
        rows[:, idx] -= t.tensor(list(origin), dtype=v.dtype, device=v.device)
    return v


class BatchedSim:
    """nenv independent copies of one model, stepped by one fused kernel launch per env-step."""

    def __init__(self, model, nenv, n_substeps=10, outputs=("site_xpos", "act_force", "ncon", "warn"), debug=False,
                 contact_capacity=0, row_capacity=0, dofs_per_contact=0):
        """Capacities per environment (0 = engine default 32 / 64 / 16, see include/robogym_b200.h: rg_batch_create_ex); the
        reference's compiled sizes are nconmax=100 / njmax=500 (assets.xml:5-6)."""
        import torch

        if not torch.cuda.is_available():
            raise EngineError("BatchedSim needs a CUDA device (sm_90a, H100); there is no CPU fallback")
        self.torch = torch
        self.model = model
        self.nenv = int(nenv)
        self.n_substeps = int(n_substeps)
        self.device = torch.device("cuda", model.device)
        m = model.host
        f32 = dict(dtype=torch.float32, device=self.device)
        i32 = dict(dtype=torch.int32, device=self.device)
        n = self.nenv
        self.qpos = torch.tensor(m["qpos0"], **f32).repeat(n, 1).contiguous()
        self.qvel = torch.zeros(n, m["nv"], **f32)
        self.ctrl = torch.zeros(n, m["nu"], **f32)
        self.pid = torch.zeros(n, modelblob.pid_stride(m) * m["nu"], **f32)
        self.qacc_warmstart = torch.zeros(n, m["nv"], **f32)
        self.time = torch.zeros(n, **f32)
        h = ctypes.c_void_p()
        _check(lib().rg_batch_create_ex(model.h, n, int(contact_capacity), int(row_capacity), int(dofs_per_contact), ctypes.byref(h)))
        self.h = h
        c1, c2, c3 = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib().rg_batch_capacity(h, ctypes.byref(c1), ctypes.byref(c2), ctypes.byref(c3))
        self.contact_capacity, self.row_capacity, self.dofs_per_contact = c1.value, c2.value, c3.value
        self._bound = {}
        for fid, t in ((QPOS, self.qpos), (QVEL, self.qvel), (CTRL, self.ctrl), (PID, self.pid),
                       (WARMSTART, self.qacc_warmstart), (TIME, self.time)):
            self._bind(fid, t)
        shapes = dict(site_xpos=(SITE_XPOS, (n, m["nsite"], 3), f32), body_xpos=(BODY_XPOS, (n, m["nbody"], 3), f32),
                      body_xquat=(BODY_XQUAT, (n, m["nbody"], 4), f32), geom_xpos=(GEOM_XPOS, (n, m["ngeom"], 3), f32),
                      body_xvel=(BODY_XVEL, (n, m["nbody"], 6), f32), act_force=(ACT_FORCE, (n, m["nu"]), f32), qacc=(QACC, (n, m["nv"]), f32),
                      contact=(CONTACT, (n, self.contact_capacity, 4), f32), sensordata=(SENSORDATA, (n, m["nsensordata"]), f32), ncon=(NCON, (n,), i32), warn=(WARN, (n,), i32))
        for name in outputs:
            fid, shape, kw = shapes[name]
            t = torch.zeros(*shape, **kw)
            setattr(self, name, t)
            self._bind(fid, t)
        self.dbg = None
        if debug:
            self.dbg = torch.zeros(n, lib().rg_batch_dbg_size(self.h), **f32)
            self._bind(DBG, self.dbg)
        self.xfrc_applied = None
        self.timestep = None
        # data.mocap_pos / mocap_quat (world coordinates), one row per environment, initialised like mj_resetData does: the
        # model pose of the mocap bodies (robogym/robot/control/tcp/mocap_solver.py:41-46 then writes them every step)
        self.mocap_pos = self.mocap_quat = None
        if m["nmocap"]:
            ids = [b for b in range(m["nbody"]) if m["body_mocapid"][b] >= 0]
            ids.sort(key=lambda b: m["body_mocapid"][b])
            self.mocap_pos = torch.tensor(m["body_pos"].reshape(-1, 3)[ids], **f32).repeat(n, 1, 1).contiguous()
            self.mocap_quat = torch.tensor(m["body_quat"].reshape(-1, 4)[ids], **f32).repeat(n, 1, 1).contiguous()
            self._bind(MOCAP_POS, self.mocap_pos)
            self._bind(MOCAP_QUAT, self.mocap_quat)

    def _bind(self, fid, t):
        assert t.is_contiguous()
        self._bound[fid] = t  # keep alive
        _check(lib().rg_batch_bind(self.h, fid, ctypes.c_void_p(t.data_ptr())))

    def enable_xfrc(self):
        m = self.model.host
        self.xfrc_applied = self.torch.zeros(self.nenv, m["nbody"], 6, dtype=self.torch.float32, device=self.device)
        self._bind(XFRC, self.xfrc_applied)
        return self.xfrc_applied

    def set_param(self, name, values, idx=None):
        """Per-environment override of a float model array (domain randomisation): `values` is [nenv, count]
        (float64/float32 host array or tensor), or [len(idx), count] for the rows `idx` of an array that is already bound.
        The device copy is created on first use and updated in place; rows in world coordinates get the engine's fp32 world
        shift on EVERY write.  `geom_dataid` (per-environment mesh draws) is the one int array: it is kept as int32, and the
        pair lists of the rows written are marked stale, so the next step rederives them unless update_pairs() does first.
        Besides the blob's arrays: `mesh_scale` ([nmesh]) and `geom_mesh_scale` ([ngeom], a mesh geom's own scale on top of
        its hull's; finite and > 0, 1 while unbound), the engine's uniform hull scales."""
        t = self.torch
        m = self.model.host
        rows = self.nenv if idx is None else len(idx)
        if name == "geom_dataid":
            v = t.as_tensor(np.asarray(values) if not t.is_tensor(values) else values).to(t.int64).reshape(rows, -1)
            if v.shape[1] != m["ngeom"]:
                raise EngineError(f"set_param(geom_dataid): expected {m['ngeom']} values per environment, got {v.shape[1]}")
            check_geom_dataid(v, m)
            out = self._store_param(name, v.to(device=self.device, dtype=t.int32).contiguous(), idx)
            mp = None
            if idx is not None:
                mk = t.zeros(self.nenv, dtype=t.uint8, device=self.device)
                mk[t.as_tensor(idx, device=self.device).long()] = 1
                self._keep_stale = mk            # alive until the launch has consumed it
                mp = ctypes.c_void_p(mk.data_ptr())
            _check(lib().rg_batch_mark_pairs_stale(self.h, mp, self._stream()))
            return out
        v = t.as_tensor(np.asarray(values, dtype=np.float64) if not t.is_tensor(values) else values).to(t.float64).reshape(rows, -1).clone()
        # mesh_scale / geom_mesh_scale: the engine's per-hull / per-mesh-geom scales, not blob arrays
        count = {"mesh_scale": m["nmesh"], "geom_mesh_scale": m["ngeom"]}[name] if name in ("mesh_scale", "geom_mesh_scale") else m[name].size
        if v.shape[1] != count:
            raise EngineError(f"set_param({name}): expected {count} values per environment, got {v.shape[1]}")
        if name in ("mesh_scale", "geom_mesh_scale"):
            check_mesh_scale(v, name)
        if name in ("body_pos", "geom_pos", "site_pos"):
            # keep the engine's fp32 world shift: bodies attached to the world, and geoms / sites attached to the world body
            o = (ctypes.c_float * 3)()
            _check(lib().rg_model_origin(self.model.h, o))
            world_shift_rows(t, v, name, m, list(o))
        return self._store_param(name, v.to(device=self.device, dtype=t.float32).contiguous(), idx)

    def _store_param(self, name, dev, idx):
        if idx is not None and name not in getattr(self, "_params", {}):
            raise EngineError(f"set_param({name}, idx=...): bind the full array first")
        if not hasattr(self, "_params"):
            self._params = {}
        if idx is not None:
            self._params[name][idx] = dev
        elif name in self._params:
            self._params[name].copy_(dev)
        else:
            self._params[name] = dev
            _check(lib().rg_batch_bind_param(self.h, name.encode(), ctypes.c_void_p(dev.data_ptr())))
        return self._params[name]

    def update_pairs(self, mask=None):
        """Rederive the per-environment pair lists from the bound geom_dataid rows (all environments, or those of `mask`):
        each keeps the static candidate pairs whose two geoms are enabled in its row (include/robogym_b200.h)."""
        mp = None
        if mask is not None:
            mask = mask.to(device=self.device, dtype=self.torch.uint8).contiguous()
            mp = ctypes.c_void_p(mask.data_ptr())
            self._keep_mask = mask
        _check(lib().rg_batch_update_pairs(self.h, mp, self._stream()))

    def set_pair_capacity(self, capacity):
        """Pairs each environment's list can hold (0: npair); the lists are derived again before the next step."""
        _check(lib().rg_batch_set_pair_capacity(self.h, int(capacity)))

    def pair_counts(self):
        """Length of every environment's pair list ([nenv] int32 device tensor, a copy), or None when the batch streams the
        static list."""
        cap, ptr = ctypes.c_int(), ctypes.c_void_p()
        _check(lib().rg_batch_pair_info(self.h, ctypes.byref(cap), ctypes.byref(ptr)))
        if not ptr.value:
            return None
        view = type("EngineInts", (), {"__cuda_array_interface__": dict(shape=(self.nenv,), typestr="<i4", data=(ptr.value, False), version=2)})()
        return self.torch.as_tensor(view, device=self.device).clone()

    def enable_per_env_timestep(self):
        self.timestep = self.torch.full((self.nenv,), float(self.model.host["opt_timestep"][0]), dtype=self.torch.float32, device=self.device)
        self._bind(TIMESTEP, self.timestep)
        return self.timestep

    def _stream(self):
        return ctypes.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def step(self, n_substeps=None, final_forward=True, mask=None):
        """SimulationInterface.step(): nsubsteps x mj_step then mj_forward, for every environment (or, with `mask`
        -- a [nenv] bool/uint8 device tensor -- only for the selected ones; the launch then covers just those).
        final_forward may be an integer > 1 to fuse the extra sim.forward() calls of the reference's observation path."""
        nsub = self.n_substeps if n_substeps is None else int(n_substeps)
        if mask is None:
            _check(lib().rg_step(self.h, nsub, int(final_forward), self._stream()))
        else:
            mk = mask.to(device=self.device, dtype=self.torch.uint8).contiguous()
            _check(lib().rg_step_subset(self.h, ctypes.c_void_p(mk.data_ptr()), nsub, int(final_forward), self._stream()))
            self._keep_mask = mk   # alive until the launch has consumed it

    def forward(self, mask=None, count=1):
        if mask is None and count == 1:
            _check(lib().rg_forward(self.h, self._stream()))
        else:
            self.step(0, count, mask)

    def reset(self, mask=None):
        mp = None
        if mask is not None:
            mask = mask.to(device=self.device, dtype=self.torch.uint8).contiguous()
            mp = ctypes.c_void_p(mask.data_ptr())
        _check(lib().rg_reset(self.h, mp, self._stream()))

    SET_CONST_FIELDS = ("dof_invweight0", "body_invweight0", "tendon_invweight0", "tendon_length0", "body_subtreemass", "opt_meaninertia")

    def set_const(self, mask=None, fields=("dof_invweight0", "body_invweight0", "tendon_invweight0", "opt_meaninertia")):
        """SimulationInterface.set_constants() for every (or the masked) environment: mj_setConst from each environment's own
        parameters (set_param), on the device, written into per-environment rows of `fields` (bound here on first use with the
        model's values).  Returns the dict of those tensors."""
        m = self.model.host
        for name in fields:
            if name not in self.SET_CONST_FIELDS:
                raise EngineError(f"set_const: {name} is not a constant mj_setConst derives")
            if name not in getattr(self, "_params", {}) and m[name].size:
                self.set_param(name, np.repeat(np.asarray(m[name], dtype=np.float64).reshape(1, -1), self.nenv, axis=0))
        mp = None
        if mask is not None:
            mask = mask.to(device=self.device, dtype=self.torch.uint8).contiguous()
            mp = ctypes.c_void_p(mask.data_ptr())
            self._keep_mask = mask
        _check(lib().rg_set_const(self.h, mp, self._stream()))
        return {k: self._params[k] for k in fields if k in self._params}

    def set_balance(self, on):
        """Work-ordered scheduling on/off (include/robogym_b200.h: rg_batch_set_balance); results do not depend on it."""
        _check(lib().rg_batch_set_balance(self.h, int(bool(on))))

    def launch_info(self):
        a, b, c = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib().rg_batch_launch_info(self.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
        return dict(ctas=a.value, warps_per_cta=b.value, smem_bytes=c.value, scratch_bytes_per_env=lib().rg_batch_scratch_bytes(self.h),
                    contact_capacity=self.contact_capacity, row_capacity=self.row_capacity, dofs_per_contact=self.dofs_per_contact)

    def dbg_view(self, env=0):
        """Decode the stage dump of one environment (tests)."""
        m = self.model.host
        nv, nt, nu = m["nv"], m["ntendon"], m["nu"]
        g = self.dbg[env].cpu().numpy()
        o = 0
        out = {}
        out["M"] = g[o:o + nv * nv].reshape(nv, nv); o += nv * nv
        for k in ("bias", "passive", "qfa", "smooth", "qacc", "qfc"):
            out[k] = g[o:o + nv]; o += nv
        out["tlen"] = g[o:o + nt]; o += nt
        out["alen"] = g[o:o + nu]; o += nu
        out["aforce"] = g[o:o + nu]; o += nu
        out["ncon"], out["nel"], out["niter"], out["warn"] = [int(x) for x in g[o:o + 4]]; o += 4
        K = self.contact_capacity
        out["con"] = g[o:o + K * CON_STRIDE].reshape(K, CON_STRIDE); o += K * CON_STRIDE
        out["tJ"] = g[o:o + nt * nv].reshape(nt, nv)
        return out

    def __del__(self):
        if getattr(self, "h", None) is not None and _lib is not None:
            _lib.rg_batch_destroy(self.h)
            self.h = None
