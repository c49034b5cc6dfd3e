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

_vp, _ci, _cd, _u32, _str, _P = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_uint32, ctypes.c_char_p, ctypes.POINTER


class GoalIn(ctypes.Structure):
    """rg_goal_in (include/robogym_b200.h)"""
    _fields_ = [("nenv", _ci), ("nobj", _ci), ("pos", _vp), ("quat", _vp), ("pos_stride", ctypes.c_longlong), ("quat_stride", ctypes.c_longlong),
                ("rows", _vp), ("goal_pos", _vp), ("goal_quat", _vp), ("group", _vp), ("pos_offset", _vp), ("rot_weight", _vp), ("table", _cd * 6),
                ("rot_dist_type", _ci), ("success_keys", _ci), ("pos_threshold", _cd), ("rot_threshold", _cd), ("reward_per_object", _cd),
                ("gripper_pos", _vp), ("gripper_stride", ctypes.c_longlong), ("grasped", _vp), ("gripper_threshold", _cd), ("grasped_threshold", _cd)]


class GoalOut(ctypes.Structure):
    """rg_goal_out (include/robogym_b200.h)"""
    _fields_ = [("obj_rot", _vp), ("rel_pos", _vp), ("rel_rot", _vp), ("dist_pos", _vp), ("dist_rot", _vp), ("success", _vp), ("off_table", _vp),
                ("num_success", _vp), ("reward", _vp), ("achieved", _vp), ("any_off", _vp), ("pick", _vp), ("rel_gripper", _vp), ("dist_gripper", _vp)]


class ObsIn(ctypes.Structure):
    """rg_obs_in (include/robogym_b200.h)"""
    _fields_ = [("nenv", _ci), ("nobj", _ci), ("body_xpos", _vp), ("body_xquat", _vp), ("body_xvel", _vp), ("qpos", _vp), ("qvel", _vp),
                ("ctrl", _vp), ("sensordata", _vp), ("contact", _vp), ("ncon", _vp), ("nbody", _ci), ("nq", _ci), ("nv", _ci), ("nu", _ci),
                ("nsensordata", _ci), ("ncontact", _ci), ("ngeom", _ci), ("obj_body", _vp), ("obj_qpos", _vp), ("tcp_body", _ci),
                ("narm", _ci), ("arm_qpos", _ci * 8), ("ngrip", _ci), ("grip_qpos", _ci * 4), ("grip_qvel", _ci * 4), ("grip_act", _ci),
                ("force_adr", _ci), ("torque_adr", _ci), ("geom_object", _vp), ("geom_flags", _vp), ("table_plane", _ci), ("wrist_sphere", _ci),
                ("pad", _ci * 2), ("goal_pos", _vp), ("goal_quat", _vp), ("rel_pos", _vp), ("rel_rot", _vp), ("achieved", _vp), ("off_table", _vp),
                ("group", _vp), ("qpos_at_goal", _vp), ("bbox_size", _vp), ("colors", _vp), ("boundary", _vp), ("penalty", _cd * 4),
                ("mask_obs", _ci), ("mask_margin", _cd)]


class ObsOut(ctypes.Structure):
    """rg_obs_out (include/robogym_b200.h): one output pointer per observation key"""
    _fields_ = [(k, _vp) for k in (
        "obj_pos obj_rel_pos obj_vel_pos obj_rot obj_vel_rot robot_joint_pos gripper_pos gripper_velp gripper_controls gripper_qpos "
        "gripper_vel qpos qpos_goal goal_obj_pos goal_obj_rot rel_goal_obj_pos rel_goal_obj_rot is_goal_achieved obj_gripper_contact "
        "obj_bbox_size obj_colors safety_stop tcp_force tcp_torque placement_mask goal_placement_mask masked_obj_pos masked_obj_rot "
        "masked_obj_rel_pos masked_obj_vel_pos masked_obj_vel_rot masked_obj_gripper_contact masked_obj_bbox_size masked_obj_colors "
        "masked_goal_obj_pos masked_goal_obj_rot masked_rel_goal_obj_pos masked_rel_goal_obj_rot gripper_table_contact wrist_cam_contacts "
        "sim_reward sim_done").split()]


class ArmTables(ctypes.Structure):
    """rg_arm_tables (include/robogym_b200.h)"""
    _fields_ = [("narm", _ci), ("arm_qpos_main", _ci * 8), ("arm_qpos_solver", _ci * 8), ("arm_act_main", _ci * 8), ("grip_qpos_main", _ci),
                ("grip_qpos_solver", _ci), ("grip_act_main", _ci), ("grip_act_solver", _ci), ("tcp_body", _ci), ("nweld", _ci), ("weld_mocap", _ci * 4),
                ("weld_body", _ci * 4), ("ndof", _ci), ("euler_index", _ci * 3), ("dof_joint", _ci * 3), ("align_axis", _ci), ("speed", _cd * 3),
                ("lo_lim", _cd * 8), ("hi_lim", _cd * 8), ("max_position_change", _cd), ("grip_lo", _cd), ("grip_hi", _cd), ("grip_half", _cd)]


class ArmSim(ctypes.Structure):
    """rg_arm_sim (include/robogym_b200.h)"""
    _fields_ = [("nq", _ci), ("nu", _ci), ("nbody", _ci), ("nmocap", _ci), ("qpos", _vp), ("ctrl", _vp), ("body_xpos", _vp), ("body_xquat", _vp),
                ("mocap_pos", _vp), ("mocap_quat", _vp)]


# rg_arm_phase phase bits
ARM_SYNC, ARM_GRIP, ARM_SEAT, ARM_PRESOLVE, ARM_POSTSOLVE = 1, 2, 4, 8, 16


class GroupsIn(ctypes.Structure):
    """rg_groups_in (include/robogym_b200.h)"""
    _fields_ = [("nenv", _ci), ("nobj", _ci), ("active", _vp), ("group_mode", _ci), ("lam_low", _cd), ("lam_high", _cd), ("fixed_counts", _vp),
                ("n_materials", _ci), ("color_mode", _ci), ("palette", _vp), ("n_palette", _ci), ("scale_low", _cd), ("scale_high", _cd),
                ("mesh_mode", _ci), ("n_candidates", _ci), ("seed", _u32), ("epoch", _u32)]


class GroupsOut(ctypes.Structure):
    """rg_groups_out (include/robogym_b200.h)"""
    _fields_ = [(k, _vp) for k in "group count material rgba scale mesh yaw quat ngroups".split()]


# name -> (restype, argtypes) of every function include/robogym_b200.h declares, in its order (tests/test_abi.py checks the
# table against the header)
SIGNATURES = {
    "rg_model_load": (_ci, [_vp, ctypes.c_size_t, _ci, _P(_vp)]),
    "rg_model_destroy": (None, [_vp]),
    "rg_model_dim": (_ci, [_vp, _str]),
    "rg_model_name2id": (_ci, [_vp, _str, _str]),
    "rg_model_id2name": (_str, [_vp, _str, _ci]),
    "rg_model_set_field": (_ci, [_vp, _str, _vp, ctypes.c_size_t]),
    "rg_model_set_field_async": (_ci, [_vp, _str, _vp, ctypes.c_size_t, _vp]),
    "rg_dbg_size": (_ci, [_vp]),
    "rg_scratch_bytes": (_ci, [_vp]),
    "rg_batch_create": (_ci, [_vp, _ci, _P(_vp)]),
    "rg_batch_create_ex": (_ci, [_vp, _ci, _ci, _ci, _ci, _P(_vp)]),
    "rg_batch_capacity": (_ci, [_vp, _P(_ci), _P(_ci), _P(_ci)]),
    "rg_batch_dbg_size": (_ci, [_vp]),
    "rg_batch_scratch_bytes": (_ci, [_vp]),
    "rg_batch_destroy": (None, [_vp]),
    "rg_batch_bind": (_ci, [_vp, _ci, _vp]),
    "rg_batch_bind_param": (_ci, [_vp, _str, _vp]),
    "rg_batch_update_pairs": (_ci, [_vp, _vp, _vp]),
    "rg_batch_mark_pairs_stale": (_ci, [_vp, _vp, _vp]),
    "rg_batch_set_pair_capacity": (_ci, [_vp, _ci]),
    "rg_batch_pair_info": (_ci, [_vp, _P(_ci), _P(_vp)]),
    "rg_model_origin": (_ci, [_vp, _P(ctypes.c_float)]),
    "rg_batch_set_balance": (_ci, [_vp, _ci]),
    "rg_batch_launch_info": (_ci, [_vp, _P(_ci), _P(_ci), _P(_ci)]),
    "rg_batch_env_warps": (_ci, [_vp, _P(_ci)]),
    "rg_step": (_ci, [_vp, _ci, _ci, _vp]),
    "rg_forward": (_ci, [_vp, _vp]),
    "rg_step_subset": (_ci, [_vp, _vp, _ci, _ci, _vp]),
    "rg_step_settle": (_ci, [_vp, _vp, _vp, _ci, _cd, _ci, _ci, _vp]),
    "rg_set_const": (_ci, [_vp, _vp, _vp]),
    "rg_reset": (_ci, [_vp, _vp, _vp]),
    "rg_batch_body_aabb": (_ci, [_vp, _vp, _ci, _vp, _vp, _vp, _vp]),
    "rg_place_objects": (_ci, [_ci, _ci, _vp, _vp, _vp, _vp, _ci, _ci, _ci, _cd, _cd, _vp, _u32, _u32, _vp, _vp, _vp, _vp]),
    "rg_goal_modify": (_ci, [_ci, _ci, _ci, _vp, _vp, _vp, _vp, _cd, _cd, _cd, _cd, _ci, _u32, _u32, _vp, _vp, _vp]),
    "rg_layout_goals": (_ci, [_ci, _ci, _ci, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _ci, _u32, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "rg_rearrange_goal": (_ci, [_P(GoalIn), _vp, _vp, _P(GoalOut), _vp]),
    "rg_goal_orientations": (_ci, [_ci, _ci, _vp, _vp, _ci, _u32, _u32, _vp, _vp, _vp]),
    "rg_rearrange_obs": (_ci, [_P(ObsIn), _vp, _P(ObsOut), _vp]),
    "rg_arm_phase": (_ci, [_P(ArmTables), _ci, _ci, _P(ArmSim), _P(ArmSim), _vp, _ci, _vp, _ci, _vp]),
    "rg_arm_sample_actions": (_ci, [_ci, _ci, _u32, _u32, _vp, _ci, _vp, _vp]),
    "rg_object_groups": (_ci, [_P(GroupsIn), _vp, _ci, _P(GroupsOut), _vp]),
    "rg_last_error": (_str, []),
}

_lib = None


class EngineError(RuntimeError):
    pass


def lib():
    """Load librobogym_b200.so (built in-tree by `python -m robogym_b200.build`) with the signatures of SIGNATURES."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise EngineError(
                f"{LIB_PATH} is missing: build it with `python -m robogym_b200.build` "
                "(nvcc, sm_90a). There is no CPU fallback."
            )
        L = ctypes.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SIGNATURES.items():
            f = getattr(L, name)
            f.restype, f.argtypes = restype, argtypes
        _lib = L
    return _lib


def _check(rc):
    if rc != 0:
        raise EngineError(lib().rg_last_error().decode())


def ptr(x):
    """The data pointer of a tensor as a pointer argument; None (NULL) for None."""
    return None if x is None else ctypes.c_void_p(x.data_ptr())


def current_stream(t, device):
    """torch's current stream on `device` as the stream argument (cudaStream_t) of a launch."""
    return ctypes.c_void_p(t.cuda.current_stream(device).cuda_stream)


def as_device(t, x, dtype, shape, name, device):
    """`x` (a tensor or anything numpy takes) broadcast to `shape` as a contiguous `dtype` tensor on `device`; ValueError
    naming `name` when it does not broadcast."""
    x = x if t.is_tensor(x) else t.as_tensor(np.asarray(x))
    if tuple(x.shape) != tuple(shape):
        try:
            x = x.expand(*shape)
        except RuntimeError:
            raise ValueError(f"{name}: expected shape {tuple(shape)}, got {tuple(x.shape)}") from None
    return x.to(device=device, dtype=dtype).contiguous()


def device_mask(t, mask, nenv, device):
    """A [nenv] environment mask (bool or uint8, tensor or array; None: every environment) as the contiguous uint8 tensor on
    `device` that the launches read, or None.

    Lifetime: the result, like every other temporary as_device makes for a launch, may be dropped as soon as the launch is
    enqueued, with no synchronisation.  It is allocated on torch's current stream of `device`, the stream the launch is
    enqueued on, and the caching allocator gives its memory only to later work on that stream, which runs after the launch."""
    return None if mask is None else as_device(t, mask, t.uint8, (nenv,), "mask", device)


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
            stream = current_stream(t, self.device) if t is not None and t.cuda.is_available() else None
        _check(lib().rg_model_set_field_async(self.h, name.encode(), buf.ctypes.data, buf.size, stream))

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
        _check(lib().rg_batch_bind(self.h, fid, ptr(t)))

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
            mask = None
            if idx is not None:
                mask = t.zeros(self.nenv, dtype=t.uint8, device=self.device)
                mask[t.as_tensor(idx, device=self.device).long()] = 1
            _check(lib().rg_batch_mark_pairs_stale(self.h, ptr(mask), current_stream(t, self.device)))
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
            _check(lib().rg_batch_bind_param(self.h, name.encode(), ptr(dev)))
        return self._params[name]

    def update_pairs(self, mask=None):
        """Rederive the per-environment pair lists from the bound geom_dataid rows (all environments, or those of `mask`):
        each keeps the static candidate pairs whose two geoms are enabled in its row (include/robogym_b200.h)."""
        mask = device_mask(self.torch, mask, self.nenv, self.device)
        _check(lib().rg_batch_update_pairs(self.h, ptr(mask), current_stream(self.torch, self.device)))

    def set_pair_capacity(self, capacity):
        """Pairs each environment's list can hold (0: npair); the lists are derived again before the next step."""
        _check(lib().rg_batch_set_pair_capacity(self.h, int(capacity)))

    def pair_counts(self):
        """Length of every environment's pair list ([nenv] int32 device tensor, a copy), or None when the batch streams the
        static list."""
        cap, counts = ctypes.c_int(), ctypes.c_void_p()
        _check(lib().rg_batch_pair_info(self.h, ctypes.byref(cap), ctypes.byref(counts)))
        if not counts.value:
            return None
        view = type("EngineInts", (), {"__cuda_array_interface__": dict(shape=(self.nenv,), typestr="<i4", data=(counts.value, False), version=2)})()
        return self.torch.as_tensor(view, device=self.device).clone()

    def enable_per_env_timestep(self):
        self.timestep = self.torch.full((self.nenv,), float(self.model.host["opt_timestep"][0]), dtype=self.torch.float32, device=self.device)
        self._bind(TIMESTEP, self.timestep)
        return self.timestep

    def step(self, n_substeps=None, final_forward=True, mask=None):
        """SimulationInterface.step(): nsubsteps x mj_step then mj_forward, for every environment (or, with `mask`
        -- a [nenv] bool/uint8 device tensor -- only for the selected ones; the launch then covers just those).
        final_forward may be an integer > 1 to fuse the extra sim.forward() calls of the reference's observation path."""
        nsub = self.n_substeps if n_substeps is None else int(n_substeps)
        stream = current_stream(self.torch, self.device)
        if mask is None:
            _check(lib().rg_step(self.h, nsub, int(final_forward), stream))
        else:
            mask = device_mask(self.torch, mask, self.nenv, self.device)
            _check(lib().rg_step_subset(self.h, ptr(mask), nsub, int(final_forward), stream))

    def settle(self, dofs, damping, n_substeps, mask=None, final_forward=True):
        """`n_substeps` x mj_step with dof_damping = `damping` on the dof ids `dofs` (1 to 64 of them), then `final_forward`
        x mj_forward with each environment's own damping: the reference's stabilize_objects step loop
        (robogym/envs/rearrange/common/utils.py:76-93) in one launch for every environment, or with `mask` for the selected
        ones only (the launch covers just those).  The damping is a launch constant: no per-environment dof_damping row is
        bound, and neither the model nor a bound row changes (include/robogym_b200.h: rg_step_settle)."""
        d = np.ascontiguousarray(np.asarray(dofs, dtype=np.int64).ravel())
        if d.size and (d.min() < np.iinfo(np.int32).min or d.max() > np.iinfo(np.int32).max):
            raise EngineError("settle: dof id out of range")
        d = d.astype(np.int32)
        stream = current_stream(self.torch, self.device)
        mask = device_mask(self.torch, mask, self.nenv, self.device)
        _check(lib().rg_step_settle(self.h, ptr(mask), d.ctypes.data, int(d.size), float(damping), int(n_substeps), int(final_forward), stream))

    def forward(self, mask=None, count=1):
        if mask is None and count == 1:
            _check(lib().rg_forward(self.h, current_stream(self.torch, self.device)))
        else:
            self.step(0, count, mask)

    def reset(self, mask=None):
        mask = device_mask(self.torch, mask, self.nenv, self.device)
        _check(lib().rg_reset(self.h, ptr(mask), current_stream(self.torch, self.device)))

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
        mask = device_mask(self.torch, mask, self.nenv, self.device)
        _check(lib().rg_set_const(self.h, ptr(mask), current_stream(self.torch, self.device)))
        return {k: self._params[k] for k in fields if k in self._params}

    def set_balance(self, on):
        """Work-ordered scheduling on/off (include/robogym_b200.h: rg_batch_set_balance); results do not depend on it."""
        _check(lib().rg_batch_set_balance(self.h, int(bool(on))))

    def launch_info(self):
        a, b, c, w = ctypes.c_int(), ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        lib().rg_batch_launch_info(self.h, ctypes.byref(a), ctypes.byref(b), ctypes.byref(c))
        _check(lib().rg_batch_env_warps(self.h, ctypes.byref(w)))
        return dict(ctas=a.value, warps_per_cta=b.value, warps_per_env=w.value, smem_bytes=c.value, scratch_bytes_per_env=lib().rg_batch_scratch_bytes(self.h),
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
