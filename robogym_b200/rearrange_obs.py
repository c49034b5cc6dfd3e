"""What the policy of a rearrange batch observes, and the simulation part of its reward and `done`, on the device, every env-step.

The reference assembles these per environment in numpy: `RearrangeEnv._observe_simple` (robogym/envs/rearrange/common/base.py:
376-421) from the simulation's getters (envs/rearrange/simulation/base.py:420-647, padded to max_num_objects as
`_get_object_obs_with_prefix` pads, :1015-1024) and the robot's `MujocoObservation` (robot/ur16e/mujoco/joint_controlled_arm.py:
22-85); the placement-area masks of `_mask_goal_observation` / `_mask_object_observation` (common/base.py:311-374) with the
hard rule of `check_objects_in_placement_area` (simulation/base.py:847-902); and the penalties of
`_get_simulation_reward_with_done` (common/base.py:768-795) from the contact queries `get_gripper_table_contact` /
`get_wrist_cam_collisions`.  Here one launch does all of it, one warp per environment (`rg_rearrange_obs`,
robogym_b200/csrc/rg_obs.inl), reading the sim's rows in place and the outputs of `BatchedRearrangeGoal.evaluate()` of the
same env-step.

    goal = BatchedRearrangeGoal(sim, scene.bodies, groups, table)
    obs_fn = BatchedRearrangeObservation(sim, goal, scene.bodies, bbox_size=scene.bounding_boxes(identity)[..., 1, :],
                                         colors=colors, placement_area_boundary=placement_area_boundary(table, area))
    goal.set_goal(goal_pos, goal_quat); obs_fn.set_goal_qpos()     # per goal reset
    sim.step(); goal.evaluate()
    obs, info = obs_fn.observe()                                   # per env-step, after goal.evaluate() on the same stream

`soft_mask` is not provided: the reference draws it from the global `np.random` (simulation/base.py:887-889).
"""
import ctypes

import numpy as np

from . import engine, modelblob
from .engine import ObsIn, ObsOut, as_device, current_stream, device_mask, ptr
from .rearrange_contacts import GRIPPER_BODIES
from .rearrange_goal import MAX_OBJECTS

# envs/rearrange/simulation/base.py:110-112; safety_stop has no default (penalty.get("safety_stop", 0.0))
PENALTY = {"table_collision": 0.0, "wrist_collision": 0.0, "objects_off_table": 1.0, "safety_stop": 0.0}
GEOM_GRIPPER, GEOM_ROBOT = 1, 2
WRIST_KEYS = ("table_collision_plane", "robot", "object", "any")
OBJECT_KEYS = ("obj_pos", "obj_rot", "obj_rel_pos", "obj_vel_pos", "obj_vel_rot", "obj_gripper_contact", "obj_bbox_size", "obj_colors")
GOAL_KEYS = ("goal_obj_pos", "goal_obj_rot", "rel_goal_obj_pos", "rel_goal_obj_rot")
OUT_FIELDS = tuple(k for k, _ in ObsOut._fields_)


def placement_area_boundary(table, area):
    """`extract_placement_area_boundary` (simulation/base.py:834-845) per environment: table = rearrange_placement.
    table_dimensions(model), area = rearrange_placement.placement_area(...) [nenv, 6] (offset, size).  Returns [nenv, 6] float64
    (min x y z, max x y z)."""
    table_pos, table_size = np.asarray(table[0], dtype=np.float64), np.asarray(table[1], dtype=np.float64)
    area = np.asarray(area, dtype=np.float64).reshape(-1, 6)
    out = np.empty((area.shape[0], 6))
    for e in range(area.shape[0]):
        size = np.array(area[e, 3:]) / 2
        pos = np.array(area[e, :3]) + table_pos - table_size + size
        out[e, :3], out[e, 3:] = pos - size, pos + size
    return out


def _penalty(penalty):
    p = dict(PENALTY)
    if penalty is not None:
        bad = set(penalty) - set(PENALTY)
        if bad:
            raise ValueError(f"penalty: keys among {sorted(PENALTY)}, not {sorted(bad)}")
        p.update({k: float(v) for k, v in penalty.items()})
    if not all(np.isfinite(v) for v in p.values()):
        raise ValueError("penalty: finite weights")
    return [p["table_collision"], p["wrist_collision"], p["objects_off_table"], p["safety_stop"]]


def index_tables(m, names, object_bodies, prefix="robot0:"):
    """The index tables of rg_rearrange_obs from a model's arrays `m` and name tables `names` (modelblob.unpack /
    unpack_names): each slot's free-joint qpos address (`object<k>:joint` of the body object<k>), the tool body, the arm joints
    (`<prefix>J*`) and the gripper joints (`<prefix>r_gripper_RJ0_outer*`) as register_joint_group collects them, the gripper
    actuator, the force / torque sensor addresses, the geom -> slot table, the gripper / robot geom flags and the four geoms
    of the contact queries."""
    def find(kind, name):
        try:
            return names[kind].index(name)
        except ValueError:
            raise ValueError(f"the model has no {kind} {name!r}") from None

    jnt = [n or "" for n in names["joint"]]
    arm = [j for j, n in enumerate(jnt) if n.startswith(prefix + "J")]
    grip = [j for j, n in enumerate(jnt) if n.startswith(prefix + "r_gripper_RJ0_outer")]
    if not 1 <= len(arm) <= 8 or not 1 <= len(grip) <= 4:
        raise ValueError(f"the model needs 1 to 8 arm joints {prefix}J* and 1 to 4 gripper joints {prefix}r_gripper_RJ0_outer*")
    qadr, dadr, sadr = np.asarray(m["jnt_qposadr"]), np.asarray(m["jnt_dofadr"]), np.asarray(m["sensor_adr"])
    ng = int(m["ngeom"])
    geom_body = np.asarray(m["geom_bodyid"])
    geom_names = [n or "" for n in names["geom"]]
    gb = {find("body", b) for b in GRIPPER_BODIES}
    flags = [(GEOM_GRIPPER if int(geom_body[g]) in gb else 0) | (GEOM_ROBOT if geom_names[g].startswith(prefix) else 0) for g in range(ng)]
    gobj = np.full(ng, -1, dtype=np.int64)
    for k, b in enumerate(object_bodies):
        gobj[geom_body == int(b)] = k
    return dict(obj_qpos=[int(qadr[find("joint", names["body"][int(b)] + ":joint")]) for b in object_bodies], tcp_body=find("body", prefix + "gripper_tcp"),
                arm_qpos=[int(qadr[j]) for j in arm], grip_qpos=[int(qadr[j]) for j in grip], grip_qvel=[int(dadr[j]) for j in grip],
                grip_act=find("actuator", prefix + "r_gripper_finger_joint"), force_adr=int(sadr[find("sensor", "toolhead_force")]),
                torque_adr=int(sadr[find("sensor", "toolhead_torque")]), geom_object=gobj.tolist(), geom_flags=flags,
                table_plane=find("geom", "table_collision_plane"), wrist_sphere=find("geom", prefix + "wrist_cam_collision_sphere"),
                pad=[find("geom", prefix + "left_contact_v"), find("geom", prefix + "right_contact_v")])


class BatchedRearrangeObservation:
    """The observation dict and the simulation reward / done of every environment of a rearrange batch.

    sim: a BatchedSim with the outputs body_xpos, body_xquat, body_xvel, contact, ncon and sensordata; goal: the batch's
    BatchedRearrangeGoal (its goals, groups and evaluate() outputs are read); object_bodies: the body id of each object slot
    (BatchedBlockScene.bodies / BatchedMeshScene.bodies, the same as the goal's), each named object<k> with a free joint
    object<k>:joint.  Per reset: bbox_size [nenv, nobj, 3] (bounding_boxes(identity)[..., 1, :], `_get_bounding_box(n)[1]`),
    colors [nenv, nobj, 4] (rgba), placement_area_boundary [nenv, 6] (placement_area_boundary()).  penalty: weights of
    table_collision, wrist_collision, objects_off_table, safety_stop (the reference's defaults otherwise);
    mask_obs_outside_placement_area / mask_margin as the reference's constants; soft_mask is refused.

    Differences from the reference: goal_placement_mask is recomputed every call from the goals and the current boundary (the
    reference keeps goal_objects_in_placement_area from goal time; the same while neither changes between goal resets);
    qpos / qpos_goal are the model's full rows, parked slots included; the wrist-collision penalty always applies (the
    reference's default camera set, with vision_cam_wrist)."""

    def __init__(self, sim, goal, object_bodies, *, bbox_size, colors, placement_area_boundary, penalty=None, mask_obs_outside_placement_area=False,
                 mask_margin=0.02, soft_mask=False, prefix="robot0:"):
        t = sim.torch
        if soft_mask:
            raise ValueError("soft_mask is not provided: the reference draws it from the global np.random (simulation/base.py:887-889), "
                             "which cannot be reproduced")
        for k in ("body_xpos", "body_xquat", "body_xvel", "contact", "ncon", "sensordata"):
            if getattr(sim, k, None) is None:
                raise ValueError(f"the sim needs the outputs body_xpos, body_xquat, body_xvel, contact, ncon and sensordata (missing {k})")
        bodies = np.asarray(object_bodies, dtype=np.int64).reshape(-1)
        m, model = sim.model.host, sim.model
        nbody, nq, ng = int(m["nbody"]), int(m["nq"]), int(m["ngeom"])
        if not 1 <= len(bodies) <= MAX_OBJECTS or (bodies < 0).any() or (bodies >= nbody).any():
            raise ValueError(f"object_bodies: 1 to {MAX_OBJECTS} body ids in [0, {nbody})")
        if goal.sim is not sim or goal.nobj != len(bodies) or not np.array_equal(goal._e.rows, bodies):
            raise ValueError("goal: the BatchedRearrangeGoal of this sim over the same object bodies")
        self.sim, self.goal, self.t, self.nenv, self.nobj = sim, goal, t, sim.nenv, len(bodies)
        self.mask_obs = bool(mask_obs_outside_placement_area)
        if not np.isfinite(float(mask_margin)):
            raise ValueError("mask_margin: finite")
        dev, nenv, nobj = sim.device, sim.nenv, len(bodies)

        T = index_tables(m, modelblob.unpack_names(model.blob), bodies, prefix)
        self.obj_body = np.ascontiguousarray(bodies, dtype=np.int32)
        self.obj_qpos = np.ascontiguousarray(T["obj_qpos"], dtype=np.int32)
        self.geom_flags = t.as_tensor(np.asarray(T["geom_flags"], dtype=np.uint8), device=dev)
        self.geom_object = t.as_tensor(np.asarray(T["geom_object"], dtype=np.int32), device=dev)

        f64 = dict(dtype=t.float64, device=dev)
        self.bbox_size = t.zeros(nenv, nobj, 3, **f64)
        self.colors = t.zeros(nenv, nobj, 4, **f64)
        self.boundary = t.zeros(nenv, 6, **f64)
        self.qpos_at_goal = sim.qpos.clone()
        self.set_reset_rows(bbox_size, colors, placement_area_boundary)

        c = self.cin = ObsIn()
        c.nenv, c.nobj = nenv, nobj
        c.body_xpos, c.body_xquat, c.body_xvel = ptr(sim.body_xpos), ptr(sim.body_xquat), ptr(sim.body_xvel)
        c.qpos, c.qvel, c.ctrl, c.sensordata = ptr(sim.qpos), ptr(sim.qvel), ptr(sim.ctrl), ptr(sim.sensordata)
        c.contact, c.ncon = ptr(sim.contact), ptr(sim.ncon)
        c.nbody, c.nq, c.nv, c.nu, c.nsensordata, c.ncontact, c.ngeom = nbody, nq, int(m["nv"]), int(m["nu"]), int(m["nsensordata"]), int(sim.contact.shape[1]), ng
        c.obj_body, c.obj_qpos = self.obj_body.ctypes.data, self.obj_qpos.ctypes.data
        c.tcp_body, c.narm, c.ngrip, c.grip_act = T["tcp_body"], len(T["arm_qpos"]), len(T["grip_qpos"]), T["grip_act"]
        c.arm_qpos[:c.narm] = T["arm_qpos"]
        c.grip_qpos[:c.ngrip] = T["grip_qpos"]
        c.grip_qvel[:c.ngrip] = T["grip_qvel"]
        c.force_adr, c.torque_adr = T["force_adr"], T["torque_adr"]
        c.geom_object, c.geom_flags = ptr(self.geom_object), ptr(self.geom_flags)
        c.table_plane, c.wrist_sphere = T["table_plane"], T["wrist_sphere"]
        c.pad[:] = T["pad"]
        e, go = goal._e, goal._e.out
        c.goal_pos, c.goal_quat, c.group = ptr(e.goal_pos), ptr(e.goal_quat), ptr(e.groups)
        c.rel_pos, c.rel_rot = ptr(go["rel_goal_obj_pos"]), ptr(go["rel_goal_obj_rot"])
        c.achieved, c.off_table = ptr(go["goal_achieved"]), ptr(go["objects_off_table"])
        c.qpos_at_goal = ptr(self.qpos_at_goal)
        c.bbox_size, c.colors, c.boundary = ptr(self.bbox_size), ptr(self.colors), ptr(self.boundary)
        c.penalty[:] = _penalty(penalty)
        c.mask_obs, c.mask_margin = int(self.mask_obs), float(mask_margin)

        b = dict(dtype=t.bool, device=dev)
        v3 = lambda: t.zeros(nenv, nobj, 3, **f64)
        o = dict(obj_pos=v3(), obj_rel_pos=v3(), obj_vel_pos=v3(), obj_rot=v3(), obj_vel_rot=v3(), robot_joint_pos=t.zeros(nenv, c.narm, **f64),
                 gripper_pos=t.zeros(nenv, 3, **f64), gripper_velp=t.zeros(nenv, 3, **f64), gripper_controls=t.zeros(nenv, 1, **f64),
                 gripper_qpos=t.zeros(nenv, c.ngrip, **f64), gripper_vel=t.zeros(nenv, c.ngrip, **f64), qpos=t.zeros(nenv, nq, **f64),
                 qpos_goal=t.zeros(nenv, nq, **f64), goal_obj_pos=v3(), goal_obj_rot=v3(), rel_goal_obj_pos=v3(), rel_goal_obj_rot=v3(),
                 is_goal_achieved=t.zeros(nenv, 1, dtype=t.int32, device=dev), obj_gripper_contact=t.zeros(nenv, nobj, 2, **f64), obj_bbox_size=v3(),
                 obj_colors=t.zeros(nenv, nobj, 4, **f64), safety_stop=t.zeros(nenv, 1, **b), tcp_force=t.zeros(nenv, 3, **f64),
                 tcp_torque=t.zeros(nenv, 3, **f64))
        if self.mask_obs:
            o.update(placement_mask=t.ones(nenv, nobj, 1, **f64), goal_placement_mask=t.ones(nenv, nobj, 1, **f64))
            for k in OBJECT_KEYS + GOAL_KEYS:
                o["masked_" + k] = t.zeros_like(o[k])
        self.obs = o
        self.info = dict(gripper_table_contact=t.zeros(nenv, **b), wrist_cam_contacts=t.zeros(nenv, 4, **b), sim_reward=t.zeros(nenv, **f64),
                         sim_done=t.zeros(nenv, **b))
        self.cout = ObsOut(**{k: ptr(o.get(k, self.info.get(k))) for k in OUT_FIELDS})

    def set_reset_rows(self, bbox_size=None, colors=None, placement_area_boundary=None, mask=None):
        """Per-reset rows, for every environment or those of `mask` [nenv]: bbox_size [nenv, nobj, 3] (half sizes), colors
        [nenv, nobj, 4], placement_area_boundary [nenv, 6]; None keeps a row as it is."""
        t, dev, nenv, nobj = self.t, self.sim.device, self.nenv, self.nobj
        mk = None if mask is None else as_device(t, mask, t.bool, (nenv,), "mask", dev)
        for x, dst, shape, name in ((bbox_size, self.bbox_size, (nenv, nobj, 3), "bbox_size"), (colors, self.colors, (nenv, nobj, 4), "colors"),
                                    (placement_area_boundary, self.boundary, (nenv, 6), "placement_area_boundary")):
            if x is None:
                continue
            v = as_device(t, x, t.float64, shape, name, dev)
            if not bool(t.isfinite(v).all()):
                raise ValueError(f"{name}: finite")
            if mk is None:
                dst.copy_(v)
            else:
                dst[mk] = v[mk]

    def set_goal_qpos(self, qpos=None, mask=None):
        """The qpos the goal was set on (next_goal copies the simulation's qpos into qpos_goal, object_state.py:381-390): `qpos`
        [nenv, nq] or None for the sim's current qpos, for every environment or those of `mask`.  Call it at every goal reset."""
        t, dev = self.t, self.sim.device
        q = self.sim.qpos if qpos is None else as_device(t, qpos, t.float32, tuple(self.qpos_at_goal.shape), "qpos", dev)
        if mask is None:
            self.qpos_at_goal.copy_(q)
        else:
            mk = as_device(t, mask, t.bool, (self.nenv,), "mask", dev)
            self.qpos_at_goal[mk] = q[mk]

    def observe(self, mask=None):
        """(obs, info) of the current state and the goal's latest evaluate(), for every environment or those of `mask` (the others
        keep their previous values): dicts of device tensors, overwritten by the next call.  obs has the keys of
        `_observe_simple` (plus placement_mask, goal_placement_mask and masked_* with mask_obs_outside_placement_area); info
        gripper_table_contact [nenv], wrist_cam_contacts [nenv, 4] (WRIST_KEYS), objects_off_table [nenv, nobj] (the goal's),
        sim_reward [nenv] (minus the penalties that apply) and sim_done [nenv] (an active object off the table)."""
        t = self.t
        mk = device_mask(t, mask, self.nenv, self.sim.device)
        with t.cuda.device(self.sim.device):
            engine._check(engine.lib().rg_rearrange_obs(ctypes.byref(self.cin), ptr(mk), ctypes.byref(self.cout), current_stream(t, self.sim.device)))
        info = dict(self.info)
        info["objects_off_table"] = self.goal._e.out["objects_off_table"]
        return self.obs, info
