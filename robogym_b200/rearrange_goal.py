"""How far each rearrange object is from its goal, for a whole batch on the device, every env-step.

The reference evaluates goals per environment in numpy: `ObjectStateGoal.relative_goal` / `goal_distance`
(robogym/envs/rearrange/goals/object_state.py:492-599) with the rotation distance of its `rot_dist_type` (full, or the nearest
of the 24 / 4 parallel quaternions for mod90 / mod180), a greedy object-to-goal matching within every group of duplicate
objects, then `RearrangeEnv._calculate_num_success` / `_calculate_goal_distance_reward` (envs/rearrange/common/base.py:824-848),
`RobotEnv._is_successful` / `_get_goal_info` (robot_env.py:569-625) and `check_objects_off_table`
(envs/rearrange/simulation/base.py:805-832).  Here one launch does all of it, one warp per environment (`rg_rearrange_goal`,
robogym_b200/csrc/rg_goal.inl), reading the objects' poses in place from the sim's `body_xpos` / `body_xquat`.  At goal reset
`goal_orientations` samples the reference's `randomize_quaternion_along_z` / `randomize_quaternion_block` with the placement
kernel's counter-based random numbers.

ObjectStackGoal's extra keys (goals/object_stack_goal.py) come from the same launch when a gripper position is bound
(`gripper_site`, or `gripper_pos` of goal_distance): goal_distance["gripper_pos"] is |obj_pos - gripper_pos| per slot,
goal_distance["grasped"] the pad-contact sum passed to evaluate(), and both may appear in success_threshold.  With
goal_pos_offset 0, goal_rot_weight 1 and distinct groups the other keys are ObjectStackGoal's too.  `achieved_site` evaluates
ObjectReachGoal instead: the achieved position is that site's position, its rotation zero.

Padded slots (group -1) are zero on both sides, so they come out at distance max(goal_pos_offset, 0) and count as successes,
as in the reference: that is why the reward is a difference of success counts.

    goal = BatchedRearrangeGoal(sim, scene.bodies, groups, rp.table_dimensions(model), rot_dist_type="mod90")
    quat = goal_orientations(base_quat, active, *seed.next(), mode="block")
    valid = goal.set_goal(goal_pos, quat)            # per goal reset (mask: only some environments)
    info = goal.evaluate()                           # per env-step: info["reward"], info["goal_achieved"], info["done"], ...
"""
import ctypes

import numpy as np

from . import engine
from .engine import GoalIn, GoalOut, as_device, current_stream, device_mask, ptr

ROT_DIST = {"full": 0, "mod90": 1, "mod180": 2}
ROT_RANDOMIZE = {"z_axis": 1, "block": 2}
SUCCESS_KEYS = {"obj_pos": 1, "obj_rot": 2, "gripper_pos": 4, "grasped": 8}
# envs/rearrange/common/base.py:130-137
SUCCESS_THRESHOLD = {"obj_pos": 0.04, "obj_rot": 0.2}
MAX_OBJECTS = 64


def _settings(rot_dist_type, success_threshold):
    if rot_dist_type not in ROT_DIST:
        raise ValueError(f"rot_dist_type: one of {sorted(ROT_DIST)} (icp is not provided)")
    thr = dict(SUCCESS_THRESHOLD if success_threshold is None else success_threshold)
    if not thr or set(thr) - set(SUCCESS_KEYS):
        raise ValueError(f"success_threshold: a non-empty dict over {sorted(SUCCESS_KEYS)}")
    for k, v in thr.items():
        if not np.isfinite(float(v)):
            raise ValueError(f"success_threshold[{k!r}]: finite")
    keys = sum(SUCCESS_KEYS[k] for k in thr)
    return ROT_DIST[rot_dist_type], keys, float(thr.get("obj_pos", 0.0)), float(thr.get("obj_rot", 0.0))


def _per_env(t, x, nenv, name, dev):
    v = as_device(t, x, t.float64, (nenv,), name, dev)
    if not bool(t.isfinite(v).all()):
        raise ValueError(f"{name}: finite")
    return v


def _groups(t, groups, nenv, nobj, dev):
    g = as_device(t, groups, t.int64, (nenv, nobj), "groups", dev)
    if bool(((g < -1) | (g >= nobj)).any()):
        raise ValueError(f"groups: ids in [-1, {nobj}) (-1: an inactive slot)")
    return g.to(t.int32).contiguous()


def _quat_ok(t, q, name):
    if not bool(t.isfinite(q).all()) or bool((q.norm(dim=-1) == 0).any()):
        raise ValueError(f"{name}: finite and non-zero")


def _table(table):
    return np.concatenate([np.asarray(table[0], dtype=np.float64).reshape(3), np.asarray(table[1], dtype=np.float64).reshape(3)])


class _Evaluation:
    """the arguments and output buffers of one rg_rearrange_goal call site: the pose rows `pos` / `quat` (float32, `rows` slot ->
    row id, `pos_stride` / `quat_stride` floats per environment), the goals, groups and settings.  The outputs are kept and
    overwritten by every call."""

    def __init__(self, t, dev, nenv, nobj, rows, table, rot_dist_type, success_threshold, goal_reward_per_object, goal_pos_offset,
                 goal_rot_weight):
        self.t, self.dev, self.nenv, self.nobj = t, dev, nenv, nobj
        rd, keys, tp, tr = _settings(rot_dist_type, success_threshold)
        self.rows = np.ascontiguousarray(rows, dtype=np.int32)
        self.goal_pos = t.zeros(nenv, nobj, 3, dtype=t.float64, device=dev)
        self.goal_quat = t.zeros(nenv, nobj, 4, dtype=t.float64, device=dev)
        self.goal_quat[..., 0] = 1.0
        self.groups = t.full((nenv, nobj), -1, dtype=t.int32, device=dev)
        self.pos_offset = _per_env(t, goal_pos_offset, nenv, "goal_pos_offset", dev)
        self.rot_weight = _per_env(t, goal_rot_weight, nenv, "goal_rot_weight", dev)
        self.prev = t.full((nenv,), float("nan"), dtype=t.float64, device=dev)
        f64 = dict(dtype=t.float64, device=dev)
        b = dict(dtype=t.bool, device=dev)
        self.out = dict(obj_rot=t.zeros(nenv, nobj, 3, **f64), rel_goal_obj_pos=t.zeros(nenv, nobj, 3, **f64), rel_goal_obj_rot=t.zeros(nenv, nobj, 3, **f64),
                        dist_obj_pos=t.zeros(nenv, nobj, **f64), dist_obj_rot=t.zeros(nenv, nobj, **f64), success=t.zeros(nenv, nobj, **b),
                        objects_off_table=t.zeros(nenv, nobj, **b), num_success=t.zeros(nenv, **f64), reward=t.zeros(nenv, **f64),
                        goal_achieved=t.zeros(nenv, **b), done=t.zeros(nenv, **b), pick=t.zeros(nenv, nobj, dtype=t.int32, device=dev))
        o = self.out
        self.cout = GoalOut(ptr(o["obj_rot"]), ptr(o["rel_goal_obj_pos"]), ptr(o["rel_goal_obj_rot"]), ptr(o["dist_obj_pos"]), ptr(o["dist_obj_rot"]),
                            ptr(o["success"]), ptr(o["objects_off_table"]), ptr(o["num_success"]), ptr(o["reward"]), ptr(o["goal_achieved"]),
                            ptr(o["done"]), ptr(o["pick"]))
        self.cin = GoalIn()
        self.cin.nenv, self.cin.nobj = nenv, nobj
        self.cin.rows = self.rows.ctypes.data
        self.cin.goal_pos, self.cin.goal_quat, self.cin.group = ptr(self.goal_pos), ptr(self.goal_quat), ptr(self.groups)
        self.cin.pos_offset, self.cin.rot_weight = ptr(self.pos_offset), ptr(self.rot_weight)
        self.cin.table[:] = _table(table).tolist()
        self.cin.rot_dist_type, self.cin.success_keys = rd, keys
        self.cin.pos_threshold, self.cin.rot_threshold, self.cin.reward_per_object = tp, tr, float(goal_reward_per_object)
        if not np.isfinite(self.cin.reward_per_object):
            raise ValueError("goal_reward_per_object: finite")
        thr = SUCCESS_THRESHOLD if success_threshold is None else success_threshold
        self.cin.gripper_threshold, self.cin.grasped_threshold = float(thr.get("gripper_pos", 0.0)), float(thr.get("grasped", 0.0))
        self.grasped = None

    def bind_gripper(self, pos, stride):
        """ObjectStackGoal's gripper position, float32, read in place: environment e's at pos[e * stride] (pos: a tensor whose
        first element is environment 0's x, or (tensor, offset in floats))"""
        t, f64 = self.t, dict(dtype=self.t.float64, device=self.dev)
        base, off = pos if isinstance(pos, tuple) else (pos, 0)
        self._grip = base                                # alive while bound
        self.cin.gripper_pos = ctypes.c_void_p(base.data_ptr() + 4 * int(off))
        self.cin.gripper_stride = int(stride)
        o = self.out
        o["rel_gripper_pos"], o["dist_gripper_pos"] = t.zeros(self.nenv, self.nobj, 3, **f64), t.zeros(self.nenv, self.nobj, **f64)
        self.cout.rel_gripper, self.cout.dist_gripper = ptr(o["rel_gripper_pos"]), ptr(o["dist_gripper_pos"])

    def bind_poses(self, pos, quat, pos_stride, quat_stride):
        self._poses = (pos, quat)                        # alive while bound
        self.cin.pos, self.cin.quat = ptr(pos), ptr(quat)
        self.cin.pos_stride, self.cin.quat_stride = int(pos_stride), int(quat_stride)

    def run(self, mask=None, grasped=None):
        t = self.t
        mk = device_mask(t, mask, self.nenv, self.dev)
        self.grasped = None if grasped is None else as_device(t, grasped, t.float64, (self.nenv, self.nobj), "grasped", self.dev)
        self.cin.grasped = ptr(self.grasped)
        with t.cuda.device(self.dev):
            engine._check(engine.lib().rg_rearrange_goal(ctypes.byref(self.cin), ptr(mk), ptr(self.prev), ctypes.byref(self.cout),
                                                         current_stream(t, self.dev)))
        o = self.out
        r = dict(rel_goal_obj_pos=o["rel_goal_obj_pos"], rel_goal_obj_rot=o["rel_goal_obj_rot"], goal_achieved=o["goal_achieved"],
                 goal_distance=dict(obj_pos=o["dist_obj_pos"], obj_rot=o["dist_obj_rot"]), success=o["success"], num_success=o["num_success"],
                 obj_rot=o["obj_rot"], reward=o["reward"], objects_off_table=o["objects_off_table"], done=o["done"], pick=o["pick"])
        if "rel_gripper_pos" in o:
            r["rel_gripper_pos"] = o["rel_gripper_pos"]
            r["goal_distance"]["gripper_pos"] = o["dist_gripper_pos"]
        if self.grasped is not None:
            r["goal_distance"]["grasped"] = self.grasped
        return r


def _objects_off_table(t, pos, active, table):
    """check_objects_off_table of the active slots (fp64, as the kernel): z below 0.75 x table height, or x / y beyond the table"""
    tab = t.as_tensor(_table(table), device=pos.device)
    lo, hi = tab[:3] - tab[3:], tab[:3] + tab[3:]
    off = (pos[..., 2] < (tab[5] + tab[2]) * 0.75) | (pos[..., 0] < lo[0]) | (pos[..., 0] > hi[0]) | (pos[..., 1] < lo[1]) | (pos[..., 1] > hi[1])
    return off & active


class BatchedRearrangeGoal:
    """The goal of every environment of a rearrange batch and its evaluation after each env-step.

    sim: a BatchedSim with the outputs body_xpos and body_xquat; object_bodies: the body id of each object slot (<= 64);
    groups: [nenv, nobj] (or [nobj]) group id per slot, duplicates sharing one, -1 for an inactive (padded) slot;
    table: rearrange_placement.table_dimensions(model).  rot_dist_type, success_threshold, goal_reward_per_object are the
    reference's constants; goal_pos_offset and goal_rot_weight its randomisable simulation parameters, scalars or [nenv].
    gripper_site (a site name, e.g. "robot0:grip"; the sim needs the output site_xpos) adds ObjectStackGoal's gripper_pos key.
    achieved_site evaluates ObjectReachGoal: one slot whose achieved position is that site's (site_xpos) and whose rotation is
    zero; object_bodies is then not read (None)."""

    def __init__(self, sim, object_bodies, groups, table, rot_dist_type="full", success_threshold=None, goal_reward_per_object=1.0,
                 goal_pos_offset=0.0, goal_rot_weight=1.0, gripper_site=None, achieved_site=None):
        t = sim.torch
        sites = {}
        for name in (gripper_site, achieved_site):
            if name is not None:
                if getattr(sim, "site_xpos", None) is None:
                    raise ValueError("a gripper or achieved site needs the sim output site_xpos")
                sites[name] = sim.model.name2id("site", name)
        nsite = 0 if getattr(sim, "site_xpos", None) is None else int(sim.site_xpos.shape[1])
        if achieved_site is not None:
            sid = sites[achieved_site]
            self.sim, self.t, self.nenv, self.nobj, self.table = sim, t, sim.nenv, 1, table
            self._e = _Evaluation(t, sim.device, sim.nenv, 1, [sid], table, rot_dist_type, success_threshold, goal_reward_per_object,
                                  goal_pos_offset, goal_rot_weight)
            # the site's rotation is the identity: quaternion rows up to the site's id, all (1, 0, 0, 0)
            self._identity = t.zeros(sim.nenv, sid + 1, 4, dtype=t.float32, device=sim.device)
            self._identity[..., 0] = 1.0
            self._e.bind_poses(sim.site_xpos, self._identity, 3 * nsite, 4 * (sid + 1))
        else:
            if getattr(sim, "body_xpos", None) is None or getattr(sim, "body_xquat", None) is None:
                raise ValueError("the sim needs the outputs body_xpos and body_xquat")
            bodies = np.asarray(object_bodies, dtype=np.int64).reshape(-1)
            nbody = int(sim.body_xpos.shape[1])
            if not 1 <= len(bodies) <= MAX_OBJECTS or (bodies < 0).any() or (bodies >= nbody).any():
                raise ValueError(f"object_bodies: 1 to {MAX_OBJECTS} body ids in [0, {nbody})")
            self.sim, self.t, self.nenv, self.nobj, self.table = sim, t, sim.nenv, len(bodies), table
            self._e = _Evaluation(t, sim.device, sim.nenv, len(bodies), bodies, table, rot_dist_type, success_threshold, goal_reward_per_object,
                                  goal_pos_offset, goal_rot_weight)
            self._e.bind_poses(sim.body_xpos, sim.body_xquat, 3 * nbody, 4 * nbody)
        if gripper_site is not None:
            self._e.bind_gripper((sim.site_xpos, 3 * sites[gripper_site]), 3 * nsite)
        self.set_groups(groups)

    @property
    def goal_pos(self):
        return self._e.goal_pos

    @property
    def goal_quat(self):
        return self._e.goal_quat

    @property
    def groups(self):
        return self._e.groups

    def set_groups(self, groups):
        """group id per slot, [nenv, nobj] or [nobj]; -1 marks an inactive slot"""
        self._e.groups.copy_(_groups(self.t, groups, self.nenv, self.nobj, self.sim.device))

    def set_params(self, goal_pos_offset=None, goal_rot_weight=None):
        """the randomisable goal_pos_offset / goal_rot_weight, scalars or [nenv]"""
        if goal_pos_offset is not None:
            self._e.pos_offset.copy_(_per_env(self.t, goal_pos_offset, self.nenv, "goal_pos_offset", self.sim.device))
        if goal_rot_weight is not None:
            self._e.rot_weight.copy_(_per_env(self.t, goal_rot_weight, self.nenv, "goal_rot_weight", self.sim.device))

    def set_goal(self, pos, quat, mask=None):
        """New goals, pos [nenv, nobj, 3] and quat [nenv, nobj, 4] (w x y z), for every environment or those of `mask` [nenv];
        their previous success counts are cleared, so the next evaluation's reward is 0 (`_previous_goal_distance = None`).
        Returns goal_valid [nenv] bool: no active goal off the table (`next_goal`'s target_on_table)."""
        t, e, dev = self.t, self._e, self.sim.device
        p = as_device(t, pos, t.float64, (self.nenv, self.nobj, 3), "pos", dev)
        q = as_device(t, quat, t.float64, (self.nenv, self.nobj, 4), "quat", dev)
        if not bool(t.isfinite(p).all()):
            raise ValueError("pos: finite")
        _quat_ok(t, q, "quat")
        if mask is None:
            e.goal_pos.copy_(p); e.goal_quat.copy_(q); e.prev.fill_(float("nan"))
        else:
            mk = as_device(t, mask, t.bool, (self.nenv,), "mask", dev)
            e.goal_pos[mk] = p[mk]; e.goal_quat[mk] = q[mk]; e.prev[mk] = float("nan")
        return ~_objects_off_table(t, e.goal_pos, e.groups >= 0, self.table).any(dim=1)

    def evaluate(self, mask=None, grasped=None):
        """The goal information of the current poses (after a step or forward), for every environment or those of `mask` (the
        others keep their previous values): a dict of device tensors, overwritten by the next call --
        rel_goal_obj_pos / rel_goal_obj_rot [nenv, nobj, 3] (relative_goal), goal_distance {obj_pos, obj_rot} [nenv, nobj],
        success [nenv, nobj], num_success [nenv] (count x goal_reward_per_object, padded slots included), goal_achieved
        [nenv], reward [nenv] (num_success minus the previous evaluation's; 0 on the first after set_goal), obj_rot
        [nenv, nobj, 3] (get_object_rot), objects_off_table [nenv, nobj], done [nenv] (any object off the table), pick
        [nenv, nobj] (matched goal slot * 32 + parallel quaternion index, 31: none).  With a gripper_site: rel_gripper_pos
        [nenv, nobj, 3] (obj_pos - gripper_pos) and goal_distance["gripper_pos"] [nenv, nobj]; with `grasped` ([nenv, nobj], the
        two pad contact flags summed per slot, as is_object_grasped): goal_distance["grasped"]."""
        return self._e.run(mask, grasped)


def goal_distance(obj_pos, obj_quat, goal_pos, goal_quat, groups, table, rot_dist_type="full", success_threshold=None, goal_reward_per_object=1.0,
                  goal_pos_offset=0.0, goal_rot_weight=1.0, previous=None, mask=None, gripper_pos=None, grasped=None):
    """The evaluation of BatchedRearrangeGoal on poses given as tensors: obj_pos [nenv, nobj, 3], obj_quat [nenv, nobj, 4] (CUDA; read
    as float32, as a sim stores them), goal_pos / goal_quat (float64), groups [nenv, nobj].  `previous` ([nenv] float64 CUDA,
    in / out) carries the success count from one call to the next (NaN: none; None: a fresh one, reward 0).  gripper_pos
    ([nenv, 3], read as float32) and grasped ([nenv, nobj]) add ObjectStackGoal's keys.  Returns the dict of evaluate() (new
    tensors) and "previous"."""
    import torch as t

    if not t.is_tensor(obj_pos) or not obj_pos.is_cuda:
        raise ValueError("obj_pos: a CUDA tensor [nenv, nobj, 3]")
    if obj_pos.dim() != 3 or obj_pos.shape[2] != 3:
        raise ValueError("obj_pos: [nenv, nobj, 3]")
    nenv, nobj = int(obj_pos.shape[0]), int(obj_pos.shape[1])
    if not 1 <= nobj <= MAX_OBJECTS:
        raise ValueError(f"1 to {MAX_OBJECTS} objects per environment")
    dev = obj_pos.device
    p = as_device(t, obj_pos, t.float32, (nenv, nobj, 3), "obj_pos", dev)
    q = as_device(t, obj_quat, t.float32, (nenv, nobj, 4), "obj_quat", dev)
    gp = as_device(t, goal_pos, t.float64, (nenv, nobj, 3), "goal_pos", dev)
    gq = as_device(t, goal_quat, t.float64, (nenv, nobj, 4), "goal_quat", dev)
    if not bool(t.isfinite(p).all()) or not bool(t.isfinite(gp).all()):
        raise ValueError("positions: finite")
    _quat_ok(t, q, "obj_quat")
    _quat_ok(t, gq, "goal_quat")
    e = _Evaluation(t, dev, nenv, nobj, np.arange(nobj), table, rot_dist_type, success_threshold, goal_reward_per_object, goal_pos_offset,
                    goal_rot_weight)
    e.goal_pos.copy_(gp); e.goal_quat.copy_(gq)
    e.groups.copy_(_groups(t, groups, nenv, nobj, dev))
    if previous is not None:
        if not t.is_tensor(previous) or previous.dtype != t.float64 or tuple(previous.shape) != (nenv,) or previous.device != dev or not previous.is_contiguous():
            raise ValueError("previous: a contiguous float64 tensor [nenv] on the device of obj_pos")
        e.prev = previous
    e.bind_poses(p, q, 3 * nobj, 4 * nobj)
    if gripper_pos is not None:
        g = as_device(t, gripper_pos, t.float32, (nenv, 3), "gripper_pos", dev)
        if not bool(t.isfinite(g).all()):
            raise ValueError("gripper_pos: finite")
        e.bind_gripper(g, 3)
    out = e.run(mask, grasped)
    out["previous"] = e.prev
    return out


def goal_orientations(base_quat, active, seed, epoch, mode="z_axis", mask=None):
    """Goal quaternions at goal reset: `randomize_quaternion_along_z` ("z_axis": a uniform yaw times base) or
    `randomize_quaternion_block` ("block": yaw times base times one of the 24 parallel quaternions) for the active slots
    ([nenv, nobj]) of every environment (or those of `mask`), base_quat [nenv, nobj, 4] (CUDA, w x y z: the current target
    quaternions).  Returns a new [nenv, nobj, 4] float64 tensor, base_quat elsewhere.  seed, epoch: PlacementSeed.next().
    "full" needs numpy's normal draws and is not provided."""
    import torch as t

    if mode == "full":
        raise ValueError('rot_randomize_type "full" is not provided (it draws numpy\'s legacy normal variates): use "z_axis" or "block"')
    if mode not in ROT_RANDOMIZE:
        raise ValueError(f"rot_randomize_type: one of {sorted(ROT_RANDOMIZE)}")
    if not t.is_tensor(base_quat) or not base_quat.is_cuda or base_quat.dim() != 3 or base_quat.shape[2] != 4:
        raise ValueError("base_quat: a CUDA tensor [nenv, nobj, 4]")
    nenv, nobj = int(base_quat.shape[0]), int(base_quat.shape[1])
    if not 1 <= nobj <= MAX_OBJECTS:
        raise ValueError(f"1 to {MAX_OBJECTS} objects per environment")
    if not (0 <= int(seed) < 1 << 32 and 0 <= int(epoch) < 1 << 32):
        raise ValueError("seed and epoch: 32-bit unsigned integers")
    dev = base_quat.device
    out = base_quat.to(t.float64).contiguous().clone()
    _quat_ok(t, out, "base_quat")
    act = as_device(t, active, t.uint8, (nenv, nobj), "active", dev)
    mk = device_mask(t, mask, nenv, dev)
    with t.cuda.device(dev):
        engine._check(engine.lib().rg_goal_orientations(nenv, nobj, ptr(out), ptr(act), ROT_RANDOMIZE[mode], int(seed), int(epoch), ptr(mk),
                                                        ptr(out), current_stream(t, dev)))
    return out
