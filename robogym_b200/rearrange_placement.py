"""Where a rearrange reset puts the objects and their goals, for a whole batch on the device.

The reference places objects from their rotated bounding boxes at every reset (`RearrangeEnv._generate_object_placements`,
robogym/envs/rearrange/common/base.py:797-822): `place_objects_in_grid`, and when that fails the rejection sampler
`place_objects_with_no_constraint` (100 restarts x 21 proposals per object), inside `get_placement_area`
(simulation/base.py:992-1010).  State goals are placed the same way (`ObjectStateGoal._sample_next_goal_positions`,
goals/object_state.py:434-457), and `TrainStateGoal` pulls each goal toward its object with
`place_targets_with_goal_distance_ratio` (common/utils.py:922-994).

Here the boxes come from `BatchedMeshScene.bounding_boxes` / `BatchedBlockScene.bounding_boxes` (`rg_batch_body_aabb`) and
the placement from `rg_place_objects`, one warp per environment (robogym_b200/csrc/rg_place.inl), with the reference's
semantics and defaults, draw for draw: for the same random numbers the positions are the reference's float64 results.  The
random numbers are Philox4x32-10 keyed by (seed, environment) and addressed by an `epoch` per call, so a masked re-placement
draws the same numbers for an environment as a full one; `PlacementSeed` hands out a fresh epoch for every call.

The reference's other goal generators edit such a placement (`rg_goal_modify`, one thread per environment, same random-number
scheme under its own purpose): `stack_goals` (ObjectStackGoal), `pick_and_place_goals` (PickAndPlaceGoal), `train_goals`
(TrainStateGoal with pickup / stacking tasks) and `reach_goals` (ObjectReachGoal).  The generators that lay blocks out in a
pattern compute goals and rotations from the boxes directly (`rg_layout_goals`, one warp per environment, its own purpose):
`domino_goals` (DominoStateGoal), `attached_goals` (AttachedBlockStateGoal) and `fixed_goals` (ObjectFixedStateGoal).

An environment no algorithm could place comes back with status 0 (its active slots zeroed).  The reference raises
`InvalidSimulationError` there and `safe_reset_env` rebuilds the whole scene; here the caller redraws the flagged
environments (objects, scales, yaws) and places them again under a mask.

    table = table_dimensions(model)
    area = placement_area(table, active.sum(1), used_table_portion)
    seed = PlacementSeed(0)
    bbox = scene.bounding_boxes(quat)
    pos, status = object_placements(bbox, active, table, area, *seed.next())
"""
import numpy as np

from . import engine, modelblob
from .engine import as_device, current_stream, device_mask, ptr

MODES = {"grid": 1, "uniform": 2, "goal_distance_ratio": 3, "grid_then_uniform": 4}
STATUS = {0: None, 1: "grid", 2: "uniform", 3: "goal_distance_ratio"}
# simulation/base.py:83-84, :89-90
MAX_PLACEMENT_RETRY, MAX_PLACEMENT_RETRY_PER_OBJECT = 100, 20
GOAL_DISTANCE_MIN = 0.06
MAX_OBJECTS = 64
MODIFY = {"stack": 1, "lift": 2, "train": 3, "reach": 4}
# goals/pickandplace.py:15, goals/object_state.py GoalArgs.height_range
HEIGHT_RANGE = (0.05, 0.25)
LAYOUT = {"domino": 1, "attached": 2, "fixed": 3}
DOMINO_MAX_RETRY = 1000         # goals/dominos.py MAX_RETRY
ATTACHED_BLOCKS = 8             # goals/attached_block_state.py: the pattern's cells


def table_dimensions(model):
    """`get_table_dimensions` (simulation/base.py:923-932): (table body pos, table geom half size, table height = size_z + pos_z),
    float64, of a model blob (or anything with `.blob`)."""
    blob = getattr(model, "blob", model)
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    size = np.asarray(m["geom_size"], dtype=np.float64).reshape(-1, 3)[names["geom"].index("table")].copy()
    pos = np.asarray(m["body_pos"], dtype=np.float64).reshape(-1, 3)[names["body"].index("table")].copy()
    return pos, size, size[-1] + pos[-1]


def placement_area(table, num_objects, used_table_portion=1.0):
    """`get_placement_area` with `get_table_setting`'s clip (simulation/base.py:981-1010) per environment: num_objects is each
    environment's active count ([nenv] or a scalar), used_table_portion a scalar or [nenv].  Returns [nenv, 6] float64
    (offset x y z, size x y z)."""
    _, table_size, _ = table
    n = np.atleast_1d(np.asarray(num_objects.cpu() if hasattr(num_objects, "cpu") else num_objects))
    used = np.asarray(used_table_portion.cpu() if hasattr(used_table_portion, "cpu") else used_table_portion, dtype=np.float64)
    n, used = np.broadcast_arrays(n, used)
    table_size_x, table_size_y = table_size[:2] * 2
    used = np.clip(used, n * 0.1, 1.0)
    place_size_x = 0.5 * table_size_x * used
    place_size_y = 0.38 * table_size_y * used
    out = np.empty(n.shape + (6,))
    out[..., 0] = 0.5 * table_size_x - place_size_x / 2.0
    out[..., 1] = 0.44 * table_size_y - place_size_y / 2.0
    out[..., 2] = 2 * table_size[2]
    out[..., 3], out[..., 4], out[..., 5] = place_size_x, place_size_y, 0.26
    return out


class PlacementSeed:
    """A batch's placement seed and its epoch counter: every `next()` returns (seed, epoch) with a fresh epoch, so successive
    resets draw fresh numbers."""

    def __init__(self, seed=0):
        self.seed = int(seed) & 0xFFFFFFFF
        self.epoch = 0

    def next(self):
        e = self.epoch
        self.epoch = (self.epoch + 1) & 0xFFFFFFFF
        return self.seed, e


def _place(bbox, active, table, area, seed, epoch, mode, mask, out, max_trials, max_per_object, anchor, ratio, dmin):
    import torch as t

    if mode not in MODES:
        raise ValueError(f"mode: one of {sorted(MODES)}")
    if not t.is_tensor(bbox) or not bbox.is_cuda:
        raise ValueError("bbox: a CUDA tensor [nenv, nobj, 2, 3] (bounding_boxes)")
    if bbox.dim() != 4 or tuple(bbox.shape[2:]) != (2, 3):
        raise ValueError("bbox: [nenv, nobj, 2, 3] (center, half size)")
    nenv, nobj = int(bbox.shape[0]), int(bbox.shape[1])
    if nobj > MAX_OBJECTS:
        raise ValueError(f"at most {MAX_OBJECTS} objects per environment")
    dev = bbox.device
    bb = bbox.to(t.float64).contiguous()
    if not bool(t.isfinite(bb).all()) or bool((bb[:, :, 1] < 0).any()):
        raise ValueError("bbox: finite, with half sizes >= 0")
    act = as_device(t, active, t.uint8, (nenv, nobj), "active", dev)
    ar = as_device(t, area, t.float64, (nenv, 6), "area", dev)
    tab = np.concatenate([np.asarray(table[0], dtype=np.float64).reshape(3), np.asarray(table[1], dtype=np.float64).reshape(3)])
    if not (0 <= int(seed) < 1 << 32 and 0 <= int(epoch) < 1 << 32):
        raise ValueError("seed and epoch: 32-bit unsigned integers")
    if int(max_trials) < 1 or int(max_per_object) < 1:
        raise ValueError("max_trials and max_per_object must be >= 1")
    anc = None
    if mode == "goal_distance_ratio":
        if anchor is None:
            raise ValueError("goal_distance_ratio: the object placements (anchor) are needed")
        anc = as_device(t, anchor, t.float64, (nenv, nobj, 3), "anchor", dev)
    mk = device_mask(t, mask, nenv, dev)
    pos = t.zeros(nenv, nobj, 3, dtype=t.float64, device=dev) if out is None else out
    if pos.dtype != t.float64 or tuple(pos.shape) != (nenv, nobj, 3) or not pos.is_contiguous() or pos.device != dev:
        raise ValueError("out: a contiguous float64 tensor [nenv, nobj, 3] on the device of bbox")
    status = t.full((nenv,), -1, dtype=t.int32, device=dev)
    with t.cuda.device(dev):
        engine._check(engine.lib().rg_place_objects(nenv, nobj, ptr(bb), ptr(act), tab.ctypes.data, ptr(ar), MODES[mode], int(max_trials),
                                                    int(max_per_object), float(ratio), float(dmin), ptr(anc), int(seed), int(epoch), ptr(mk),
                                                    ptr(pos), ptr(status), current_stream(t, dev)))
    return pos, status


def object_placements(bbox, active, table, area, seed, epoch, mode="grid_then_uniform", mask=None, out=None,
                      max_trials=MAX_PLACEMENT_RETRY, max_per_object=MAX_PLACEMENT_RETRY_PER_OBJECT):
    """Body-origin positions of the objects, `_generate_object_placements` (mode "grid_then_uniform"), or one of its parts
    ("grid": place_objects_in_grid, "uniform": place_objects_with_no_constraint), for every environment (or those of `mask`).
    bbox [nenv, nobj, 2, 3] (CUDA, center relative to the body origin and half size: bounding_boxes), active [nenv, nobj]
    (placed in slot order; inactive slots are not written), table = table_dimensions(...), area [nenv, 6] (placement_area).
    `out` ([nenv, nobj, 3] float64 CUDA) is written in place for the placed slots, so masked-out environments and inactive
    slots keep what it held.  Returns (pos, status [nenv] int32: 1 grid, 2 uniform, 0 invalid -- redraw those environments --, -1 not selected by
    `mask`)."""
    return _place(bbox, active, table, area, seed, epoch, mode, mask, out, max_trials, max_per_object, None, 1.0, GOAL_DISTANCE_MIN)


def goal_placements(bbox, active, table, area, seed, epoch, mode="goal_distance_ratio", anchor=None, goal_distance_ratio=1.0,
                    goal_distance_min=GOAL_DISTANCE_MIN, mask=None, out=None, max_trials=MAX_PLACEMENT_RETRY,
                    max_per_object=MAX_PLACEMENT_RETRY_PER_OBJECT):
    """Goal positions: "goal_distance_ratio" is `TrainStateGoal` (place_targets_with_goal_distance_ratio: each goal drawn in the
    area, then pulled toward its object's placement `anchor` [nenv, nobj, 3] to goal_distance_ratio of the distance, never
    closer than goal_distance_min); "grid_then_uniform" is `ObjectStateGoal._sample_next_goal_positions`.  Otherwise as
    object_placements; status 3 marks a goal-distance placement."""
    if mode not in ("goal_distance_ratio", "grid_then_uniform"):
        raise ValueError('goal modes: "goal_distance_ratio" or "grid_then_uniform"')
    return _place(bbox, active, table, area, seed, epoch, mode, mask, out, max_trials, max_per_object, anchor, goal_distance_ratio, goal_distance_min)


def _active_counts(t, active, mask, nenv, nobj, dev):
    """the active mask as the launches read it, and each selected environment's active count ([nenv] int64 on the host)"""
    act = as_device(t, active, t.uint8, (nenv, nobj), "active", dev)
    n = act.sum(1).cpu().numpy().astype(np.int64)
    if mask is not None:
        n = np.where(np.asarray(as_device(t, mask, t.bool, (nenv,), "mask", "cpu")), n, -1)
    return act, n


def _modify(kind, pos, act, seed, epoch, mask, object_size=None, ratio=None, target_height=None, height_range=(0.0, 0.0), pickup=0.0,
            stacking=0.0, fixed_order=True):
    import torch as t

    nenv, nobj, dev = int(pos.shape[0]), int(pos.shape[1]), pos.device
    per = {}
    for name, v in (("object_size", object_size), ("goal_distance_ratio", ratio), ("target_height", target_height)):
        if v is not None:
            per[name] = as_device(t, v, t.float64, (nenv,), name, dev)
            if not bool(t.isfinite(per[name]).all()):
                raise ValueError(f"{name}: finite")
    mk = device_mask(t, mask, nenv, dev)
    with t.cuda.device(dev):
        engine._check(engine.lib().rg_goal_modify(nenv, nobj, MODIFY[kind], ptr(act), ptr(per.get("object_size")), ptr(per.get("goal_distance_ratio")),
                                                  ptr(per.get("target_height")), float(height_range[0]), float(height_range[1]), float(pickup),
                                                  float(stacking), int(bool(fixed_order)), int(seed), int(epoch), ptr(mk), ptr(pos),
                                                  current_stream(t, dev)))
    return pos


def _height_range(height_range):
    lo, hi = (float(x) for x in height_range)
    if not (np.isfinite(lo) and np.isfinite(hi) and lo <= hi):
        raise ValueError("height_range: finite (min, max) with min <= max")
    return lo, hi


def _bbox_shape(bbox):
    import torch as t

    if not t.is_tensor(bbox) or not bbox.is_cuda or bbox.dim() != 4:
        raise ValueError("bbox: a CUDA tensor [nenv, nobj, 2, 3] (bounding_boxes)")
    return int(bbox.shape[0]), int(bbox.shape[1]), bbox.device


def stack_goals(bbox, active, table, area, seed, epoch, object_size, fixed_order=False, mask=None, out=None, max_trials=MAX_PLACEMENT_RETRY,
                max_per_object=MAX_PLACEMENT_RETRY_PER_OBJECT):
    """`ObjectStackGoal._sample_next_goal_positions` (goals/object_stack_goal.py): the first active object placed alone by
    place_objects_with_no_constraint, then every active object on that spot in block order (slot order with fixed_order, else
    a shuffle), object i of the order raised by i * object_size * 2.  object_size: [nenv] or a scalar (each environment's block
    size).  Every selected environment needs two or more active objects.  Returns (pos, status) as goal_placements; status is
    the bottom object's placement (2, or 0: the tower is built on zeros, as the reference's)."""
    import torch as t

    nenv, nobj, dev = _bbox_shape(bbox)
    act, n = _active_counts(t, active, mask, nenv, nobj, dev)
    if ((n >= 0) & (n < 2)).any():
        raise ValueError("stack_goals: every selected environment needs two or more active objects")
    first = t.zeros_like(act)
    first[t.arange(nenv, device=dev), act.argmax(1)] = 1
    first &= act
    pos, status = _place(bbox, first, table, area, seed, epoch, "uniform", mask, out, max_trials, max_per_object, None, 1.0, GOAL_DISTANCE_MIN)
    return _modify("stack", pos, act, seed, epoch, mask, object_size=object_size, fixed_order=fixed_order), status


def pick_and_place_goals(bbox, active, table, area, seed, epoch, height_range=HEIGHT_RANGE, mask=None, out=None, max_trials=MAX_PLACEMENT_RETRY,
                         max_per_object=MAX_PLACEMENT_RETRY_PER_OBJECT):
    """`PickAndPlaceGoal._sample_next_goal_positions` (goals/pickandplace.py): ObjectStateGoal's goals (grid, then uniform), then
    one active object, randint(n), lifted by uniform(*height_range).  Returns (pos, status) as goal_placements."""
    import torch as t

    hr = _height_range(height_range)
    nenv, nobj, dev = _bbox_shape(bbox)
    act, n = _active_counts(t, active, mask, nenv, nobj, dev)
    if (n == 0).any():
        raise ValueError("pick_and_place_goals: every selected environment needs an active object")
    pos, status = _place(bbox, act, table, area, seed, epoch, "grid_then_uniform", mask, out, max_trials, max_per_object, None, 1.0, GOAL_DISTANCE_MIN)
    return _modify("lift", pos, act, seed, epoch, mask, height_range=hr), status


def train_goals(bbox, active, table, area, seed, epoch, anchor, goal_distance_ratio=1.0, pickup_proba=0.0, stacking_proba=0.0,
                height_range=HEIGHT_RANGE, object_size=0.0254, goal_distance_min=GOAL_DISTANCE_MIN, mask=None, out=None,
                max_trials=MAX_PLACEMENT_RETRY, max_per_object=MAX_PLACEMENT_RETRY_PER_OBJECT):
    """`TrainStateGoal._sample_next_goal_positions` (goals/train_state.py): goals pulled toward the object placements `anchor`
    (goal_placements' "goal_distance_ratio"), then `move_one_object_to_the_air_with_restrictions`: p = random(); nothing when
    p > pickup_proba + stacking_proba, a lift of uniform(*height_range) * goal_distance_ratio when p < pickup_proba, otherwise a
    tower of randint(2, n + 1) active objects on the first one's xy, member k + 1 raised by object_size * (k + 1) * 2 (an
    environment with fewer than two active objects is left as placed).  The reference draws the tower's members with the global
    np.random.choice; here they are a partial Fisher-Yates draw from the environment's own stream.  goal_distance_ratio: a
    scalar (the placement takes one); object_size: [nenv] or a scalar.  Returns (pos, status) as goal_placements."""
    import torch as t

    hr = _height_range(height_range)
    pickup, stacking = float(pickup_proba), float(stacking_proba)
    if not (pickup >= 0.0 and stacking >= 0.0 and 0.0 <= pickup + stacking <= 1.0):
        raise ValueError("pickup_proba and stacking_proba: >= 0, with pickup_proba + stacking_proba in [0, 1]")
    nenv, nobj, dev = _bbox_shape(bbox)
    act, n = _active_counts(t, active, mask, nenv, nobj, dev)
    if pickup > 0.0 and (n == 0).any():
        raise ValueError("train_goals: a pickup draw needs an active object in every selected environment")
    pos, status = _place(bbox, act, table, area, seed, epoch, "goal_distance_ratio", mask, out, max_trials, max_per_object, anchor,
                         goal_distance_ratio, goal_distance_min)
    return _modify("train", pos, act, seed, epoch, mask, object_size=object_size, ratio=float(goal_distance_ratio), height_range=hr, pickup=pickup,
                   stacking=stacking), status


def reach_goals(bbox, active, table, area, seed, epoch, target_height, mask=None, out=None, max_trials=MAX_PLACEMENT_RETRY,
                max_per_object=MAX_PLACEMENT_RETRY_PER_OBJECT):
    """`ObjectReachGoal._sample_next_goal_positions` (goals/object_reach_goal.py): the one object placed by
    place_objects_with_no_constraint, then the goal target_height ([nenv] or a scalar) above it.  Every selected environment
    must have exactly one active object (the reference asserts num_objects == 1).  Returns (goal_pos, object_pos, status):
    object_pos is the placement the reference writes into the object's joint (set_object_pos)."""
    import torch as t

    nenv, nobj, dev = _bbox_shape(bbox)
    act, n = _active_counts(t, active, mask, nenv, nobj, dev)
    if ((n >= 0) & (n != 1)).any():
        raise ValueError("reach_goals: every selected environment needs exactly one active object")
    pos, status = _place(bbox, act, table, area, seed, epoch, "uniform", mask, out, max_trials, max_per_object, None, 1.0, GOAL_DISTANCE_MIN)
    obj = pos.clone()
    return _modify("reach", pos, act, seed, epoch, mask, target_height=target_height), obj, status


def _layout(kind, bbox, active, table, area, seed, epoch, mask, out, object_size=None, distance_mul=None, rel=None, max_retry=1):
    """rg_layout_goals: (pos, quat, status, angle, retry); angle and retry only for dominoes (else None)"""
    import torch as t

    nenv, nobj, dev = _bbox_shape(bbox)
    if tuple(bbox.shape[2:]) != (2, 3):
        raise ValueError("bbox: [nenv, nobj, 2, 3] (center, half size)")
    if nobj > MAX_OBJECTS:
        raise ValueError(f"at most {MAX_OBJECTS} objects per environment")
    bb = bbox.to(t.float64).contiguous()
    if not bool(t.isfinite(bb).all()) or bool((bb[:, :, 1] < 0).any()):
        raise ValueError("bbox: finite, with half sizes >= 0")
    if not (0 <= int(seed) < 1 << 32 and 0 <= int(epoch) < 1 << 32):
        raise ValueError("seed and epoch: 32-bit unsigned integers")
    act, n = _active_counts(t, active, mask, nenv, nobj, dev)
    ar = as_device(t, area, t.float64, (nenv, 6), "area", dev)
    tab = np.concatenate([np.asarray(table[0], dtype=np.float64).reshape(3), np.asarray(table[1], dtype=np.float64).reshape(3)])
    per = {}
    for name, v in (("object_size", object_size), ("distance_mul", distance_mul)):
        if v is not None:
            per[name] = as_device(t, v, t.float64, (nenv,), name, dev)
            if not bool((t.isfinite(per[name]) & (per[name] > 0)).all()):
                raise ValueError(f"{name}: finite and > 0")
    if out is None:
        pos = t.zeros(nenv, nobj, 3, dtype=t.float64, device=dev)
        quat = t.zeros(nenv, nobj, 4, dtype=t.float64, device=dev)
        quat[..., 0] = 1.0
    else:
        pos, quat = out
        for name, x, w in (("pos", pos, 3), ("quat", quat, 4)):
            if not t.is_tensor(x) or x.dtype != t.float64 or tuple(x.shape) != (nenv, nobj, w) or not x.is_contiguous() or x.device != dev:
                raise ValueError(f"out: (pos, quat), contiguous float64 tensors [nenv, nobj, 3] and [nenv, nobj, 4] on the device of bbox ({name})")
    status = t.full((nenv,), -1, dtype=t.int32, device=dev)
    angle = retry = None
    if kind == "domino":
        angle = t.zeros(nenv, nobj, dtype=t.float64, device=dev)
        retry = t.full((nenv,), -1, dtype=t.int32, device=dev)
    mk = device_mask(t, mask, nenv, dev)
    with t.cuda.device(dev):
        engine._check(engine.lib().rg_layout_goals(nenv, nobj, LAYOUT[kind], ptr(bb), ptr(act), tab.ctypes.data, ptr(ar), ptr(per.get("object_size")),
                                                   ptr(per.get("distance_mul")), ptr(rel), int(max_retry), int(seed), int(epoch), ptr(mk), ptr(pos),
                                                   ptr(quat), ptr(status), ptr(angle), ptr(retry), current_stream(t, dev)))
    return pos, quat, status, angle, retry


def domino_goals(bbox, active, table, area, seed, epoch, object_size, distance_mul, max_retry=DOMINO_MAX_RETRY, mask=None, out=None, details=False):
    """`DominoStateGoal._sample_next_goal_positions` (goals/dominos.py): the dominoes on a circle arc.  Each of up to max_retry
    tries draws the arc's offset and step, turns domino i by i * step + (offset + step / 2) about z, lays the dominoes
    object_size * distance_mul apart along the arc and keeps the first arc whose turned boxes fit in the placement area, moved
    to a uniform spot in it.  bbox: the unrotated boxes ([nenv, nobj, 2, 3] CUDA, bounding_boxes with the identity);
    object_size and distance_mul (domino_distance_mul): [nenv] or scalars, > 0.  Every selected environment needs an active
    object.  Returns (pos [nenv, nobj, 3], quat [nenv, nobj, 4] the z rotations, status [nenv] int32: 1 placed, 0 no arc fitted
    within max_retry -- positions zeroed, as the reference returns with goal_valid False --, -1 not selected by `mask`).
    `out` = (pos, quat) is written in place on the selected environments' active slots.  details=True adds angle [nenv, nobj]
    (the z angles) and retry [nenv] (the arc that fitted, -1 none).  Evaluate with rot_dist_type="mod180", as the reference's
    dominos environment does."""
    import torch as t

    if int(max_retry) < 1:
        raise ValueError("max_retry must be >= 1")
    nenv, nobj, dev = _bbox_shape(bbox)
    _, n = _active_counts(t, active, mask, nenv, nobj, dev)
    if (n == 0).any():
        raise ValueError("domino_goals: every selected environment needs an active object")
    pos, quat, status, angle, retry = _layout("domino", bbox, active, table, area, seed, epoch, mask, out, object_size=object_size,
                                              distance_mul=distance_mul, max_retry=max_retry)
    return (pos, quat, status, angle, retry) if details else (pos, quat, status)


def attached_goals(bbox, active, table, area, seed, epoch, object_size, mask=None, out=None):
    """`AttachedBlockStateGoal._sample_next_goal_positions` (goals/attached_block_state.py): eight blocks tightly attached in
    the reference's pattern (two rows of two around a row of four, cells of object_size * 2 in placement-area units), the rows
    permuted among the blocks and the pattern moved to a uniform origin in the area, then place_targets_with_fixed_position.
    object_size: [nenv] or a scalar, > 0.  Every selected environment needs exactly 8 active blocks, as the reference's
    blocks_attached environment has.  Returns (pos, quat, status) as domino_goals, with identity rotations and status 1."""
    import torch as t

    nenv, nobj, dev = _bbox_shape(bbox)
    _, n = _active_counts(t, active, mask, nenv, nobj, dev)
    if ((n >= 0) & (n != ATTACHED_BLOCKS)).any():
        raise ValueError(f"attached_goals: every selected environment needs exactly {ATTACHED_BLOCKS} active blocks")
    return _layout("attached", bbox, active, table, area, seed, epoch, mask, out, object_size=object_size)[:3]


def fixed_goals(bbox, active, table, area, relative_placements, init_quat=None, mask=None, out=None):
    """`ObjectFixedStateGoal._sample_next_goal_positions` (goals/object_state_fixed.py, the table_setting and wordblocks
    goals): place_targets_with_fixed_position of relative_placements ([nenv, nobj, 2] or [nobj, 2], each object's (x, y) as a
    fraction of the placement area; values outside [0, 1] are used as they are, as the reference does).  init_quat ([nenv,
    nobj, 4] or [nobj, 4], w x y z; None = identity) becomes the goal rotation with w >= 0 (set_target_quat's
    quat_normalize).  No random numbers.  Returns (pos, quat, status) as domino_goals, status 1."""
    import torch as t

    nenv, nobj, dev = _bbox_shape(bbox)
    rp = t.as_tensor(relative_placements.cpu() if t.is_tensor(relative_placements) else np.asarray(relative_placements, dtype=np.float64))
    if tuple(rp.shape) not in ((nobj, 2), (nenv, nobj, 2)):
        raise ValueError("relative_placements: [nobj, 2] or [nenv, nobj, 2]")
    rel = rp.to(device=dev, dtype=t.float64).expand(nenv, nobj, 2).contiguous()
    if not bool(t.isfinite(rel).all()):
        raise ValueError("relative_placements: finite")
    q0 = None
    if init_quat is not None:
        iq = t.as_tensor(init_quat.cpu() if t.is_tensor(init_quat) else np.asarray(init_quat, dtype=np.float64))
        if tuple(iq.shape) not in ((nobj, 4), (nenv, nobj, 4)):
            raise ValueError("init_quat: [nobj, 4] or [nenv, nobj, 4]")
        q0 = iq.to(device=dev, dtype=t.float64).expand(nenv, nobj, 4)
        if not bool(t.isfinite(q0).all()) or bool((q0.norm(dim=2) == 0).any()):
            raise ValueError("init_quat: finite and non-zero")
        q0 = t.where(q0[..., :1] < 0, -q0, q0)
    pos, quat, status = _layout("fixed", bbox, active, table, area, 0, 0, mask, out, rel=rel)[:3]
    if q0 is not None:
        act = as_device(t, active, t.bool, (nenv, nobj), "active", dev)
        if mask is not None:
            act = act & as_device(t, mask, t.bool, (nenv,), "mask", dev)[:, None]
        quat.copy_(t.where(act[..., None], q0, quat))
    return pos, quat, status


def body_aabb(sim, bodies, quat=None, mask=None):
    """rg_batch_body_aabb: (center, half size) [nenv, len(bodies), 2, 3] float64 of the bodies rotated by quat
    ([nenv, len(bodies), 4], w x y z; None = unrotated), relative to the body origin, from each environment's bound rows (the
    model's arrays where none is bound)."""
    t = sim.torch
    bodies = np.ascontiguousarray(np.asarray(bodies, dtype=np.int32).reshape(-1))
    n = len(bodies)
    if quat is None:
        quat = t.tensor([1.0, 0.0, 0.0, 0.0], dtype=t.float64)
    q = as_device(t, quat, t.float64, (sim.nenv, n, 4), "quat", sim.device)
    if not bool(t.isfinite(q).all()) or bool((q.norm(dim=2) == 0).any()):
        raise ValueError("quat: finite and non-zero")
    mk = device_mask(t, mask, sim.nenv, sim.device)
    out = t.zeros(sim.nenv, n, 2, 3, dtype=t.float64, device=sim.device)
    engine._check(engine.lib().rg_batch_body_aabb(sim.h, bodies.ctypes.data, n, ptr(q), ptr(mk), ptr(out), current_stream(t, sim.device)))
    return out
