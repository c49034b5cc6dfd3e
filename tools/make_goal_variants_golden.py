"""Record the reference's stacking, pick-and-place, training and reach goals, and ObjectStackGoal's goal distance, into
tests/golden/reference_goal_variants.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_goal_variants_golden.py`.  It imports
the reference on the mujoco_py shim (as tools/make_placement_golden.py does) and runs the reference's OWN functions on
generator instances over a minimal simulation stand-in:

- `ObjectStackGoal._sample_next_goal_positions` with fixed and shuffled block order (goals/object_stack_goal.py);
- `PickAndPlaceGoal._sample_next_goal_positions` (goals/pickandplace.py: ObjectStateGoal's grid-then-uniform goals, then
  `move_one_object_to_the_air`);
- `TrainStateGoal._sample_next_goal_positions` (goals/train_state.py: place_targets_with_goal_distance_ratio, then
  `move_one_object_to_the_air_with_restrictions`), with `np.random.choice` patched to the replay's `choice`;
- `ObjectReachGoal._sample_next_goal_positions` (goals/object_reach_goal.py), recording what it writes with set_object_pos;
- `ObjectStackGoal.goal_distance` / `is_object_grasped` on recorded object, goal and gripper states with pad contacts, and
  `RearrangeEnv._calculate_num_success` over thresholds that include the gripper_pos and grasped keys.

Random numbers come from the replay RandomState of tests/goal_variants_rng.py: placement draws as the placement kernel's, the
modifier's draws (random, scalar uniform, randint, the block-order shuffle, the tower's choice) as rg_goal_modify's.  Blocks
have 2 to 5 of 5 slots active; ycb cases use the library's recorded bounding boxes (tests/golden/reference_placement.json.gz)
with padded slots.  Every recorded placement succeeded (the reference returns its last rejected trial on failure, the kernel
zeros)."""
import gzip
import json
import logging
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
REF = os.environ.get("ROBOGYM_REFERENCE", "/root/reference")
for p in (os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests"), REF, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_goal_variants.json.gz")
PLACEMENT = os.path.join(ROOT, "tests", "golden", "reference_placement.json.gz")
TABLE = [1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2]          # rearrange scenes: table body pos, table geom half size


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def main():
    import robogym_b200.mujoco_py_shim as shim
    from goal_variants_rng import GoalVariantsReplayRandomState

    shim.install()
    logging.disable(logging.WARNING)
    import robogym.envs.rearrange.goals.object_state as osg
    import robogym.envs.rearrange.goals.train_state as ts
    from robogym.envs.rearrange.common.base import RearrangeEnv
    from robogym.envs.rearrange.goals.object_reach_goal import ObjectReachGoal
    from robogym.envs.rearrange.goals.object_stack_goal import ObjectStackGoal
    from robogym.envs.rearrange.goals.pickandplace import PickAndPlaceGoal
    from robogym.envs.rearrange.simulation.base import RearrangeSimulationInterface as RSI
    from robogym.utils import rotation

    table_pos, table_size = np.array(TABLE[:3]), np.array(TABLE[3:])
    ref_table = RSI.compute_table_dimension(table_pos.copy(), table_size.copy())

    class Sim:
        """what the goal generators read and write of a rearrange simulation"""
        max_placement_retry, max_placement_retry_per_object = 100, 20
        get_table_setting = RSI.get_table_setting

        def __init__(self, bbox, portion, anchor=None, ratio=1.0, object_size=0.0254, target_height=0.1):
            self.bbox, self.num_objects, self.used_table_portion = bbox, len(bbox), portion
            self.anchor, self.goal_distance_ratio, self.goal_distance_min = anchor, ratio, 0.06
            self.simulation_params = SimpleNamespace(object_size=object_size, target_height=target_height)
            self.written = None

        def get_object_bounding_boxes(self):
            return self.bbox.copy()

        def get_table_dimensions(self):
            return ref_table

        def get_placement_area(self):
            return RSI.get_placement_area(self)

        def get_object_pos(self):
            return self.anchor.copy()

        def set_object_pos(self, p):
            self.written = np.array(p)

    grid_valid = []
    orig_grid = osg.place_objects_in_grid

    def grid_spy(*a, **k):
        out = orig_grid(*a, **k)
        grid_valid.append(bool(out[1]))
        return out

    osg.place_objects_in_grid = grid_spy

    def generator(cls, sim, **attrs):
        g = object.__new__(cls)
        g.mujoco_simulation = sim
        for k, v in attrs.items():
            setattr(g, k, v)
        return g

    def run(kind, bbox, active, portion, seed, env, epoch, **kw):
        """one environment's goals by the reference generator of `kind`; None when its placement failed"""
        bbox, active = np.asarray(bbox, dtype=np.float64), np.asarray(active, dtype=bool)
        sel = np.nonzero(active)[0]
        nobj = len(bbox)
        anchor = None if kw.get("anchor") is None else np.asarray(kw["anchor"], dtype=np.float64)
        sim = Sim(bbox[sel], portion, None if anchor is None else anchor[sel], kw.get("ratio", 1.0), kw.get("object_size", 0.0254),
                  kw.get("target_height", 0.1))
        area = sim.get_placement_area()
        rs = GoalVariantsReplayRandomState(seed, env, epoch)
        grid_valid.clear()
        obj = None
        if kind == "stack":
            rs.shuffle = rs.modifier_shuffle          # the block-order shuffle is the modifier's; the bottom placement never shuffles
            pl, ok = ObjectStackGoal._sample_next_goal_positions(generator(ObjectStackGoal, sim, fixed_order=kw["fixed_order"]), rs)
            status = 2 if ok else 0
        elif kind == "pick_and_place":
            pl, ok = PickAndPlaceGoal._sample_next_goal_positions(generator(PickAndPlaceGoal, sim, height_range=kw["height_range"]), rs)
            status = (1 if grid_valid[0] else 2) if ok else 0
        elif kind == "train":
            args = SimpleNamespace(height_range=kw["height_range"], pickup_proba=kw["pickup"], stacking_proba=kw["stacking"])
            saved = np.random.choice
            np.random.choice = rs.choice
            try:
                pl, ok = ts.TrainStateGoal._sample_next_goal_positions(generator(ts.TrainStateGoal, sim, args=args), rs)
            finally:
                np.random.choice = saved
            status = 3 if ok else 0
        else:
            pl, ok = ObjectReachGoal._sample_next_goal_positions(generator(ObjectReachGoal, sim), rs)
            status = 2 if ok else 0
            obj = np.zeros((nobj, 3))
            obj[sel] = sim.written
        if not ok:
            return None
        pos = np.zeros((nobj, 3))
        pos[sel] = pl
        return dict(kind=kind, bbox=bbox.tolist(), active=active.astype(int).tolist(), area=list(area.offset) + list(area.size), portion=portion,
                    seed=seed, env=env, epoch=epoch, fixed_order=bool(kw.get("fixed_order", True)), height_range=list(kw.get("height_range", (0.0, 0.0))),
                    pickup=kw.get("pickup", 0.0), stacking=kw.get("stacking", 0.0), ratio=kw.get("ratio", 1.0), object_size=kw.get("object_size", 0.0),
                    target_height=kw.get("target_height", 0.0), anchor=None if anchor is None else anchor.tolist(), status=status, pos=pos.tolist(),
                    obj_pos=None if obj is None else obj.tolist(), draws=rs.modifier_draws)

    rng = np.random.RandomState(20261017)
    cases = []

    def add(kind, bbox, active, portion, **kw):
        """the case at the first seed whose placement succeeds"""
        for _ in range(20):
            c = run(kind, bbox, active, portion, int(rng.randint(1 << 31)), int(rng.randint(4096)), int(rng.randint(64)), **kw)
            if c is not None:
                cases.append(c)
                return c
        raise RuntimeError(f"no successful placement for {kind}")

    def block_boxes(n, size):
        return np.array([[np.zeros(3), np.full(3, size)]] * n)

    def anchor_for(bbox, active, portion):
        """object placements for the training goals: the reference's grid-then-uniform placement of the same objects"""
        c = run("pick_and_place", bbox, active, portion, int(rng.randint(1 << 31)), 0, 0, height_range=(0.0, 0.0))
        return np.array(c["pos"])

    ycb = [np.array(b["bbox"]) for b in json.loads(gzip.decompress(open(PLACEMENT, "rb").read()))["boxes"] if b["kind"] == "mesh"]
    ycb_active = []
    for k in range(len(ycb)):
        a = np.ones(8, dtype=bool)
        a[rng.choice(8, 4 + k, replace=False)] = False        # 4 and 3 of 8 active: the library's boxes crowd the area
        ycb_active.append(a)

    # stacking: blocks with 2 to 5 of 5 slots active (first slot inactive in some), both orders, several block sizes
    for n in (2, 3, 4, 5):
        for fixed in (True, False):
            for rep in range(2):
                active = np.zeros(5, dtype=bool)
                active[rng.choice(5, n, replace=False) if rep else np.arange(n)] = True
                add("stack", block_boxes(5, 0.0254), active, 1.0, fixed_order=fixed, object_size=float(rng.uniform(0.02, 0.05)))
    for k, (bb, a) in enumerate(zip(ycb, ycb_active)):
        add("stack", bb, a, 1.0, fixed_order=bool(k % 2), object_size=0.0254)
    # pick-and-place: blocks and ycb, default and custom height ranges
    for n in (2, 3, 4, 5):
        active = np.zeros(5, dtype=bool)
        active[rng.choice(5, n, replace=False)] = True
        for hr in ((0.05, 0.25), (0.1, 0.1)):
            add("pick_and_place", block_boxes(5, 0.025), active, float(rng.choice([1.0, 0.8])), height_range=hr)
    for bb, a in zip(ycb, ycb_active):
        add("pick_and_place", bb, a, 1.0, height_range=(0.05, 0.25))
    # training goals: every task mix, goal_distance_ratio 1 and below, blocks and ycb
    mixes = ((0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (0.3, 0.4))
    for pickup, stacking in mixes:
        for n in (2, 3, 4, 5):
            for ratio in (1.0, 0.5):
                active = np.zeros(5, dtype=bool)
                active[rng.choice(5, n, replace=False)] = True
                bb = block_boxes(5, 0.0254)
                add("train", bb, active, 1.0, anchor=anchor_for(bb, active, 1.0), ratio=ratio, pickup=pickup, stacking=stacking,
                    height_range=(0.05, 0.25), object_size=float(rng.uniform(0.02, 0.05)))
        for bb, a in zip(ycb, ycb_active):
            add("train", bb, a, 1.0, anchor=anchor_for(bb, a, 1.0), ratio=0.3, pickup=pickup, stacking=stacking, height_range=(0.0, 0.2),
                object_size=0.0254)
        # one active object: a stacking draw leaves it as placed
        one = np.zeros(5, dtype=bool)
        one[2] = True
        bb = block_boxes(5, 0.0254)
        add("train", bb, one, 1.0, anchor=anchor_for(bb, one, 1.0), ratio=0.7, pickup=pickup, stacking=stacking, height_range=(0.05, 0.25),
            object_size=0.0254)
    # reach: one block in any slot, several target heights
    for k in range(6):
        one = np.zeros(5, dtype=bool)
        one[k % 5] = True
        add("reach", block_boxes(5, float(rng.uniform(0.02, 0.05))), one, float(rng.choice([1.0, 0.6])), target_height=float(rng.uniform(0.0, 0.2)))

    # ObjectStackGoal.goal_distance on recorded states: object, goal and gripper positions, pad contacts
    class EvalSim:
        def __init__(self, n, nmax, contacts):
            self.object_groups = [SimpleNamespace(object_ids=[i]) for i in range(n)]
            self.num_groups = self.num_objects = n
            self.max_num_objects = nmax
            self.goal_pos_offset, self.goal_rot_weight = 0.0, 1.0
            self.contacts = contacts

        def get_object_gripper_contact(self):
            return self.contacts.copy()

    def state(pos, quat, n, nmax, normalize):
        p, r = np.zeros((nmax, 3)), np.zeros((nmax, 3))
        p[:n] = pos[:n]
        for i in range(n):
            e = rotation.mat2euler(rotation.quat2mat(quat[i]))
            r[i] = rotation.normalize_angles(e) if normalize else e
        return {"obj_pos": p, "obj_rot": r}

    top = TABLE[2] + TABLE[5]
    thresholds = [{"obj_pos": 0.04, "obj_rot": 0.2}, {"obj_pos": 0.04, "gripper_pos": 0.12}, {"obj_pos": 0.05, "grasped": 1.5},
                  {"gripper_pos": 0.1, "grasped": 1.0}, {"obj_pos": 0.04, "obj_rot": 0.3, "gripper_pos": 0.15, "grasped": 2.0}]
    evals = []
    for i, (n, nmax) in enumerate(((2, 2), (3, 5), (5, 5), (4, 8), (1, 3), (5, 5), (2, 6), (3, 3))):
        mode = ("full", "mod90", "mod180")[i % 3]
        gp = np.stack([rng.uniform(1.0, 1.6, n), rng.uniform(0.3, 1.2, n), top + 0.03 + 0.05 * np.arange(n)], -1)
        gq = rng.normal(size=(n, 4)); gq /= np.linalg.norm(gq, axis=1, keepdims=True)
        near = rng.rand(n) < 0.6
        op = np.where(near[:, None], gp + rng.normal(scale=0.02, size=gp.shape), gp + rng.normal(scale=0.2, size=gp.shape))
        oq = np.where(near[:, None], gq + rng.normal(scale=0.05, size=gq.shape), rng.normal(size=gq.shape))
        grip = op[rng.randint(n)] + rng.normal(scale=0.06, size=3)
        contacts = np.zeros((nmax, 2))                 # float 0 / 1 per pad, as get_object_gripper_contact returns them
        contacts[:n] = rng.rand(n, 2) < 0.4
        gp, gq, op, oq, grip = f32(gp), f32(gq), f32(op), f32(oq), f32(grip)
        sim = EvalSim(n, nmax, contacts)
        gen = ObjectStackGoal(sim, osg.GoalArgs(rot_dist_type=mode), fixed_order=True)
        goal = state(gp, gq, n, nmax, False)
        cur = state(op, oq, n, nmax, True)
        cur.update({"gripper_pos": np.array([grip]), "grasped": gen.is_object_grasped()})
        gd = gen.goal_distance(goal, cur)
        rel = gd.pop("relative_goal")
        nums = []
        for thr in thresholds:
            env = SimpleNamespace(constants=SimpleNamespace(success_threshold=thr, goal_reward_per_object=1.0))
            nums.append(float(RearrangeEnv._calculate_num_success(env, gd)))
        pad = lambda a, w: np.concatenate([a, np.zeros((nmax - n, w))])
        evals.append(dict(mode=mode, n=n, nmax=nmax, goal_pos=pad(gp, 3).tolist(), goal_quat=pad(gq, 4).tolist(), pos=pad(op, 3).tolist(),
                          quat=pad(oq, 4).tolist(), gripper=grip.tolist(), contacts=contacts.astype(int).tolist(), rel_pos=rel["obj_pos"].tolist(),
                          rel_gripper=rel["gripper_pos"].tolist(), dist_pos=gd["obj_pos"].tolist(), dist_rot=gd["obj_rot"].tolist(),
                          dist_gripper=gd["gripper_pos"].tolist(), grasped=np.asarray(gd["grasped"], dtype=np.float64).tolist(), num_success=nums))

    doc = dict(table=TABLE, cases=cases, evals=evals, thresholds=thresholds,
               source="robogym v1.0.0 goals/object_stack_goal.py, goals/pickandplace.py, goals/train_state.py, goals/object_reach_goal.py, "
                      "common/base.py _calculate_num_success; replay RandomState of tests/goal_variants_rng.py")
    with open(OUT, "wb") as f:
        f.write(gzip.compress(json.dumps(doc).encode(), mtime=0))
    kinds = {}
    for c in cases:
        kinds[c["kind"]] = kinds.get(c["kind"], 0) + 1
    print(f"{OUT}: {len(cases)} cases {kinds}, {len(evals)} goal-distance states")


if __name__ == "__main__":
    main()
