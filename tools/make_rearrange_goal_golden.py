"""Record the reference's rearrange goal evaluation and goal orientation sampling into tests/golden/reference_rearrange_goal.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_rearrange_goal_golden.py`.  It imports the
reference on the mujoco_py shim (as tools/make_placement_golden.py does) and runs the reference's OWN functions:

- `ObjectStateGoal.relative_goal` / `goal_distance` (robogym/envs/rearrange/goals/object_state.py) on a minimal simulation
  stand-in (num_objects, num_groups, object_groups, max_num_objects, goal_pos_offset, goal_rot_weight), with the current state
  as `get_object_pos` / `get_object_rot` and the goal as `get_target_pos` / `get_target_rot` build them from body poses
  (quat2mat of the body quaternion in place of body_xmat; zero padding);
- `RearrangeEnv._calculate_num_success`, `RearrangeEnv._calculate_goal_distance_reward` (envs/rearrange/common/base.py),
  `RobotEnv._is_successful` (robot_env.py) and `RearrangeSimulationInterface.check_objects_off_table`;
- `randomize_quaternion_along_z` / `randomize_quaternion_block` with the replay RandomState of tests/goal_rng.py
  (GoalRotReplayRandomState), whose draws are the goal-orientation kernel's Philox counters.

Every case evaluates two object states against one goal: the first as the first evaluation after a goal reset (reward 0),
the second against the first.  Inputs are float32-representable, so float32 pose rows carry them exactly.  Besides the
reference's outputs the tool records, per slot, the goal the greedy matching gave the object and the parallel quaternion the
rotation distance took, each with its margin (the gap to the runner-up), and each distance's gap to its threshold, so that a
test can tell a decision that last-bit differences may flip from one they may not."""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
REF = os.environ.get("ROBOGYM_REFERENCE", "/root/reference")
for p in (os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests"), REF, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_rearrange_goal.json.gz")
TABLE = [1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2]          # rearrange scenes: table body pos, table geom half size
THRESHOLD = {"obj_pos": 0.04, "obj_rot": 0.2}


def f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def main():
    import robogym_b200.mujoco_py_shim as shim
    from goal_rng import GoalRotReplayRandomState

    shim.install()
    import robogym.envs.rearrange.goals.object_state as osg
    from robogym.envs.rearrange.common.base import RearrangeEnv
    from robogym.envs.rearrange.simulation.base import RearrangeSimulationInterface as RSI
    from robogym.robot_env import RobotEnv
    from robogym.utils import rotation

    table_pos, table_size = np.array(TABLE[:3]), np.array(TABLE[3:])
    ref_table = RSI.compute_table_dimension(table_pos.copy(), table_size.copy())

    class Group:
        def __init__(self, ids):
            self.object_ids = ids

    class Sim:
        """what relative_goal, goal_distance, check_objects_off_table and the goal orientation samplers read"""

        def __init__(self, groups, max_num_objects, offset=0.0, weight=1.0, target_quat=None):
            self.object_groups = [Group(g) for g in groups]
            self.num_groups = len(groups)
            self.num_objects = sum(len(g) for g in groups)
            self.max_num_objects = max_num_objects
            self.goal_pos_offset, self.goal_rot_weight = offset, weight
            self.target_quat = target_quat

        def get_table_dimensions(self):
            return ref_table

        def get_target_quat(self, pad=True):
            assert not pad
            return self.target_quat.copy()

        check_objects_off_table = RSI.check_objects_off_table

    class Constants:
        def __init__(self, thr, reward):
            self.success_threshold, self.goal_reward_per_object = thr, reward

    class Env:
        def __init__(self, thr, reward):
            self.constants = Constants(thr, reward)

        _calculate_num_success = RearrangeEnv._calculate_num_success

    def state(pos, quat, n, nmax, normalize):
        """get_object_pos / get_object_rot (normalize) or get_target_pos / get_target_rot, zero-padded to nmax"""
        p, r = np.zeros((nmax, 3)), np.zeros((nmax, 3))
        p[:n] = pos[:n]
        for i in range(n):
            e = rotation.mat2euler(rotation.quat2mat(quat[i]))
            r[i] = rotation.normalize_angles(e) if normalize else e
        return {"obj_pos": p, "obj_rot": r}

    def decisions(goal, cur, sim, mode):
        """per object slot: (matched goal slot, its margin, parallel quaternion, its margin) -- the greedy rounds and the argmin
        over the parallel quaternions restated here to find their runner-ups (checked against the reference's outputs)"""
        n = sim.num_objects
        match, mmargin = list(range(sim.max_num_objects)), [np.inf] * sim.max_num_objects
        if sim.num_objects != sim.num_groups:
            for g in sim.object_groups:
                ids = g.object_ids
                if len(ids) == 1:
                    continue
                d = np.linalg.norm(cur["obj_pos"][ids][:, None] - goal["obj_pos"][ids][None], axis=-1)
                for _ in ids:
                    flat = np.argmin(d, axis=None)
                    i, j = np.unravel_index(flat, d.shape)
                    rest = np.delete(d.ravel(), flat)
                    rest = rest[np.isfinite(rest)]
                    match[ids[i]], mmargin[ids[i]] = ids[j], float(rest.min() - d[i, j]) if len(rest) else np.inf
                    d[i, :] = np.inf
                    d[:, j] = np.inf
        pick, pmargin = [-1] * sim.max_num_objects, [np.inf] * sim.max_num_objects
        if mode != "full":
            pq = osg.PARALLEL_QUATS if mode == "mod90" else osg.PARALLEL_QUATS_180
            for k in range(n):
                q1 = rotation.euler2quat(goal["obj_rot"][match[k]])
                q2 = rotation.euler2quat(cur["obj_rot"][k])
                if np.allclose(q1, q2):
                    continue
                dists = rotation.quat_magnitude(np.array([rotation.quat_difference(rotation.quat_mul(q1, p), q2) for p in pq]))
                pick[k] = int(np.argmin(dists))
                pmargin[k] = float(np.sort(dists)[1] - dists[pick[k]])
        return match, mmargin, pick, pmargin

    def evaluate(case):
        g, nmax = case["groups"], case["nmax"]
        sim = Sim(g, nmax, case["offset"], case["weight"])
        n = sim.num_objects
        gen = osg.ObjectStateGoal(sim, osg.GoalArgs(rot_dist_type=case["mode"]))
        env = Env(case["threshold"], case["reward_per_object"])
        goal = state(np.array(case["goal_pos"]), np.array(case["goal_quat"]), n, nmax, False)
        out, prev = [], None
        for st in case["states"]:
            cur = state(np.array(st["pos"]), np.array(st["quat"]), n, nmax, True)
            gd = gen.goal_distance(goal, cur)
            rel = gd.pop("relative_goal")
            if prev is None:
                prev = gd
            reward = RearrangeEnv._calculate_goal_distance_reward(env, prev, gd)
            prev = gd
            num = RearrangeEnv._calculate_num_success(env, gd)
            succ = np.all(np.stack([gd[k] < case["threshold"][k] for k in case["threshold"]]), axis=0)
            off = np.zeros(nmax, bool)
            off[:n] = sim.check_objects_off_table(np.array(st["pos"])[:n])
            match, mm, pick, pm = decisions(goal, cur, sim, case["mode"])
            # the restated decisions reproduce the reference's relative goal exactly
            for k in range(n):
                assert np.array_equal(rel["obj_pos"][k], goal["obj_pos"][match[k]] - cur["obj_pos"][k]), (case["name"], k)
            out.append(dict(obj_rot=cur["obj_rot"].tolist(), rel_pos=rel["obj_pos"].tolist(), rel_rot=rel["obj_rot"].tolist(),
                            dist_pos=gd["obj_pos"].tolist(), dist_rot=gd["obj_rot"].tolist(), success=succ.astype(int).tolist(),
                            num_success=float(num), achieved=bool(RobotEnv._is_successful(env, gd)), reward=float(reward),
                            off_table=off.astype(int).tolist(), any_off=bool(off.any()), match=match, match_margin=mm, pick=pick,
                            pick_margin=pm, pos_gap=(gd["obj_pos"] - case["threshold"].get("obj_pos", np.nan)).tolist(),
                            rot_gap=(gd["obj_rot"] - case["threshold"].get("obj_rot", np.nan)).tolist()))
        return out

    rng = np.random.RandomState(20261016)
    top = TABLE[2] + TABLE[5]

    def rand_quat(n):
        q = rng.normal(size=(n, 4))
        return q / np.linalg.norm(q, axis=1, keepdims=True)

    def yaw_quat(a):
        return np.stack([np.cos(0.5 * a), 0 * a, 0 * a, np.sin(0.5 * a)], -1)

    def on_table(n):
        return np.stack([rng.uniform(1.0, 1.6, n), rng.uniform(0.3, 1.2, n), np.full(n, top + 0.03)], -1)

    cases = []

    def add(name, mode, groups, nmax, goal_pos, goal_quat, states, offset=0.0, weight=1.0, threshold=THRESHOLD, reward_per_object=1.0):
        n = sum(len(g) for g in groups)
        pad = lambda a, w: np.concatenate([np.asarray(a, dtype=np.float64)[:n], np.zeros((nmax - n, w))])
        c = dict(name=name, mode=mode, groups=groups, nmax=nmax, offset=float(f32(offset)), weight=float(f32(weight)), threshold=dict(threshold),
                 reward_per_object=reward_per_object, goal_pos=f32(pad(goal_pos, 3)).tolist(), goal_quat=f32(pad(goal_quat, 4)).tolist(),
                 states=[dict(pos=f32(pad(p, 3)).tolist(), quat=f32(pad(q, 4)).tolist()) for p, q in states])
        c["table"] = TABLE
        c["out"] = evaluate(c)
        cases.append(c)

    def near(gp, gq, dpos, drot, n):
        """object states around the goals: positions dpos away in a random direction, rotations drot about a random axis"""
        d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
        ax = rng.normal(size=(n, 3)); ax /= np.linalg.norm(ax, axis=1, keepdims=True)
        dq = np.concatenate([np.cos(0.5 * drot)[:, None], np.sin(0.5 * drot)[:, None] * ax], 1)
        return gp + d * np.asarray(dpos)[:, None], rotation.quat_mul(dq, gq)

    modes = ("full", "mod90", "mod180")
    # distinct objects, random poses and poses near their goals, with and without padding
    for mode in modes:
        for n, nmax in ((5, 5), (3, 8), (1, 4)):
            groups = [[i] for i in range(n)]
            gp, gq = on_table(n), rand_quat(n)
            s1 = (on_table(n), rand_quat(n))
            s2 = near(gp, gq, rng.uniform(0, 0.06, n), rng.uniform(0, 0.3, n), n)
            add(f"distinct-{mode}-{n}of{nmax}", mode, groups, nmax, gp, gq, [s1, s2])
    # duplicates: groups of 2 to 5 mixed with singletons, objects near permuted goals
    layouts = [[[0, 1], [2], [3]], [[0], [1, 2, 3], [4]], [[0, 1, 2, 3], [4], [5, 6]], [[0, 1, 2, 3, 4]], [[0], [1], [2, 3, 4, 5, 6], [7]]]
    for mode in modes:
        for li, groups in enumerate(layouts):
            n = sum(len(g) for g in groups)
            nmax = n + (li % 2) * 2
            gp, gq = on_table(n), yaw_quat(rng.uniform(-np.pi, np.pi, n))
            perm = np.arange(n)
            for g in groups:
                perm[g] = rng.permutation(g)
            p2, q2 = near(gp[perm], gq[perm], rng.uniform(0, 0.05, n), rng.uniform(0, 0.25, n), n)
            add(f"groups-{mode}-{li}", mode, groups, nmax, gp, gq, [(on_table(n), rand_quat(n)), (p2, q2)])
    # goal_pos_offset and goal_rot_weight, with padding (padded slots at max(offset, 0))
    for mode in modes:
        for off, w in ((-0.02, 0.5), (0.01, 0.0), (-0.04, 1.0), (0.05, 0.75)):
            n, nmax = 4, 6
            gp, gq = on_table(n), rand_quat(n)
            add(f"offset-{mode}-{off}-{w}", mode, [[0, 1], [2], [3]], nmax, gp, gq,
                [near(gp, gq, rng.uniform(0, 0.08, n), rng.uniform(0, 0.4, n), n), near(gp, gq, rng.uniform(0, 0.03, n), rng.uniform(0, 0.1, n), n)],
                offset=off, weight=w)
    # just inside and just outside both thresholds: positions along x, rotations about z
    for mode in modes:
        n = 4
        gp, gq = on_table(n), yaw_quat(rng.uniform(-0.5, 0.5, n))
        for eps in (-2e-5, 2e-5):
            dp = np.array([0.04 + eps, 0.0, 0.0, 0.04 + eps])
            dr = np.array([0.0, 0.2 + 10 * eps, 0.2 + 10 * eps, 0.0])
            p = gp + np.stack([dp, 0 * dp, 0 * dp], -1)
            q = rotation.quat_mul(yaw_quat(dr), gq)
            add(f"threshold-{mode}-{eps}", mode, [[i] for i in range(n)], n, gp, gq, [(gp, gq), (p, q)])
        for thr in ({"obj_pos": 0.04}, {"obj_rot": 0.2}):
            p = gp + np.array([0.05, 0, 0])
            add(f"one-key-{mode}-{sorted(thr)[0]}", mode, [[i] for i in range(n)], n, gp, gq, [(gp, gq), (p, gq)], threshold=thr, reward_per_object=2.5)
    # objects off each table edge and below 0.75 x table height
    lo, hi = table_pos - table_size, table_pos + table_size
    for mode in ("full", "mod90"):
        n = 6
        gp, gq = on_table(n), rand_quat(n)
        p = gp.copy()
        p[0, 0] = lo[0] - 1e-3; p[1, 0] = hi[0] + 1e-3; p[2, 1] = lo[1] - 1e-3; p[3, 1] = hi[1] + 1e-3; p[4, 2] = 0.75 * top - 1e-3
        p2 = gp.copy()
        p2[:, 0] = lo[0] + 1e-3; p2[5, 2] = 0.75 * top + 1e-3
        add(f"off-table-{mode}", mode, [[0, 1], [2], [3], [4], [5]], 8, gp, gq, [(p2, gq), (p, gq)])
    # rotations at exact 90 / 180 degree multiples: several parallel quaternions tie
    exact = np.array([[0.5, 0.5, 0.5, 0.5], [0.0, 0.0, 0.0, 1.0], [0.0, 1.0, 0.0, 0.0], [0.5, -0.5, 0.5, -0.5], [1.0, 0.0, 0.0, 0.0],
                      [0.0, 0.0, 1.0, 0.0]])
    for mode in modes:
        n = len(exact)
        gp = on_table(n)
        gq = np.tile([1.0, 0.0, 0.0, 0.0], (n, 1))
        pq = np.array(osg.PARALLEL_QUATS)[rng.randint(0, 24, n)]
        add(f"exact-{mode}", mode, [[i] for i in range(n)], n, gp, gq, [(gp, exact), (gp, rotation.quat_mul(gq, pq))])
        add(f"exact-yaw-{mode}", mode, [[0, 1, 2], [3, 4, 5]], n, gp, yaw_quat(np.array([0, 0.5, 1, 1.5, 2, 2.5]) * np.pi),
            [(gp[[1, 0, 2, 3, 5, 4]], exact), (gp, yaw_quat(np.array([1, 0.5, 0, -0.5, 2, 1]) * np.pi))])

    # goal orientations: randomize_quaternion_along_z / randomize_quaternion_block
    rots = []
    for mode, fn in (("z_axis", osg.randomize_quaternion_along_z), ("block", osg.randomize_quaternion_block)):
        for k, n in enumerate((1, 3, 5, 8)):
            base = f32(rand_quat(n) if k % 2 else yaw_quat(rng.uniform(-np.pi, np.pi, n)))
            seed, env, epoch = int(rng.randint(1 << 31)), int(rng.randint(4096)), int(rng.randint(64))
            rs = GoalRotReplayRandomState(seed, env, epoch)
            q = fn(Sim([[i] for i in range(n)], n, target_quat=base), rs)
            angle = GoalRotReplayRandomState(seed, env, epoch).uniform(low=0.0, high=2.0 * np.pi, size=n)
            face = GoalRotReplayRandomState(seed, env, epoch).randint(low=0, high=24, size=n)
            rots.append(dict(mode=mode, base=base.tolist(), seed=seed, env=env, epoch=epoch, quat=np.asarray(q).tolist(), angle=angle.tolist(),
                             face=face.tolist() if mode == "block" else None))

    doc = dict(table=TABLE, cases=cases, rotations=rots, parallel_quats=np.array(osg.PARALLEL_QUATS).tolist(),
               parallel_quats_180=np.array(osg.PARALLEL_QUATS_180).tolist(),
               source="robogym v1.0.0 goals/object_state.py ObjectStateGoal.relative_goal / goal_distance, randomize_quaternion_along_z / "
                      "randomize_quaternion_block; common/base.py _calculate_num_success / _calculate_goal_distance_reward; robot_env.py "
                      "_is_successful; simulation/base.py check_objects_off_table; replay RandomState of tests/goal_rng.py")
    with open(OUT, "wb") as f:
        f.write(gzip.compress(json.dumps(doc).encode(), mtime=0))
    ties = sum(1 for c in cases for o in c["out"] for m in o["pick_margin"] if m <= 1e-9)
    print(f"{OUT}: {len(cases)} cases, {len(rots)} orientation draws, {ties} slots whose parallel quaternion ties")


if __name__ == "__main__":
    main()
