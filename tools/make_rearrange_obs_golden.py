"""Record the reference's rearrange observations, placement masks, contact flags and simulation penalties into
tests/golden/reference_rearrange_obs.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_rearrange_obs_golden.py`.  The
unmodified reference environments run on the mujoco_py shim with the fp64 oracle as engine (as tools/make_reference_goldens.py
runs them); at every recorded env-step the tool

1. rounds every row rg_rearrange_obs reads (body poses and velocities, qpos, qvel, ctrl, sensordata, contact distances) to
   float32 and writes the rounded rows back into the shim's data, so the reference's functions see exactly what the kernel reads;
2. stores those rows, the goal (`_goal`) and the index tables the reference's own name lookups give;
3. stores the reference's `_observe_simple()`, `_get_simulation_info()`, `get_gripper_table_contact()` and the
   `_get_simulation_reward_with_done` reward and done.

Cases: blocks with 5 of 5 objects and with 3 of 5 (padded slots), the ycb environment with mask_obs_outside_placement_area, all
with non-zero penalties.  The arm is driven onto block 3 and then onto the table, so the record has finger-pad contacts on a slot
other than 0 and gripper-table contacts; object states are edited to put one object outside the placement area, one off the
table and one into the wrist camera's collision sphere; in the ycb case one goal is moved outside the placement area."""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
REF = os.environ["ROBOGYM_REFERENCE"]
for p in (os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests"), REF, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_rearrange_obs.json.gz")
PENALTY = dict(table_collision=0.5, wrist_collision=0.25, objects_off_table=2.0, safety_stop=0.125)
PREFIX = "robot0:"
GRIPPER_BODIES = ("robot0:gripper_base", "left_gripper", "left_inner_follower", "left_outer_driver", "right_gripper", "right_inner_follower",
                  "right_outer_driver")


def _l(x):
    return np.asarray(x, dtype=np.float64).ravel().tolist()


def _f32(x):
    return np.asarray(x, dtype=np.float32).astype(np.float64)


def _round_state(mj):
    """round the rows the kernel reads to float32, in place in the shim's data"""
    d = mj.data
    for name in ("qpos", "qvel", "ctrl", "sensordata", "body_xpos", "body_xquat", "body_xvelp", "body_xvelr"):
        a = getattr(d, name)
        a[...] = _f32(a)
    for i in range(d.ncon):
        d.contact[i].dist = float(np.float32(d.contact[i].dist))


def _tables(env):
    """index tables from the reference's own lookups"""
    from robogym.envs.rearrange.common.utils import geom_ids_of_body   # the lookup get_object_gripper_contact uses

    sim = env.mujoco_simulation
    mj = sim.mj_sim
    model = mj.model
    n, nmax = sim.num_objects, sim.max_num_objects
    ng = model.ngeom
    geom_body = np.asarray(model.geom_bodyid)
    gobj = np.full(ng, -1)
    for k in range(n):
        gobj[geom_ids_of_body(mj, f"object{k}")] = k
    gb = {model.body_name2id(b) for b in GRIPPER_BODIES}
    names = [model.geom_id2name(g) for g in range(ng)]
    flags = [(1 if int(geom_body[g]) in gb else 0) | (2 if names[g] is not None and names[g].startswith(PREFIX) else 0) for g in range(ng)]
    force, torque = model.sensor_name2id("toolhead_force"), model.sensor_name2id("toolhead_torque")
    return dict(nobj=nmax, num_objects=n, obj_body=[model.body_name2id(f"object{k}") for k in range(n)] + [0] * (nmax - n),
                obj_qpos=[model.get_joint_qpos_addr(f"object{k}:joint")[0] for k in range(n)] + [0] * (nmax - n),
                tcp_body=model.body_name2id(PREFIX + "gripper_tcp"), arm_qpos=list(map(int, sim.qpos_idxs[PREFIX + "arm_joint_angles"])),
                grip_qpos=list(map(int, sim.qpos_idxs[PREFIX + "gripper_joint_angles"])), grip_qvel=list(map(int, sim.qvel_idxs[PREFIX + "gripper_joint_angles"])),
                grip_act=int(model.actuator_name2id(PREFIX + "r_gripper_finger_joint")), force_adr=int(model.sensor_adr[force]),
                torque_adr=int(model.sensor_adr[torque]), geom_object=gobj.tolist(), geom_flags=flags,
                table_plane=model.geom_name2id("table_collision_plane"), wrist_sphere=model.geom_name2id(PREFIX + "wrist_cam_collision_sphere"),
                pad=[model.geom_name2id(PREFIX + "left_contact_v"), model.geom_name2id(PREFIX + "right_contact_v")],
                nbody=model.nbody, nq=model.nq, nv=model.nv, nu=model.nu, nsensordata=model.nsensordata, ngeom=ng)


def _record(env, note):
    from robogym.utils import rotation

    sim = env.mujoco_simulation
    mj = sim.mj_sim
    d = mj.data
    n, nmax = sim.num_objects, sim.max_num_objects
    goal = env._goal
    gp = np.asarray(goal["obj_pos"])
    # the goal quaternions: the target bodies' own, which get_target_rot turned into goal["obj_rot"] (checked)
    tq = np.zeros((nmax, 4))
    tq[:, 0] = 1.0
    for k in range(n):
        b = mj.model.body_name2id(f"target:object{k}")
        assert np.array_equal(d.body_xpos[b], gp[k]), "target moved"
        tq[k] = d.body_xquat[b]
        assert np.array_equal(rotation.mat2euler(d.get_body_xmat(f"target:object{k}")), goal["obj_rot"][k])
    _round_state(mj)
    # the qpos the goal was set on is a row the kernel reads too: round its entries outside the object joints (next_goal wrote
    # those from target_pos / target_rot, object_state.py:381-390)
    qg = np.asarray(goal["qpos_goal"])
    keep = np.zeros(len(qg), bool)
    for k in range(n):
        a = mj.model.get_joint_qpos_addr(f"object{k}:joint")[0]
        keep[a:a + 7] = True
    goal["qpos_goal"] = np.where(keep, qg, _f32(qg))
    obs = env._observe_simple()
    info = env._get_simulation_info()
    reward, done = env._get_simulation_reward_with_done(info)
    off = np.zeros(nmax, bool)
    off[:n] = info["objects_off_table"]
    rows = dict(body_xpos=_l(d.body_xpos), body_xquat=_l(d.body_xquat), body_xvel=_l(np.concatenate([d.body_xvelr, d.body_xvelp], 1)),
                qpos=_l(d.qpos), qvel=_l(d.qvel), ctrl=_l(d.ctrl), sensordata=_l(d.sensordata),
                contact=[[int(d.contact[i].geom1), int(d.contact[i].geom2), float(d.contact[i].dist), int(d.contact[i].dim)] for i in range(d.ncon)])
    # the reference's boxes follow each object's current rotation (get_block_bounding_box / get_mesh_bounding_box): the row the
    # kernel copies is set per step here
    return dict(note=note, rows=rows, bbox_size=_l(sim.get_object_bounding_box_sizes()), goal_pos=_l(gp), goal_quat=_l(tq), goal_rot=_l(goal["obj_rot"]), qpos_at_goal=_l(goal["qpos_goal"]),
                rel_pos=_l(obs["rel_goal_obj_pos"]), rel_rot=_l(obs["rel_goal_obj_rot"]), achieved=int(obs["is_goal_achieved"][0]),
                off_table=off.astype(int).tolist(), group=list(range(n)) + [-1] * (nmax - n),
                obs={k: _l(v) for k, v in obs.items()}, gripper_table=bool(sim.get_gripper_table_contact()),
                wrist_cam={k: bool(v) for k, v in info["wrist_cam_contacts"].items()}, objects_off_table=off.astype(int).tolist(),
                reward=float(reward), done=bool(done))


def _blocks(num_objects, max_num_objects, steps, grip_slot=0):
    from robogym.envs.rearrange.blocks import make_env
    from robogym.robot.robot_interface import ControlMode, TcpSolverMode

    env = make_env(parameters=dict(n_random_initial_steps=0, simulation_params=dict(num_objects=num_objects, max_num_objects=max_num_objects, penalty=PENALTY),
                                   robot_control_params=dict(control_mode=ControlMode.TCP_ROLL_YAW, tcp_solver_mode=TcpSolverMode.MOCAP_IK,
                                                             max_position_change=float(np.float32(0.1)))), starting_seed=3)
    env.reset()
    env = env.unwrapped
    sim = env.mujoco_simulation
    mj = sim.mj_sim
    # block `grip_slot` right under the tool: the fingers close on it, then go down onto the table
    tcp = mj.data.get_body_xpos("robot0:gripper_tcp").copy()
    adr = mj.model.get_joint_qpos_addr(f"object{grip_slot}:joint")[0]
    mj.data.qpos[adr:adr + 2] = tcp[:2]
    sim.forward()
    rec = dict(tables=_tables(env), penalty=PENALTY, mask_obs=bool(env.constants.mask_obs_outside_placement_area),
               mask_margin=float(env.constants.goal_args.mask_margin), boundary=_l(env._placement_area_boundary),
               bbox_size=_l(sim.get_object_bounding_box_sizes()), colors=_l(sim.get_object_colors()), steps=[])
    for k, a in enumerate(steps):
        env.step(np.asarray(a, dtype=np.float32))
        rec["steps"].append(_record(env, f"step {k}"))
    return env, rec


def _edits(env, rec, tag, wrist_slot):
    """object 1 pushed out of the placement area (still on the table), then object 2 off the table, then object `wrist_slot` into
    the wrist camera's collision sphere"""
    sim = env.mujoco_simulation
    mj = sim.mj_sim
    lo = np.asarray(env._placement_area_boundary)
    a1 = mj.model.get_joint_qpos_addr("object1:joint")[0]
    mj.data.qpos[a1] = lo[0] - 0.1
    sim.forward()
    rec["steps"].append(_record(env, f"{tag}: object 1 outside the placement area"))
    a2 = mj.model.get_joint_qpos_addr("object2:joint")[0]
    mj.data.qpos[a2 + 2] = 0.05
    sim.forward()
    rec["steps"].append(_record(env, f"{tag}: object 2 off the table"))
    aw = mj.model.get_joint_qpos_addr(f"object{wrist_slot}:joint")[0]
    mj.data.qpos[aw:aw + 3] = mj.data.get_geom_xpos(PREFIX + "wrist_cam_collision_sphere")
    sim.forward()
    rec["steps"].append(_record(env, f"{tag}: object {wrist_slot} in the wrist camera's sphere"))
    assert rec["steps"][-1]["wrist_cam"]["any"], tag


def _goal_outside_area(env):
    """target 0 moved 10 cm beyond the placement area's x minimum (still on the table), and the goal entries next_goal derives
    from the targets (object_state.py:359-404) recomputed with the reference's own functions"""
    from robogym.utils import rotation

    sim = env.mujoco_simulation
    mj = sim.mj_sim
    lo = np.asarray(env._placement_area_boundary)
    tp = sim.get_target_pos(pad=False).copy()
    tp[0, 0] = lo[0] - 0.1
    sim.set_target_pos(tp)
    sim.forward()
    g = env._goal
    g["obj_pos"] = sim.get_target_pos().copy()
    g["goal_objects_in_placement_area"] = sim.check_objects_in_placement_area(g["obj_pos"], margin=env.constants.goal_args.mask_margin,
                                                                              soft=env.constants.goal_args.soft_mask)
    g["obj_rot"] = sim.get_target_rot().copy()
    for i in range(sim.num_objects):
        a = mj.model.get_joint_qpos_addr(f"object{i}:joint")[0]
        g["qpos_goal"][a:a + 3] = g["obj_pos"][i]
        g["qpos_goal"][a + 3:a + 7] = rotation.euler2quat(g["obj_rot"][i])
    assert not g["goal_objects_in_placement_area"][0]


def main():
    import robogym_b200.mujoco_py_shim as shim

    shim.install()
    from oracle_engine import OracleEngine

    shim.set_engine_factory(OracleEngine)
    out = {}
    # down onto block 0 (open, then closing on it), up and away (open), then down until the fingers meet the table
    down = [[0, 0, -1, 0, 0, 1]] * 4 + [[0, 0, -1, 0, 0, -1]] * 4 + [[0, 1, 0.6, 0, 0, 1]] * 4 + [[0, 0, -1, 0, 0, 0]] * 14
    env, rec = _blocks(5, 5, down, grip_slot=3)
    _edits(env, rec, "blocks5", 4)
    out["blocks5"] = rec
    rng = np.random.RandomState(7)
    env, rec = _blocks(3, 5, rng.uniform(-1, 1, (4, 6)))
    _edits(env, rec, "blocks3of5", 0)
    out["blocks3of5"] = rec

    from robogym.envs.rearrange.ycb import make_env
    from robogym.robot.robot_interface import ControlMode, TcpSolverMode

    env = make_env(parameters=dict(n_random_initial_steps=0, simulation_params=dict(num_objects=4, max_num_objects=8, penalty=PENALTY),
                                   robot_control_params=dict(control_mode=ControlMode.TCP_ROLL_YAW, tcp_solver_mode=TcpSolverMode.MOCAP_IK,
                                                             max_position_change=float(np.float32(0.1)))),
                   constants=dict(stabilize_objects=False, mask_obs_outside_placement_area=True), starting_seed=1)
    env.reset()
    env = env.unwrapped
    sim = env.mujoco_simulation
    rec = dict(tables=_tables(env), penalty=PENALTY, mask_obs=True, mask_margin=float(env.constants.goal_args.mask_margin),
               boundary=_l(env._placement_area_boundary), bbox_size=_l(sim.get_object_bounding_box_sizes()), colors=_l(sim.get_object_colors()), steps=[])
    for k, a in enumerate(rng.uniform(-1, 1, (3, 6))):
        env.step(a.astype(np.float32))
        rec["steps"].append(_record(env, f"ycb step {k}"))
    _goal_outside_area(env)
    rec["steps"].append(_record(env, "ycb: goal 0 outside the placement area"))
    _edits(env, rec, "ycb", 3)
    out["ycb"] = rec

    out["source"] = ("robogym v1.0.0 envs/rearrange/common/base.py _observe_simple / _get_simulation_info / _get_simulation_reward_with_done, "
                     "simulation/base.py get_gripper_table_contact, on the mujoco_py shim with the fp64 oracle; rows rounded to float32")
    with open(OUT, "wb") as f:
        f.write(gzip.compress(json.dumps(out, separators=(",", ":"), default=lambda v: v.item()).encode(), compresslevel=9, mtime=0))
    for name in ("blocks5", "blocks3of5", "ycb"):
        st = out[name]["steps"]
        print(name, len(st), "steps; pad contacts", sum(any(x > 0 for x in s["obs"]["obj_gripper_contact"]) for s in st),
              "gripper-table", sum(s["gripper_table"] for s in st), "done", sum(s["done"] for s in st),
              "outside area", sum(0.0 in s["obs"].get("placement_mask", [1.0]) for s in st),
              "goal outside area", sum(0.0 in s["obs"].get("goal_placement_mask", [1.0]) for s in st), "wrist", sum(s["wrist_cam"]["any"] for s in st),
              "pad slots", sorted({k for s in st for k in range(len(s["obs"]["obj_gripper_contact"]) // 2) if max(s["obs"]["obj_gripper_contact"][2 * k:2 * k + 2]) > 0}))
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
