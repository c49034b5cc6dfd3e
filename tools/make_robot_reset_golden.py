"""Record the reference's robot reset into tests/golden/reference_robot_reset.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_robot_reset_golden.py`.  The unmodified
reference blocks environment runs on the mujoco_py shim with the fp64 oracle as engine (as tools/make_reference_goldens.py runs
it).  Its `_initialize_sim_state` and `_randomize_robot_initial_position` are wrapped on the instance, not changed: the tool
records both simulations' state before and after `_initialize_sim_state`, the state before `_randomize_robot_initial_position`,
the action (`action_space.sample` returns the Philox replay draw of tests/robot_reset_rng.py for environment `env` of `seed`,
epoch 0, as the placement fixtures replay their RandomState), and both simulations' qpos, ctrl and mocap pose after the held
steps and after every tenth zero-action step.  Cases: TCP_ROLL_YAW with arm_reset_controller_error True and False, TCP_WRIST,
and n_random_initial_steps 0, 1 and 10.  tests/test_robot_reset.py replays them on the fp64 stand-ins, and
tests/test_robot_reset_gpu.py on CUDA."""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_reference_goldens as R  # noqa: E402  (sets up sys.path for the reference, the stubs and the shim)

OUT = os.path.join(R.GOLDEN, "reference_robot_reset.json.gz")
SEED = 2024
CASES = [("TCP_ROLL_YAW", True, 10, 0), ("TCP_ROLL_YAW", False, 10, 1), ("TCP_WRIST", True, 10, 2), ("TCP_ROLL_YAW", True, 1, 3), ("TCP_ROLL_YAW", True, 0, 4)]


def _poses(mj):
    d = mj.data
    out = dict(qpos=R._l(d.qpos), ctrl=R._l(d.ctrl))
    if mj.model.nmocap:
        out.update(mocap_pos=R._l(d.mocap_pos), mocap_quat=R._l(d.mocap_quat))
    return out


def _case(mode, rce, n_random, env_index):
    from robogym.envs.rearrange.blocks import make_env
    from robogym.robot.robot_interface import ControlMode, TcpSolverMode
    from robot_reset_rng import ReplayActionSpace

    env = make_env(parameters=dict(n_random_initial_steps=n_random, simulation_params=dict(num_objects=5, max_num_objects=5),
                                   robot_control_params=dict(control_mode=getattr(ControlMode, mode), tcp_solver_mode=TcpSolverMode.MOCAP_IK,
                                                             arm_reset_controller_error=rce, max_position_change=float(np.float32(0.1)))),
                   starting_seed=env_index)
    u = env.unwrapped
    rec = dict(mode=mode, reset_controller_error=rce, n_random_initial_steps=n_random, seed=SEED, env=env_index, epoch=0)
    sims = lambda: (u.mujoco_simulation.mj_sim, u.robot.robots[0].controller_arm.mj_sim)     # rebuilt by every _recreate_sim
    init0, rand0 = u._initialize_sim_state, u._randomize_robot_initial_position

    def initialize():
        main, solver = sims()
        rec["init_before"] = dict(main=R._sim_state(main), solver=R._sim_state(solver))
        init0()
        rec["init_after"] = dict(main=R._sim_state(main), solver=R._sim_state(solver))

    def randomize():
        main, solver = sims()
        rec.update(nsub_main=int(main.nsubsteps), nsub_solver=int(solver.nsubsteps),
                   main_model=R._model_diff(main.model._cm.blob(), "rearrange_blocks5_tcp"),
                   solver_model=R._model_diff(solver.model._cm.blob(), "rearrange_solver_arm"),
                   before=dict(main=R._sim_state(main), solver=R._sim_state(solver)), after=[])
        u.action_space = ReplayActionSpace(u.action_space, SEED, env_index, 0)
        step0, count = u.mujoco_simulation.step, [0]

        def step():
            step0()
            count[0] += 1
            k = count[0] - n_random              # zero-action steps taken
            if count[0] == n_random or (k > 0 and k % 10 == 0):
                rec["after"].append(dict(step=count[0], main=_poses(main), solver=_poses(solver)))

        u.mujoco_simulation.step = step
        try:
            rand0()
        finally:
            u.mujoco_simulation.step = step0
            u.action_space = u.action_space.space
        rec["action"] = R._l(ReplayActionSpace(u.action_space, SEED, env_index, 0).sample())
        rec["n_main_steps"] = count[0]

    u._initialize_sim_state, u._randomize_robot_initial_position = initialize, randomize
    env.reset()
    return rec


def main():
    R._engine()
    cases = [_case(*c) for c in CASES]
    with open(OUT, "wb") as f:      # mtime=0: the same record gives the same bytes
        f.write(gzip.compress(json.dumps(dict(cases=cases), separators=(",", ":")).encode(), compresslevel=9, mtime=0))
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
