"""Record the reference's stabilize_objects into tests/golden/reference_settle.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_settle_golden.py`.  The unmodified
reference blocks environment runs on the mujoco_py shim with the fp64 oracle as engine (as tools/make_reference_goldens.py runs
it), with `stabilize_objects=False` so that its reset stops after the placement.  For a few seeds the tool stores the model (as
differences against the committed rearrange_blocks5_tcp asset), the state the reset left, the object dofs the reference's
get_object_damping selects, and the state after the reference's own `stabilize_objects(mujoco_simulation)`: damping 1e-3 on the
object dofs, 100 env-steps of nsubsteps mj_step each followed by a forward, the damping restored, a forward.
tests/test_settle.py replays the settle from the stored state and compares the objects' poses."""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_reference_goldens as R  # noqa: E402  (sets up sys.path for the reference, the stubs and the shim)

OUT = os.path.join(R.GOLDEN, "reference_settle.json.gz")
SEEDS = (0, 1, 2, 3)


def _case(seed, num_objects):
    from robogym.envs.rearrange.blocks import make_env
    from robogym.envs.rearrange.common.utils import stabilize_objects
    from robogym.robot.robot_interface import ControlMode, TcpSolverMode

    env = make_env(parameters=dict(n_random_initial_steps=0, simulation_params=dict(num_objects=num_objects, max_num_objects=5),
                                   robot_control_params=dict(control_mode=ControlMode.TCP_ROLL_YAW, tcp_solver_mode=TcpSolverMode.MOCAP_IK,
                                                             max_position_change=float(np.float32(0.1)))),
                   constants=dict(stabilize_objects=False), starting_seed=seed)
    env.reset()
    env = env.unwrapped
    sim = env.mujoco_simulation
    mj = sim.mj_sim
    m = mj.model
    dofs, qadr = [], []
    for i in range(sim.num_objects):
        j = m.joint_name2id(f"object{i}:joint")
        dofs += [d for d in range(m.nv) if m.dof_jntid[d] == j]
        qadr.append(int(m.jnt_qposadr[j]))
    damping0 = R._l(sim.get_object_damping())
    rec = dict(seed=seed, num_objects=int(sim.num_objects), model=R._model_diff(m._cm.blob(), "rearrange_blocks5_tcp"), nsub=int(mj.nsubsteps),
               n_steps=100, damping=1e-3, dofs=dofs, qposadr=qadr, object_damping=damping0, state0=R._sim_state(mj))
    stabilize_objects(sim)
    rec.update(qpos=R._l(mj.data.qpos), qvel=R._l(mj.data.qvel))
    assert R._l(sim.get_object_damping()) == damping0
    return rec


def main():
    R._engine()
    cases = [_case(s, 5) for s in SEEDS]
    with open(OUT, "wb") as f:      # mtime=0: the same record gives the same bytes
        f.write(gzip.compress(json.dumps(dict(cases=cases), separators=(",", ":")).encode(), compresslevel=9, mtime=0))
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
