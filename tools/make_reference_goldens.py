"""Record what the tests compare against from the ORIGINAL robogym code into tests/golden/reference_*.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_reference_goldens.py`.  The unmodified
reference environments, wrappers and helpers run on the mujoco_py shim with the fp64 oracle as engine, exactly as the tests used to
drive them live; what they return (observations, rewards, tracker statistics, perturbed model ranges, noisy observations, contact
queries, controller trajectories) is stored beside the inputs that produced it, so the tests replay the comparison without the
reference.  Models are stored as differences against the committed assets (robogym_b200/assets), never as new blobs."""
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

GOLDEN = os.path.join(ROOT, "tests", "golden")
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
OBS_KEYS = ("cube_pos", "cube_quat", "hand_angle", "fingertip_pos", "goal_quat", "qpos_goal", "qpos", "qvel")


def _l(x):
    return np.asarray(x, dtype=np.float64).ravel().tolist()


def _model_diff(blob, asset):
    """fields of `blob` that differ from the committed asset (same dimensions and names required)"""
    from robogym_b200 import modelblob

    a_blob = open(os.path.join(ASSETS, asset + ".rgm"), "rb").read()
    m, a = modelblob.unpack(blob), modelblob.unpack(a_blob)
    assert all(m[d] == a[d] for d in modelblob.DIMS), asset
    assert modelblob.unpack_names(blob) == modelblob.unpack_names(a_blob), asset
    return {k: m[k].tolist() for _, k, _ in modelblob.ARRAYS if not np.array_equal(m[k], a[k])}


def _sim_state(mj):
    from robogym_b200 import modelblob

    d = mj.data
    w = modelblob.pid_stride(mj.model._m) * mj.model.nu
    st = dict(qpos=_l(d.qpos), qvel=_l(d.qvel), ctrl=_l(d.ctrl), pid=_l(d.userdata[:w]), warm=_l(d.qacc_warmstart))
    if mj.model.nmocap:
        st.update(mocap_pos=_l(d.mocap_pos), mocap_quat=_l(d.mocap_quat))
    st.update(body_xpos=_l(d.body_xpos), body_xquat=_l(d.body_xquat))
    return st


def _engine():
    import robogym_b200.mujoco_py_shim as shim

    shim.install()
    from oracle_engine import OracleEngine

    shim.set_engine_factory(OracleEngine)


# ---------------------------------------------------------------- dactyl/locked (tests/test_locked_env.py, test_randomization.py, test_batched_facade.py)
def locked():
    from robogym.envs.dactyl.common import cube_utils
    from robogym.envs.dactyl.locked import make_simple_env

    out = dict(parallel_quats=np.asarray(cube_utils.PARALLEL_QUATS).tolist())

    # step logic: goal successes, a new-goal draw and a per-goal timeout
    consts = dict(max_timesteps_per_goal=6, successes_needed=2)
    env = make_simple_env(starting_seed=5, constants=consts)
    env.reset()
    d = env.mujoco_simulation.mj_sim.data
    tr = env.multi_goal_tracker
    rot = env.mujoco_simulation.qpos_idxs["cube_rotation"]
    rec = dict(constants=consts, state0=_sim_state(env.mujoco_simulation.mj_sim), goal_quat=_l(env._goal["cube_quat"]),
               prev_dist=float(env._previous_goal_distance["cube_quat"]),
               tracker=dict(steps_since_last_goal=int(tr._steps_since_last_goal), consecutive_success=int(tr._consecutive_steps_with_success),
                            successes_so_far=int(tr._successes_so_far), goals_so_far=int(tr._goals_so_far), success_pending=bool(tr._success_and_no_goal_reset)),
               steps=[])
    rng = np.random.RandomState(1)
    for k in range(16):
        st = {}
        if k in (2, 6):   # put the goal on top of the current orientation: the next step succeeds
            q = d.qpos[rot].copy()
            env._goal["cube_quat"] = q
            env._goal["qpos_goal"][rot] = q
            st["goal_override"] = _l(q)
        a = rng.uniform(-1, 1, 20)
        obs, rew, done, info = env.step(a)
        st.update(action=_l(a), new_goal=_l(env._goal["cube_quat"]), obs={key: _l(obs[key]) for key in OBS_KEYS},
                  is_goal_achieved=float(np.asarray(obs["is_goal_achieved"]).ravel()[0]), reward=_l(rew), done=bool(done),
                  goal_dist=float(info["goal_dist"]["cube_quat"]), goal_reset=bool(info.get("goal_reset", False)),
                  **{key: int(info[key]) for key in ("successes_so_far", "goals_so_far", "steps_since_last_goal")},
                  **{key: bool(info[key]) for key in ("trial_success", "sub_goal_is_successful")})
        rec["steps"].append(st)
        if done:
            break
    out["step_logic"] = rec

    consts = dict(max_timesteps_per_goal=3, successes_needed=2)
    env = make_simple_env(starting_seed=2, constants=consts)
    env.reset()
    rec = dict(constants=consts, state0=_sim_state(env.mujoco_simulation.mj_sim), goal_quat=_l(env._goal["cube_quat"]),
               prev_dist=float(env._previous_goal_distance["cube_quat"]), goals_so_far=int(env.multi_goal_tracker._goals_so_far), reward=[], done=[])
    for k in range(3):
        _, rew, done, info = env.step(np.zeros(20))
        rec["reward"].append(_l(rew)); rec["done"].append(bool(done))
    out["timeout"] = rec

    # InitialStatePool.randomize vs LockedEnv._randomize_cube_initial_position
    env = make_simple_env(starting_seed=11)
    rec = []
    for nrand in (1, 10):
        env.parameters.n_random_initial_steps = nrand
        for seed in (3, 4):
            env._random_state.seed(seed)
            env.mujoco_simulation.reset()
            env._randomize_cube_initial_position()
            d = env.mujoco_simulation.mj_sim.data
            rec.append(dict(n_random_initial_steps=nrand, seed=seed, qpos=_l(d.qpos), qvel=_l(d.qvel), on_palm=bool(env.mujoco_simulation.is_cube_on_palm())))
    out["reset_randomisation"] = rec
    out["action_latency"] = _action_latency()
    out["range_rules"] = _range_rules()
    return out


def _action_latency():
    from robogym.envs.dactyl.locked import make_simple_env
    from robogym.wrappers import randomizations as rz

    inner = make_simple_env(starting_seed=3)
    performed = []
    real_step = inner.step

    def spy(action):
        performed.append(np.array(action, copy=True))
        return real_step(action)

    inner.step = spy
    w = rz.RandomizedActionLatency(inner, max_delay=2)
    w.reset()
    rec = dict(max_delay=2, action_delay=[int(x) for x in np.asarray(w._action_delay)], steps=[])
    rng = np.random.RandomState(0)
    for k in range(6):
        a = rng.uniform(-1, 1, 20)
        obs, _, _, _ = w.step(a)
        rec["steps"].append(dict(action=_l(a), performed=_l(performed[-1]), action_history=_l(obs["action_history"]),
                                 action_delay=[int(x) for x in np.asarray(obs["action_delay"]).ravel()]))
    return rec


def _range_rules():
    """joint-limit / control-range and tendon-range perturbation by the reference wrappers' own _set_field, normal draws of seeds 0..2"""
    from robogym.envs.dactyl.locked import make_simple_env
    from robogym.wrappers import randomizations as rz

    env = make_simple_env(starting_seed=0)
    sim = env.unwrapped.sim
    nj = len(list(sim.model.joint_names))          # the wrapper's default: every joint
    nt = int(sim.model.ntendon)
    jw = rz.RandomizedJointLimitWrapper(env)
    tw = rz.RandomizedTendonRangeWrapper(env)
    jw._orig_value = np.array(jw._get_field(sim), copy=True)
    tw._orig_value = np.array(tw._get_field(sim), copy=True)
    rec = []
    for seed in (0, 1, 2):
        r = np.random.RandomState(seed)
        zj, zt = r.randn(nj, 2), r.randn(nt, 2)
        jw._random_noises = lambda n, z=zj: z
        jw._set_field(sim)
        env.unwrapped._random_state = type("R", (), {"randn": staticmethod(lambda *s, z=zt: z)})()
        tw._set_field(sim)
        rec.append(dict(seed=seed, jnt_range=_l(sim.model.jnt_range), actuator_ctrlrange=_l(sim.model.actuator_ctrlrange), tendon_range=_l(sim.model.tendon_range)))
    return rec


def facade():
    """robogym's own per-env host code (denormalisation, observations, on-palm test, occlusion) along 12 steps of make_env(starting_seed=3)"""
    from robogym.envs.dactyl.locked import make_env
    from robogym.utils.sensor_utils import check_occlusion

    env = make_env(starting_seed=3)
    env.reset()
    env = env.unwrapped
    sim = env.mujoco_simulation.mj_sim
    robot = env.mujoco_simulation.shadow_hand
    rec = dict(model=_model_diff(sim.model._cm.blob(), "dactyl_locked"), steps=[])
    rng = np.random.RandomState(0)
    for k in range(12):
        action = rng.uniform(-1, 1, 20)
        st = dict(action=_l(action), qpos_before=_l(sim.data.qpos),
                  want_rel=_l(robot.denormalize_position_control(action, relative_action=True)),
                  want_abs=_l(robot.denormalize_position_control(action, relative_action=False)))
        robot.set_position_control(np.asarray(st["want_rel"]))
        env.mujoco_simulation.step()
        obs = env.observe()
        d = sim.data
        st.update(qpos=_l(d.qpos), qvel=_l(d.qvel), site_xpos=_l(d.site_xpos), actuator_force=_l(d.actuator_force),
                  obs={key: _l(obs[key]) for key in ("cube_pos", "cube_quat", "hand_angle", "fingertip_pos")},
                  actuator_effort=_l(robot.observe().actuator_effort()), on_palm=bool(env.mujoco_simulation.is_cube_on_palm()),
                  contacts=[[int(d.contact[i].geom1), int(d.contact[i].geom2), float(d.contact[i].dist), int(d.contact[i].dim)] for i in range(d.ncon)],
                  occluded=[int(x) for x in np.asarray(check_occlusion(sim, dist_cutoff=-1e-4))])
        rec["steps"].append(st)
    return rec


def full_perpendicular():
    """the reference builds dactyl/full_perpendicular on the shim; five zero-action steps from its reset state on the oracle"""
    from robogym.envs.dactyl.full_perpendicular import make_simple_env

    env = make_simple_env(starting_seed=0)
    ms = env.mujoco_simulation
    cm = ms.mj_sim.model._cm
    rec = dict(dims={k: int(cm.m[k]) for k in ("nq", "nv", "nu", "njnt", "ntendon", "nbody")}, model=_model_diff(cm.blob(), "dactyl_full_perpendicular"))
    ms.reset()
    ms.forward()
    rec["state0"] = _sim_state(ms.mj_sim)
    rec["nsubsteps"] = int(ms.mj_sim.nsubsteps)
    ctrl = []
    for _ in range(5):
        ms.shadow_hand.set_position_control(ms.shadow_hand.denormalize_position_control(np.zeros(20)))
        ctrl.append(_l(ms.mj_sim.data.ctrl))
        ms.step()
    d = ms.mj_sim.data
    rec.update(ctrl=ctrl, qpos=_l(d.qpos), qvel=_l(d.qvel), ncon=int(d.ncon), on_palm=bool(ms.is_cube_on_palm()))
    return rec


# ---------------------------------------------------------------- dactyl/reach (tests/test_reach_env.py)
REACH_OBS_KEYS = ("qpos", "qvel", "fingertip_pos", "goal_fingertip_pos", "is_goal_achieved")


def _count_calls(mj, counts):
    """count mj_step / mj_forward calls of one MjSim in `counts` (mujoco-py's PID state advances in each)"""
    for name in ("step", "forward"):
        real = getattr(mj, name)

        def spy(*a, _real=real, _name=name, **kw):
            counts[_name] += 1
            return _real(*a, **kw)

        setattr(mj, name, spy)


def reach():
    """ReachEnv (make_simple_env) with small tracker constants: both simulations after the build, every RandomState.normal draw of
    FingertipPosGoal.next_goal with the goal it produced, an episode reset, forced successes, a trial success, a timeout, the
    mj_step / mj_forward counts of both simulations per phase, FingerSeparationWrapper's jnt_range for every active_finger, and
    which model arrays reach's randomisation stack changes on which simulation"""
    from robogym.envs.dactyl.goals.shadow_hand_reach_fingertip_pos import FingertipPosGoal
    from robogym.envs.dactyl.reach import make_env, make_simple_env
    from robogym.wrappers import dactyl as dw

    draws = []
    real_next_goal = FingertipPosGoal.next_goal

    class Normal:
        def __init__(self, rs):
            self.rs = rs

        def normal(self, loc, scale):
            v = self.rs.normal(loc=loc, scale=scale)
            draws.append(dict(loc=_l(loc), scale=_l(scale), normal=_l(v)))
            return v

    def next_goal(self, random_state, current_state):
        if not draws:
            out["goal_build"] = _sim_state(self.goal_simulation.mj_sim)
        goal = real_next_goal(self, Normal(random_state), current_state)
        draws[-1].update(fingertip_pos=_l(goal["fingertip_pos"]), goal_joint_pos=_l(self.goal_joint_pos), goal_state=_sim_state(self.goal_simulation.mj_sim))
        return goal

    out = {}
    FingertipPosGoal.next_goal = next_goal
    try:
        consts = dict(max_timesteps_per_goal=6, successes_needed=2)
        env = make_simple_env(starting_seed=5, constants=consts)
        ms, gs = env.mujoco_simulation, env.goal_generation.goal_simulation
        main_n, goal_n = dict(step=0, forward=0), dict(step=0, forward=0)
        _count_calls(ms.mj_sim, main_n)
        _count_calls(gs.mj_sim, goal_n)
        tr = env.multi_goal_tracker
        out.update(constants=consts, main_build=_sim_state(ms.mj_sim), nsubsteps=int(ms.mj_sim.nsubsteps),
                   goal_joint_pos0=draws[0]["loc"], goal_margin_added=_l(gs.mj_sim.model.geom_margin - ms.mj_sim.model.geom_margin),
                   success_steps_required_built=int(tr._success_steps_required), success_threshold=float(env.constants.success_threshold["fingertip_pos"]),
                   relative_action=bool(env.constants.relative_action), success_reward=float(env.constants.success_reward))

        def counts():
            c = dict(main=dict(main_n), goal=dict(goal_n))
            for d in (main_n, goal_n):
                d.update(step=0, forward=0)
            return c

        def tracker():
            return dict(steps_since_last_goal=int(tr._steps_since_last_goal), consecutive_success=int(tr._consecutive_steps_with_success),
                        successes_so_far=int(tr._successes_so_far), goals_so_far=int(tr._goals_so_far), success_pending=bool(tr._success_and_no_goal_reset),
                        success_steps_required=int(tr._success_steps_required))

        def record_reset():
            n0 = len(draws)
            counts()
            obs = env.reset()
            return dict(draws=list(range(n0, len(draws))), calls=counts(), main_state=_sim_state(ms.mj_sim), goal_state=_sim_state(gs.mj_sim),
                        obs={k: _l(obs[k]) for k in REACH_OBS_KEYS}, goal=_l(env._goal["fingertip_pos"]), prev_dist=float(env._previous_goal_distance["fingertip_pos"]),
                        tracker=tracker(), success_pause_range_s=list(env.constants.success_pause_range_s))

        out["draws_at_construction"] = len(draws)
        out["reset"] = record_reset()
        steps = []
        rng = np.random.RandomState(1)
        episode_ends = 0
        for k in range(40):
            st = {}
            if k in (1, 4):     # the goal put on the current fingertips: the next step succeeds
                cur = env.goal_generation.current_state()["fingertip_pos"].copy()
                env._goal["fingertip_pos"] = cur
                st["goal_override"] = _l(cur)
            a = rng.uniform(-1, 1, 20) * 0.3
            n0 = len(draws)
            obs, rew, done, info = env.step(a)
            st.update(action=_l(a), draws=list(range(n0, len(draws))), calls=counts(), obs={key: _l(obs[key]) for key in REACH_OBS_KEYS},
                      reward=_l(rew), done=bool(done), goal_dist=float(info["goal_dist"]["fingertip_pos"]), goal_reset=bool(info.get("goal_reset", False)),
                      goal_achieved=bool(info["goal_achieved"]), main_state=_sim_state(ms.mj_sim),
                      **{key: int(info[key]) for key in ("successes_so_far", "goals_so_far", "steps_since_last_goal")},
                      **{key: bool(info[key]) for key in ("trial_success", "sub_goal_is_successful")})
            steps.append(st)
            if done:
                episode_ends += 1
                if episode_ends == 2:
                    break
                st["reset"] = record_reset()
        out["steps"] = steps
        out["draws"] = draws[:]
    finally:
        FingertipPosGoal.next_goal = real_next_goal

    # FingerSeparationWrapper: jnt_range of the main simulation after the wrapper's reset, per active finger
    env = make_simple_env(starting_seed=0)
    jr0 = env.sim.model.jnt_range.copy()
    out["jnt_range0"] = _l(jr0)
    out["active_finger"] = {}
    for finger in ("TH", "FF", "MF", "RF", "LF", "WR"):
        env.sim.model.jnt_range[:] = jr0
        dw.FingerSeparationWrapper(env, active_finger=finger).reset()
        out["active_finger"][finger] = dict(main=_l(env.sim.model.jnt_range), goal=_l(env.goal_generation.goal_simulation.mj_sim.model.jnt_range))
    env.sim.model.jnt_range[:] = jr0

    # reach's randomisation stack (make_env(randomize=True)): which model arrays change on the main and on the goal simulation
    from robogym_b200 import modelblob

    env = make_env(starting_seed=0, constants=dict(randomize=True))
    inner = env.unwrapped
    mm, gm = inner.mujoco_simulation.mj_sim.model._cm, inner.goal_generation.goal_simulation.mj_sim.model._cm
    before = (modelblob.unpack(mm.blob()), modelblob.unpack(gm.blob()))
    env.reset()
    after = (modelblob.unpack(mm.blob()), modelblob.unpack(gm.blob()))
    out["randomized_fields"] = {side: sorted(k for _, k, _ in modelblob.ARRAYS if not np.array_equal(b[k], a[k]))
                                for side, b, a in zip(("main", "goal"), before, after)}
    w, chain = env, []
    while hasattr(w, "env"):
        chain.append(type(w).__name__)
        w = w.env
    out["wrappers"] = chain
    return out


# ---------------------------------------------------------------- observation noise (tests/test_obs_noise.py)
class _Recorder:
    """numpy RandomState look-alike that logs what it hands out"""

    def __init__(self, seed):
        self.rs, self.log = np.random.RandomState(seed), []

    def randn(self, *shape):
        v = self.rs.randn(*shape); self.log.append(("randn", v.copy())); return v

    def uniform(self, lo, hi, size=None):
        v = self.rs.uniform(lo, hi, size=size); self.log.append(("uniform", v.copy())); return v


def obs_noise():
    """the reference's RandomizeObservationWrapper with locked.py's levels on a minimal environment that serves the clean
    observations of tests/test_obs_noise.py, its random state recording every draw"""
    from collections import OrderedDict

    import gym
    from gym.spaces import Box, Dict

    import test_obs_noise as T
    from robogym.wrappers.randomizations import RandomizeObservationWrapper
    from robogym_b200.obs_noise import LOCKED_LEVELS

    clean = T.clean_observations()

    class FakeEnv(gym.Env):
        def __init__(self, e):
            self.e, self.k = e, 0
            self._random_state = _Recorder(100 + e)
            self.observation_space = Dict({k: Box(-np.inf, np.inf, (w,), np.float64) for k, w in T.WIDTHS.items()})
            self.action_space = Box(-1, 1, (1,), np.float64)

        @property
        def unwrapped(self):
            return self

        def reset(self):
            self.k = 0
            return OrderedDict((k, v.copy()) for k, v in clean[0][self.e].items())

        def step(self, a):
            self.k += 1
            return OrderedDict((k, v.copy()) for k, v in clean[self.k][self.e].items()), 0.0, False, {}

    envs = [RandomizeObservationWrapper(FakeEnv(e), levels=LOCKED_LEVELS) for e in range(T.NENV)]
    ref = [[w.reset() for w in envs]]
    for s in range(T.NSTEPS):
        ref.append([w.step(np.zeros(1))[0] for w in envs])
    return dict(draws=[[[kind, _l(v)] for kind, v in w.unwrapped._random_state.log] for w in envs],
                noisy=[[{k: _l(o["noisy_" + k]) for k in T.WIDTHS} for o in row] for row in ref])


# ---------------------------------------------------------------- rearrange (tests/test_rearrange_arm.py, test_rearrange_contacts.py)
def _rearrange_env(reset_controller_error, wrist=False):
    from robogym.envs.rearrange.blocks import make_env
    from robogym.robot.robot_interface import ControlMode, TcpSolverMode

    env = make_env(parameters=dict(n_random_initial_steps=0, simulation_params=dict(num_objects=5),
                                   robot_control_params=dict(control_mode=ControlMode.TCP_WRIST if wrist else ControlMode.TCP_ROLL_YAW, tcp_solver_mode=TcpSolverMode.MOCAP_IK,
                                                             arm_reset_controller_error=reset_controller_error,
                                                             max_position_change=float(np.float32(0.1)))), starting_seed=0)
    env.reset()
    return env.unwrapped


def _two_sims(env, main_asset, solver_asset):
    main_mj = env.mujoco_simulation.mj_sim
    solver_mj = env.robot.robots[0].controller_arm.mj_sim
    return main_mj, solver_mj, dict(main_model=_model_diff(main_mj.model._cm.blob(), main_asset), solver_model=_model_diff(solver_mj.model._cm.blob(), solver_asset),
                                    nsub_main=int(main_mj.nsubsteps), nsub_solver=int(solver_mj.nsubsteps),
                                    main0=_sim_state(main_mj), solver0=_sim_state(solver_mj))


def rearrange():
    out = {}
    # TCP_WRIST: one tool rotation, the commanded orientation re-aligned with the vertical every step
    env = _rearrange_env(True, wrist=True)
    main_mj, solver_mj, rec = _two_sims(env, "rearrange_blocks5_tcp", "rearrange_solver_arm")
    rec.update(controller_arm=type(env.robot.robots[0].controller_arm).__name__, action_dim=int(env.action_space.shape[0]), actions=[], main_qpos=[], solver_qpos=[], solver_mocap_quat=[])
    rng = np.random.RandomState(1)
    for k in range(8):
        a = rng.uniform(-1, 1, 5).astype(np.float32)
        env.step(a)
        rec["actions"].append([float(x) for x in a])
        rec["main_qpos"].append(_l(main_mj.data.qpos)); rec["solver_qpos"].append(_l(solver_mj.data.qpos)); rec["solver_mocap_quat"].append(_l(solver_mj.data.mocap_quat))
    out["wrist"] = rec

    # BASELINE configs[4]: the ycb environment (8 mesh objects of its own draw)
    from robogym.envs.rearrange.ycb import make_env
    from robogym.robot.robot_interface import ControlMode, TcpSolverMode

    env = make_env(parameters=dict(n_random_initial_steps=0, simulation_params=dict(num_objects=8, max_num_objects=8),
                                   robot_control_params=dict(control_mode=ControlMode.TCP_ROLL_YAW, tcp_solver_mode=TcpSolverMode.MOCAP_IK,
                                                             max_position_change=float(np.float32(0.1)))),
                   constants=dict(stabilize_objects=False), starting_seed=1)
    env.reset()
    env = env.unwrapped
    main_mj, solver_mj, rec = _two_sims(env, "rearrange_ycb8_tcp", "rearrange_solver_arm")
    rec.update(actions=[], main_qpos=[], solver_qpos=[])
    rng = np.random.RandomState(2)
    for k in range(5):
        a = rng.uniform(-1, 1, 6).astype(np.float32)
        env.step(a)
        rec["actions"].append([float(x) for x in a])
        rec["main_qpos"].append(_l(main_mj.data.qpos)); rec["solver_qpos"].append(_l(solver_mj.data.qpos))
    out["ycb"] = rec

    # contact queries: block 0 put under the tool, the gripper driven onto it and then onto the table
    env = _rearrange_env(True)
    sim = env.mujoco_simulation
    mj = sim.mj_sim
    rec = dict(model=_model_diff(mj.model._cm.blob(), "rearrange_blocks5_tcp"), steps=[])
    tcp = mj.data.get_body_xpos("robot0:gripper_tcp").copy()
    adr = mj.model.get_joint_qpos_addr("object0:joint")[0]
    mj.data.qpos[adr:adr + 2] = tcp[:2]
    sim.forward()
    for k in range(26):
        a = np.zeros(6, dtype=np.float32)
        if k < 8:
            a[2] = -1.0                      # straight down onto the block
            a[5] = 1.0 if k < 4 else -1.0    # open, then close on it
        elif k < 12:
            a[2], a[1], a[5] = 0.6, 1.0, 1.0  # up and away from the blocks, open
        else:
            a[2] = -1.0                      # down until the fingers meet the table
        env.step(a)
        d = mj.data
        rec["steps"].append(dict(contacts=[[int(d.contact[i].geom1), int(d.contact[i].geom2), float(d.contact[i].dist)] for i in range(d.ncon)],
                                 gripper_table=bool(sim.get_gripper_table_contact()),
                                 wrist_cam={n: bool(v) for n, v in sim.get_wrist_cam_collisions().items()},
                                 object_gripper=np.asarray(sim.get_object_gripper_contact(pad=False)).astype(int).tolist()))
    out["contacts"] = rec
    return out


def main():
    _engine()
    for name, fn in (("reference_locked", locked), ("reference_facade", facade), ("reference_full_perpendicular", full_perpendicular),
                     ("reference_obs_noise", obs_noise), ("reference_rearrange", rearrange), ("reference_reach", reach)):
        if len(sys.argv) > 1 and name not in sys.argv[1:]:      # optional: regenerate only the named fixtures
            continue
        rec = fn()
        path = os.path.join(GOLDEN, name + ".json.gz")
        with open(path, "wb") as f:      # mtime=0: the same record gives the same bytes
            f.write(gzip.compress(json.dumps(rec, separators=(",", ":")).encode(), compresslevel=9, mtime=0))
        print(name, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
