"""Batched dactyl/reach environment (robogym_b200/reach_env.py): build, goal draws on the goal simulation, goal reward, multi-goal
bookkeeping, episode reset without a simulation reset, FingerSeparationWrapper's ranges and reach's randomisation stack -- against
what the reference's own ReachEnv returned when driven through the mujoco_py shim (tests/golden/reference_reach.json.gz, written by
tools/make_reference_goldens.py), on the CPU oracle simulator, and on the CUDA engine (gpu)."""
import json
import os
import sys

import numpy as np
import pytest

from helpers import reference_golden

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "stubs"))
OBS_KEYS = ("qpos", "qvel", "fingertip_pos", "goal_fingertip_pos", "is_goal_achieved")
TRACKER = ("steps_since_last_goal", "consecutive_success", "successes_so_far", "goals_so_far", "success_pending")


@pytest.fixture(scope="module")
def ref():
    return reference_golden("reach")


@pytest.fixture(scope="module")
def reach_asset():
    blob = open(os.path.join(ROOT, "robogym_b200", "assets", "dactyl_reach.rgm"), "rb").read()
    names = json.load(open(os.path.join(ROOT, "robogym_b200", "assets", "dactyl_reach.names.json")))
    return blob, names


def cpu_env(reach_asset, nenv, factory=None, **kw):
    import torch

    from oracle_batched_sim import OracleBatchedSim
    from robogym_b200.reach_env import BatchedReachEnv

    blob, names = reach_asset
    return BatchedReachEnv(factory or OracleBatchedSim, blob, names, nenv, torch.device("cpu"), **kw)


def _t(v):
    import torch

    return torch.as_tensor(np.asarray(v, dtype=np.float64))


def _load(sim, st, e=0):
    sim.qpos[e] = _t(st["qpos"]); sim.qvel[e] = _t(st["qvel"]); sim.ctrl[e] = _t(st["ctrl"])
    sim.pid[e] = _t(st["pid"]); sim.qacc_warmstart[e] = _t(st["warm"])


def _state_err(sim, st, e=0):
    return max(float((sim.qpos[e] - _t(st["qpos"])).abs().max()), float((sim.qvel[e] - _t(st["qvel"])).abs().max()) * 1e-3,
               float((sim.pid[e] - _t(st["pid"])).abs().max()))


def _noise(ref, draws):
    """the standard-normal draws behind the reference's RandomState.normal(loc, scale) calls"""
    if not draws:
        return None
    d = ref["draws"][draws[0]]
    assert len(draws) == 1
    return ((np.asarray(d["normal"]) - np.asarray(d["loc"])) / np.asarray(d["scale"]))[None]


def test_build_and_goal_draws_match_reference(ref, reach_asset):
    """Both simulations after ReachSimulation.build, and the chain of goals FingertipPosGoal.next_goal drew from them (the
    constructor's draw, the reset's, a new goal after a success, the next episode's) from the reference's normal draws: goal
    fingertips, settled goal_joint_pos and the goal simulation's state, which carries over from draw to draw."""
    import torch

    env = cpu_env(reach_asset, 1, **ref["constants"])
    assert ref["draws_at_construction"] == 1 and env.goal_launches == 3
    assert _state_err(env.sim, ref["main_build"]) < 1e-9
    assert _state_err(env.sim, ref["goal_build"]) < 1e-9         # the goal simulation is built like the main one
    hand = env.fac.hand_qpos_idx.numpy()
    assert np.array_equal(np.asarray(ref["main_build"]["qpos"])[hand], np.asarray(ref["goal_joint_pos0"]))   # the first draw's centre
    _load(env.goal_sim, ref["goal_build"])
    env.goal_joint_pos[0] = _t(ref["goal_joint_pos0"])
    mask = torch.ones(1, dtype=torch.bool)
    for k, d in enumerate(ref["draws"]):
        assert np.abs(env.goal_joint_pos[0].numpy() - np.asarray(d["loc"])).max() < 1e-7, k
        scale = 0.1 * (env.joint_hi - env.joint_lo)
        assert np.abs(scale.numpy() - np.asarray(d["scale"])).max() < 1e-12, k
        env._draw_goals(mask, _t(_noise(ref, [k])))
        assert np.abs(env.goal[0].numpy() - np.asarray(d["fingertip_pos"])).max() < 1e-7, k
        assert np.abs(env.goal_joint_pos[0].numpy() - np.asarray(d["goal_joint_pos"])).max() < 1e-7, k
        assert _state_err(env.goal_sim, d["goal_state"]) < 1e-7, k
    assert len(ref["draws"]) == 4


def test_step_logic_matches_reference(ref, reach_asset):
    """Same build, goals and actions -> same observations, reward terms, done flags, tracker statistics and main-simulation
    states (PID state included, so the same number of forward passes) as robogym's ReachEnv, through an episode reset without a
    simulation reset, two forced successes (a new goal, then a trial success), the auto-reset that follows, and a per-goal timeout."""
    assert ref["success_steps_required_built"] == 1 and ref["reset"]["tracker"]["success_steps_required"] == 1
    assert ref["reset"]["success_pause_range_s"] == [0.0, 0.5]      # set after the tracker copied (0, 0): still one step
    assert (ref["success_threshold"], ref["success_reward"], ref["relative_action"]) == (0.025, 5.0, True)
    env = cpu_env(reach_asset, 1, **ref["constants"])
    _load(env.goal_sim, ref["draws"][0]["goal_state"])
    env.goal_joint_pos[0] = _t(ref["draws"][0]["goal_joint_pos"])

    def check_reset(rec, obs):
        assert rec["calls"]["main"] == {"step": 0, "forward": 2}
        assert _state_err(env.sim, rec["main_state"]) < 1e-7
        assert _state_err(env.goal_sim, rec["goal_state"]) < 1e-7
        assert np.abs(env.goal[0].numpy() - np.asarray(rec["goal"])).max() < 1e-7
        assert abs(float(env.prev_dist[0]) - rec["prev_dist"]) < 1e-7
        for key in TRACKER:
            assert int(getattr(env, key)[0]) == int(rec["tracker"][key]), key
        for key in OBS_KEYS:
            assert np.abs(obs[key][0].numpy().ravel() - np.asarray(rec["obs"][key])).max() < 1e-7, key

    assert ref["reset"]["main_state"]["qpos"] == ref["main_build"]["qpos"]     # the reference does not reset the simulation
    check_reset(ref["reset"], env.reset(goal_noise=_noise(ref, ref["reset"]["draws"])))
    seen = dict(success=0, newgoal=0, timeout=0, trial=0, resets=0)
    for k, st in enumerate(ref["steps"]):
        if "goal_override" in st:
            env.goal[0] = _t(st["goal_override"])
        rs = st.get("reset", {})
        assert st["calls"]["main"] == {"step": 1, "forward": 3 + 2 * len(st["draws"])}
        mo, mr, md, mi = env.step(np.asarray(st["action"])[None], goal_noise=_noise(ref, st["draws"] + rs.get("draws", [])))
        assert np.abs(mr[0].numpy() - np.asarray(st["reward"])).max() < 1e-7, (k, st["reward"], mr)
        assert bool(md[0]) == st["done"] and abs(float(mi["goal_dist"][0]) - st["goal_dist"]) < 1e-7, k
        assert bool(mi["goal_achieved"][0]) == st["goal_achieved"] and bool(mi["goal_reset"][0]) == st["goal_reset"], k
        for key in ("successes_so_far", "goals_so_far", "steps_since_last_goal"):
            assert int(mi[key][0]) == st[key], (k, key)
        for key in ("trial_success", "sub_goal_is_successful"):
            assert bool(mi[key][0]) == st[key], (k, key)
        if rs:                          # auto-reset: the state and observation after the reference's env.reset()
            check_reset(rs, mo)
            seen["resets"] += 1
        elif not st["done"]:            # (the recording ends with the timeout's step, before its reset)
            assert _state_err(env.sim, st["main_state"]) < 1e-7, k
            for key in OBS_KEYS:
                assert np.abs(mo[key][0].numpy().ravel() - np.asarray(st["obs"][key])).max() < 1e-7, (k, key)
        seen["success"] += st["sub_goal_is_successful"]; seen["newgoal"] += st["goal_reset"]
        seen["timeout"] += st["done"] and not st["trial_success"]; seen["trial"] += st["trial_success"]
    assert seen == dict(success=2, newgoal=1, timeout=1, trial=1, resets=1), seen
    assert env.episodes == 3 and ref["steps"][-1]["done"]


def test_active_finger_matches_finger_separation_wrapper(ref, reach_asset):
    """FingerSeparationWrapper's jnt_range for every active_finger, on the main AND the goal simulation (the goal generator copies
    the main ranges before every draw), as a model edit; the goal simulation's margins are the reference's + 0.002."""
    from robogym_b200.reach_env import FINGERS

    assert sorted(ref["active_finger"]) == sorted(FINGERS)
    for finger, want in ref["active_finger"].items():
        env = cpu_env(reach_asset, 1, active_finger=finger, build_steps=1)
        assert np.array_equal(env.model["jnt_range"], np.asarray(want["main"])), finger
        assert np.array_equal(env.goal_model["jnt_range"], np.asarray(want["goal"])), finger
        for sim, m in ((env.sim, env.model), (env.goal_sim, env.goal_model)):     # what the simulators were built from
            for field in ("jnt_range", "geom_margin"):
                assert np.array_equal(np.asarray(sim.om.field(field)).ravel(), m[field]), (finger, field)
        lo, hi = env.joint_lo.numpy(), env.joint_hi.numpy()
        assert (hi >= lo).all() and int(((hi - lo) < 0.0100001).sum()) >= 12, finger       # the frozen joints
    assert np.array_equal(env.goal_model["geom_margin"] - env.model["geom_margin"], np.asarray(ref["goal_margin_added"]))
    with pytest.raises(ValueError):
        cpu_env(reach_asset, 1, active_finger="XX", build_steps=1)


WRAPPER_OF_RULE = dict(body_inertia="RandomizedBodyInertiaWrapper", robot_friction="RandomizedRobotFrictionWrapper",
                       gravity="RandomizedGravityWrapper", phasespace="RandomizedPhasespaceFingersWrapper", robot_damping="RandomizedRobotDampingWrapper",
                       robot_kp="RandomizedRobotKpWrapper")


def test_reach_randomiser_applies_reachs_rules_to_the_main_simulation_only(ref, reach_asset):
    """reach.py's stack (the model wrappers of make_env(randomize=True)) and nothing else: the arrays it draws are the ones the
    reference's stack changed on the main simulation -- no derived constants, as reach's reset never calls set_constants(); the
    timestep changes per step; cube rules drop out on a model without a cube; the goal simulation keeps the nominal model."""
    import torch

    from oracle_batched_sim import OracleBatchedSim
    from robogym_b200 import modelblob
    from robogym_b200.locked_env import TorchRand
    from robogym_b200.randomization import LOCKED_RULES, REACH_RULES, LockedRandomizer

    wrappers = [w for w in ref["wrappers"] if w.startswith("Randomized") and w != "RandomizedActionLatency"]
    assert sorted(wrappers) == sorted([WRAPPER_OF_RULE[r] for r in REACH_RULES] + ["RandomizedTimestepWrapper"])   # per step: the environment
    assert "RandomizedActionLatency" in ref["wrappers"] and "RandomizeObservationWrapper" in ref["wrappers"]
    blob, names = reach_asset
    m = modelblob.unpack(blob)
    rand = TorchRand(torch, torch.device("cpu"), 0, torch.float64)
    rz = LockedRandomizer(m, names, rand, torch, torch.device("cpu"), torch.float64, rules=REACH_RULES)
    params = rz.sample(3)
    assert set(params) == set(ref["randomized_fields"]["main"])        # no set_constants(): the derived constants stay nominal
    assert ref["randomized_fields"]["goal"] == []
    assert LockedRandomizer(m, names, rand, torch, torch.device("cpu"), torch.float64, rules=LOCKED_RULES).rules == tuple(r for r in LOCKED_RULES if r not in ("cube_friction", "cube_size"))

    class ParamSim(OracleBatchedSim):           # records the per-environment rows the environment writes
        def set_param(self, name, values, idx=None):
            self._params = getattr(self, "_params", {})
            if idx is None:
                self._params[name] = torch.as_tensor(values).clone()
            else:
                self._params[name][idx] = values

        def enable_per_env_timestep(self):
            self.timestep = torch.full((self.nenv,), float(self.om.field("opt_timestep")[0]), dtype=torch.float64)
            return self.timestep

    env = cpu_env(reach_asset, 3, factory=ParamSim, randomize=True, max_timesteps_per_goal=2)
    obs = env.reset()
    assert set(env.sim._params) == set(params) and not hasattr(env.goal_sim, "_params")
    assert not hasattr(env.goal_sim, "timestep") or env.goal_sim.timestep is None
    assert float(env.sim._params["opt_gravity"].std(dim=0).min()) > 0
    assert obs["noisy_fingertip_pos"].shape == (3, 15) and obs["action_delay"].shape == (3, 20)
    assert float((obs["noisy_fingertip_pos"] - obs["fingertip_pos"]).abs().max()) < 0.02
    g0 = env.sim._params["dof_damping"].clone()
    ts0, moved = float(env.sim.timestep[0]), 0
    for _ in range(2):
        _, _, done, _ = env.step(np.zeros((3, 20)))
        # RandomizedTimestepWrapper: a new timestep every step; a restarted episode begins at the nominal one
        assert bool((env.sim.timestep[~done] != ts0).all()) and bool((env.sim.timestep[done] == ts0).all())
        moved += int((~done).sum())
    assert moved == 3 and env.episodes == 6 and not torch.equal(env.sim._params["dof_damping"], g0)       # restarted episodes got new parameters


# ---------------------------------------------------------------- GPU tier
@pytest.mark.gpu
def test_cuda_env_matches_oracle_env_teacher_forced(reach_asset):
    """The CUDA environment beside the same environment on the fp64 oracle, 64 environments, teacher-forced (before every step the
    CUDA side receives the oracle side's states of both simulations, goal_joint_pos and bookkeeping; both get the same actions and
    the same goal draws).  No cube: the fp32/fp64 gap is round-off, as in test_reach_model.py."""
    import torch

    from robogym_b200 import build
    from robogym_b200.reach_env import STATE_FIELDS, make_cuda_env

    build.build()
    n, steps = 64, 30
    kw = dict(max_timesteps_per_goal=5, successes_needed=2, success_threshold=0.05)
    ref = cpu_env(reach_asset, n, seed=5, **kw)
    env = make_cuda_env(n, seed=5, **kw)
    rng = np.random.RandomState(0)
    noise = rng.randn(n, 24)
    ref.reset(goal_noise=noise)
    env.reset(goal_noise=noise)
    book = ("goal", "goal_joint_pos", "prev_dist", "t", "steps_since_last_goal", "consecutive_success", "successes_so_far", "goals_so_far", "success_pending")
    errs, gerr, mism = [], [], 0
    for k in range(steps):
        for a, b in ((ref.sim, env.sim), (ref.goal_sim, env.goal_sim)):
            for f in STATE_FIELDS:
                getattr(b, f).copy_(getattr(a, f).to(device=env.device, dtype=getattr(b, f).dtype))
        for f in book:
            getattr(env, f).copy_(getattr(ref, f).to(device=env.device, dtype=getattr(env, f).dtype))
        if k % 4 == 1:                  # half the environments get a goal on their fingertips: successes and new goals
            sel = torch.arange(n) % 2 == 0
            ref.goal[sel] = ref.fingertips()[sel]
            env.goal[sel.to(env.device)] = ref.goal[sel].to(env.device, torch.float32)
        a = rng.uniform(-1, 1, (n, 20)) * 0.5
        noise = rng.randn(n, 24)
        o1, r1, d1, i1 = ref.step(torch.as_tensor(a), goal_noise=noise)
        o2, r2, d2, i2 = env.step(torch.as_tensor(a, dtype=torch.float32, device=env.device), goal_noise=noise)
        e = torch.stack([(o2[key].cpu().double() - o1[key]).abs().reshape(n, -1).max(1).values for key in ("qpos", "fingertip_pos", "goal_fingertip_pos")]).max(0).values
        errs.append(torch.maximum(e, (r2.cpu().double() - r1).abs().max(1).values))
        drew = i1["goal_reset"] | d1
        if drew.any():
            gerr.append((env.goal_joint_pos.cpu().double() - ref.goal_joint_pos)[drew].abs().max(1).values)
        near = (i1["goal_dist"] - ref.success_threshold).abs() < 1e-4
        same = (d2.cpu() == d1) & (i2["goal_achieved"].cpu() == i1["goal_achieved"]) & (i2["successes_so_far"].cpu() == i1["successes_so_far"]) & \
               (i2["goals_so_far"].cpu() == i1["goals_so_far"])
        mism += int((~same & ~near).sum())
    errs, gerr = torch.cat(errs), torch.cat(gerr)
    assert int(env.sim.warn.max()) == 0 and int(env.goal_sim.warn.max()) == 0, (int(env.sim.warn.max()), int(env.goal_sim.warn.max()))
    # round-off, except where a finger contact opens or closes within the env-step: those env-steps differ by up to ~1e-2
    # (the statistics of test_locked_env.py's teacher-forced test, with a median bound at round-off level)
    for e in (errs, gerr):
        stats = (float(e.median()), float((e < 2e-3).double().mean()), float(e.max()))
        assert stats[0] < 2e-5 and stats[1] >= 0.95 and stats[2] < 5e-2, stats
    assert mism == 0
    assert int(ref.successes_so_far.sum()) > 0 and gerr.numel() > n          # successes, new goals and restarts were exercised


@pytest.mark.gpu
@pytest.mark.parametrize("randomize", [False, True])
def test_cuda_env_8192_random_actions(randomize):
    """8192 environments, 300 random-action env-steps with auto-reset: finite states, no engine warning, consistent tracker counts,
    and goal-simulation launches that cover exactly the environments that drew a goal (new goal or restart)."""
    import torch

    from robogym_b200 import build
    from robogym_b200.reach_env import make_cuda_env

    build.build()
    n = 8192
    env = make_cuda_env(n, seed=2, max_timesteps_per_goal=40, success_threshold=0.05, randomize=randomize)
    env.reset()
    launched = []
    real_forward = env.goal_sim.forward
    env.goal_sim.forward = lambda mask=None, count=1: (launched.append(mask.clone()), real_forward(mask=mask, count=count))[1]
    gen = torch.Generator(device=env.device); gen.manual_seed(0)
    ndone = nnew = nsucc = 0
    for k in range(300):
        g0 = env.goals_so_far.clone()
        launched.clear()
        obs, rew, done, info = env.step(torch.rand(n, 20, device=env.device, generator=gen) * 2 - 1)
        drew = info["goal_reset"] | done
        got = torch.zeros(n, dtype=torch.bool, device=env.device)
        for mk in launched:
            assert not bool((got & mk).any())              # each environment draws at most one goal per step
            got |= mk
        assert torch.equal(got, drew), k
        assert torch.equal(info["goals_so_far"] > g0, info["goal_reset"])
        assert bool((env.goals_so_far[done] == 1).all()) and bool((env.successes_so_far[done] == 0).all())
        assert bool((info["successes_so_far"] <= info["goals_so_far"]).all())
        ndone += int(done.sum()); nnew += int(info["goal_reset"].sum()); nsucc += int(info["sub_goal_is_successful"].sum())
        if k % 50 == 0:
            assert all(bool(torch.isfinite(v).all()) for v in obs.values()) and bool(torch.isfinite(rew).all())
    for name, s in (("main", env.sim), ("goal", env.goal_sim)):
        assert bool(torch.isfinite(s.qpos).all()) and bool(torch.isfinite(s.qvel).all()), name
        assert int(s.warn.max()) == 0, (name, int(s.warn.max()), int(s.ncon.max()))
    assert ndone >= n and env.episodes == n + ndone and nnew <= nsucc
    assert env.goal_launches == 3 * (n + n + ndone + nnew)     # construction, reset, then one draw per restart and per new goal
