"""Batched dactyl/reach environment on one device (BASELINE.json configs[0]).

`BatchedReachEnv` is what `robogym.envs.dactyl.reach.make_simple_env()` is for ONE environment, for `nenv` environments at
once, around the same fused physics launch as `locked_env.BatchedLockedEnv`:

* build                       ReachSimulation.build (reach.py:133-143): absolute zero control (mid-range targets), 20 steps;
                              every environment starts there, and the goal simulation too (its margins are raised after it)
* action -> ctrl              RobotEnv._set_action via ShadowHandCubeFacade.denormalize_position_control (relative)
* goal                        FingertipPosGoal.next_goal (envs/dactyl/goals/shadow_hand_reach_fingertip_pos.py:27-73) on a
                              second batched simulation, one state per environment, launched only for the environments that
                              draw a goal
* goal distance / reward      norm of the 15-vector goal minus the absolute fingertip positions; reward = its decrease,
                              success = distance < 0.025 (reach.py:47-55)
* multi-goal bookkeeping      locked_env.track_goals (MultiGoalTracker.process)
* reset                       RobotEnv.reset: the simulation is NOT reset (RobotEnv._reset is `pass`), the tracker is, and a
                              goal is drawn; finished environments restart inside the step (vector-env auto-reset)

Neither the goal simulation's state nor `goal_joint_pos` is reset between goals or episodes, as in the reference.
The simulator is injected (`sim_factory(blob, n)`): the product path is `engine.BatchedSim`; tests drive the same host logic on
the fp64 oracle.
"""
import json
import os

import numpy as np

from . import modelblob
from .batched_env import ShadowHandCubeFacade
from .locked_env import ActionLatency, TorchRand, track_goals

GOAL_MARGIN = 0.002                     # ReachEnv.build_goal_generation (reach.py:179-190): every geom_margin + 0.002
FINGERS = ("TH", "FF", "MF", "RF", "LF", "WR")
STATE_FIELDS = ("qpos", "qvel", "ctrl", "pid", "qacc_warmstart", "time")
REACH_NOISE_LEVELS = {"fingertip_pos": {"uncorrelated": 0.001, "additive": 0.001}}       # reach.py:28-30


def finger_separation(m, names, active_finger, prefix="robot0:"):
    """FingerSeparationWrapper._freeze_joint (wrappers/dactyl.py:109-150) on the model dict `m`, in place: every finger but
    `active_finger` gets a 0.01-wide jnt_range next to one of its limits.  The same for every environment, so it is a model edit."""
    if active_finger not in FINGERS:
        raise ValueError(f"active_finger must be one of {FINGERS}, got {active_finger!r}")
    jr = m["jnt_range"].reshape(-1, 2)
    jn = names["joint"]

    def freeze(joint, limit):
        if prefix + joint in jn:
            j = jn.index(prefix + joint)
            jr[j, limit] = jr[j, 1 - limit] + (-0.01 if limit == 0 else 0.01)

    a = FINGERS.index(active_finger)
    for i, f in enumerate(FINGERS):
        if i == a:
            continue
        if "F" in f:
            limit = 0 if i < a else 1
            for jnt, lim in (("J4", 1), ("J3", limit), ("J2", 1), ("J1", 1), ("J0", 1)):
                freeze(f + jnt, lim)
        if "TH" in f:
            for jnt, lim in (("J4", 0), ("J3", 1), ("J2", 1), ("J1", 0), ("J0", 0)):
                freeze(f + jnt, lim)


def actuated_joint_range(m, names):
    """utils/dactyl_utils.py:4-14: jnt_range clipped to the control range of the actuator that drives each joint, [njnt, 2]"""
    jr = np.array(m["jnt_range"], dtype=float).reshape(-1, 2).copy()
    cr = np.asarray(m["actuator_ctrlrange"], dtype=float).reshape(-1, 2)
    jn = names["joint"]
    for a, nme in enumerate(names["actuator"]):
        j = jn.index(nme.replace("A_", ""))
        jr[j, 0] = max(jr[j, 0], cr[a, 0])
        jr[j, 1] = min(jr[j, 1], cr[a, 1])
        jr[j, 1] = max(jr[j, 0], jr[j, 1])
    return jr


class BatchedReachEnv:
    REWARD_NAMES = ("env", "goal", "success")

    def __init__(self, sim_factory, blob, names, nenv, device, seed=0, rand=None, active_finger=None, relative_action=True,
                 successes_needed=50, max_timesteps_per_goal=150, min_timesteps_per_goal=0, success_threshold=0.025,
                 success_reward=5.0, build_steps=20, auto_reset=True, randomize=False, action_latency=None):
        """`sim_factory(blob, n)` returns a batched simulator of n environments of the model `blob`."""
        import torch

        self.torch = torch
        self.nenv = n = int(nenv)
        self.device = device
        # the two models: FingerSeparationWrapper's ranges on both (the goal simulation copies the main one's ranges before every
        # draw, FingertipPosGoal.next_goal), the raised margins on the goal simulation only
        self.model = modelblob.unpack(blob)
        if active_finger is not None:
            finger_separation(self.model, names, active_finger)
        self.goal_model = {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in self.model.items()}
        self.goal_model["geom_margin"] = self.goal_model["geom_margin"] + GOAL_MARGIN
        tables = modelblob.unpack_names(blob)
        main_blob = blob if active_finger is None else modelblob.pack(self.model, tables)
        self.sim = sim_factory(main_blob, n)
        self.goal_sim = sim_factory(modelblob.pack(self.goal_model, tables), n)
        dtype = self.sim.qpos.dtype
        self.fac = ShadowHandCubeFacade(self.model, names, device, dtype=dtype)
        self.rand = rand or TorchRand(torch, device, seed, dtype)
        lim = actuated_joint_range(self.model, names)
        hand = [j for j, nme in enumerate(names["joint"]) if nme is not None and nme.startswith("robot0:")]
        self.joint_lo = torch.as_tensor(lim[hand, 0], dtype=dtype, device=device)
        self.joint_hi = torch.as_tensor(lim[hand, 1], dtype=dtype, device=device)
        self.relative_action = relative_action
        self.successes_needed, self.max_timesteps_per_goal, self.min_timesteps_per_goal = successes_needed, max_timesteps_per_goal, min_timesteps_per_goal
        self.success_threshold, self.success_reward, self.auto_reset = success_threshold, success_reward, auto_reset
        # step: SimulationInterface.step ends with sim.forward(); _observe_sync and MujocoObservationProvider.sync forward twice
        # more (mujoco-py's PID state advances in each), fused into the step launch
        self.final_forward = 3
        self.randomizer = self.obs_noise = None
        if randomize:
            # reach.py:226-240 on the main simulation; the goal simulation stays nominal, as the reference's wrappers never touch it
            from .obs_noise import BatchedObservationNoise
            from .randomization import REACH_RULES, LockedRandomizer

            self.randomizer = LockedRandomizer(self.model, names, self.rand, torch, device, dtype, rules=REACH_RULES)
            self.ts_state = self.randomizer.timestep_state(n)
            self.timestep = self.sim.enable_per_env_timestep()
            self.obs_noise = BatchedObservationNoise(torch, self.rand, n, dict(fingertip_pos=15), levels=REACH_NOISE_LEVELS)
        if action_latency is None:
            action_latency = 1 if randomize else 0
        self.latency = ActionLatency(torch, self.rand, n, int(self.model["nu"]), action_latency, dtype, device)
        z = lambda dt: torch.zeros(n, dtype=dt, device=device)
        self.goal = torch.zeros(n, 15, dtype=dtype, device=device)
        self.prev_dist = z(dtype)
        self.t = z(torch.long)
        self.steps_since_last_goal = z(torch.long)
        self.consecutive_success = z(torch.long)
        self.successes_so_far = z(torch.long)
        self.goals_so_far = z(torch.long)
        self.success_pending = z(torch.bool)
        self.episodes = 0
        self.goal_launches = 0              # environment-launches of the goal simulation (3 per goal drawn)
        self._build(sim_factory, blob, build_steps)
        # RobotEnv.__init__ draws one goal before the first reset (robot_env.py:427): it moves the goal simulation and goal_joint_pos
        self._draw_goals(torch.ones(n, dtype=torch.bool, device=device))

    # ---------------------------------------------------------------- build
    def _build(self, sim_factory, blob, steps):
        """ReachSimulation.build on the unedited model (the wrappers edit it after the build), once, copied to every environment
        of both simulations"""
        b = sim_factory(blob, 1)
        zero = self.torch.zeros(1, self.fac.P.shape[0], dtype=b.qpos.dtype, device=b.qpos.device)
        b.ctrl.copy_(self.fac.denormalize_position_control(zero, None, relative_action=False))
        for _ in range(steps):
            b.step()
        for s in (self.sim, self.goal_sim):
            for f in STATE_FIELDS:
                getattr(s, f).copy_(getattr(b, f).to(getattr(s, f).dtype).expand_as(getattr(s, f)))
        self.goal_joint_pos = self.sim.qpos[:, self.fac.hand_qpos_idx].clone()

    # ---------------------------------------------------------------- goals
    def fingertips(self, sim=None):
        return self.fac.fingertip_absolute_positions((sim or self.sim).site_xpos)

    def goal_distance(self):
        return (self.goal - self.fingertips()).norm(dim=1)

    def _draw_goals(self, mask, noise=None):
        """FingertipPosGoal.next_goal for the environments in `mask`; `noise` ([k, njoint], tests) replaces the standard-normal
        draws.  Every goal-simulation launch is masked: environments that keep their goal cost nothing."""
        torch, gs, fac = self.torch, self.goal_sim, self.fac
        idx = mask.nonzero().squeeze(1)
        k = int(idx.numel())
        if k == 0:
            return
        z = self.rand.randn(k, self.goal_joint_pos.shape[1]) if noise is None else noise
        scale = 0.1 * (self.joint_hi - self.joint_lo)
        q = torch.minimum(torch.maximum(self.goal_joint_pos[idx] + z.to(scale.dtype) * scale, self.joint_lo), self.joint_hi)
        qpos = gs.qpos[idx]
        qpos[:, fac.hand_qpos_idx] = q
        gs.qpos[idx] = qpos                                     # set_qpos: joint angles only; qvel, PID state, warm start carry over
        gs.forward(mask=mask)
        zero = torch.zeros(k, fac.P.shape[0], dtype=gs.qpos.dtype, device=gs.qpos.device)
        for _ in range(2):                                      # two steps under the relative zero action settle the contacts
            gs.ctrl[idx] = fac.denormalize_position_control(zero, gs.qpos[idx], relative_action=True)
            gs.step(mask=mask)
        self.goal_joint_pos[idx] = gs.qpos[idx][:, fac.hand_qpos_idx]
        self.goal[idx] = self.fingertips(gs)[idx]
        self.goal_launches += 3 * k

    def _set_new_goal(self, mask, noise=None):
        """RobotEnv.reset_goal (robot_env.py:893-904) for the environments in `mask`."""
        idx = mask.nonzero().squeeze(1)
        if idx.numel() == 0:
            return
        self._draw_goals(mask, None if noise is None else noise[idx])
        self.goals_so_far[idx] += 1
        self.steps_since_last_goal[idx] = 0
        self.consecutive_success[idx] = 0
        self.sim.forward(mask=mask, count=2)                    # _observe_sync
        self.prev_dist[idx] = self.goal_distance()[idx]

    # ---------------------------------------------------------------- reset
    def _reset_envs(self, mask, noise=None):
        idx = mask.nonzero().squeeze(1)
        k = int(idx.numel())
        if k == 0:
            return
        if self.randomizer is not None:
            self.randomizer.apply(self.sim, self.randomizer.sample(k), idx)
            for key, v in self.randomizer.timestep_state(k).items():
                self.ts_state[key][idx] = v
            self.timestep[idx] = self.randomizer.timestep0
        if self.obs_noise is not None:
            self.obs_noise.reset(idx)
        if self.latency.max_delay > 0:
            self.latency.reset(idx)
        self.t[idx] = 0
        self.successes_so_far[idx] = 0
        self.goals_so_far[idx] = 0
        self.success_pending[idx] = False
        self.episodes += k
        self._set_new_goal(mask, noise)

    def reset(self, goal_noise=None):
        """RobotEnv.reset (robot_env.py:757-792) for every environment: no simulation reset, a new goal.  `goal_noise` as in step()."""
        noise = None if goal_noise is None else self.torch.as_tensor(goal_noise, device=self.device)
        self._reset_envs(self.torch.ones(self.nenv, dtype=self.torch.bool, device=self.device), noise)
        return self.observe()

    # ---------------------------------------------------------------- observations
    def observe(self):
        """ReachEnv._default_observation_map (reach.py:163-172)."""
        s = self.sim
        obs = dict(qpos=s.qpos[:, self.fac.hand_qpos_idx].clone(), qvel=s.qvel[:, self.fac.hand_qvel_idx].clone(),
                   fingertip_pos=self.fingertips().clone(), goal_fingertip_pos=self.goal.clone(),
                   is_goal_achieved=(self.goal_distance() < self.success_threshold).to(s.qpos.dtype))
        if self.latency.max_delay > 0:
            self.latency.observe(obs)
        if self.obs_noise is not None:
            obs = self.obs_noise(obs)
        return obs

    # ---------------------------------------------------------------- step
    def step(self, action, goal_noise=None):
        """RobotEnv.step + step_finalize for every environment.  Returns obs, reward [nenv, 3] (env, goal, success), done [nenv],
        info.  With auto_reset, finished environments are restarted before the observation is taken; `info` describes the step
        that ended the episode.  `goal_noise` ([nenv, njoint], optional, tests) replaces the standard-normal draws of the goals
        drawn in this step (new goals and restarts)."""
        torch = self.torch
        s = self.sim
        a = torch.clamp(torch.as_tensor(action, dtype=s.qpos.dtype, device=self.device), -1.0, 1.0)
        if self.latency.max_delay > 0:
            a = self.latency(a)
        s.ctrl.copy_(self.fac.denormalize_position_control(a, s.qpos, relative_action=self.relative_action))
        s.step(final_forward=self.final_forward)
        if self.randomizer is not None:     # RandomizedTimestepWrapper.step: the timestep of the NEXT step
            self.timestep.copy_(self.randomizer.next_timestep(self.ts_state))
        self.t += 1
        dist = self.goal_distance()
        goal_reward = self.prev_dist - dist
        self.prev_dist = dist.clone()
        success = dist < self.success_threshold
        got, success_reward, done, trial_success, newgoal = track_goals(self, success, dist.dtype)
        info = dict(goal_dist=dist, goal_achieved=success, sub_goal_is_successful=got, trial_success=trial_success,
                    goal_reset=newgoal.clone(), successes_so_far=self.successes_so_far.clone())
        noise = None if goal_noise is None else torch.as_tensor(goal_noise, device=self.device)
        self._set_new_goal(newgoal, noise)
        info["goals_so_far"] = self.goals_so_far.clone()
        info["steps_since_last_goal"] = self.steps_since_last_goal.clone()
        reward = torch.stack([torch.zeros_like(dist), goal_reward, success_reward], dim=1)
        if self.auto_reset:
            self._reset_envs(done, noise)
        return self.observe(), reward, done, info


def make_cuda_env(nenv, device=0, seed=0, n_substeps=10, contact_capacity=100, **kw):
    """dactyl/reach on the CUDA engine (the product path; raises without a GPU).  Both simulations hold the reference's nconmax = 100
    contacts per environment: the hand's self-contacts under random actions, and the goal simulation's raised margins, overflow the
    engine's default of 32."""
    import torch

    from . import engine

    here = os.path.join(os.path.dirname(os.path.abspath(__file__)), "assets")
    blob = open(os.path.join(here, "dactyl_reach.rgm"), "rb").read()
    names = json.load(open(os.path.join(here, "dactyl_reach.names.json")))
    models = {}

    def factory(b, n):
        if b not in models:
            models[b] = engine.DeviceModel(b, device)
        return engine.BatchedSim(models[b], n, n_substeps, outputs=("site_xpos", "ncon", "warn"), contact_capacity=contact_capacity)

    return BatchedReachEnv(factory, blob, names, nenv, torch.device("cuda", device), seed=seed, **kw)
