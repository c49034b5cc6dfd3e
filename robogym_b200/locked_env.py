"""Batched dactyl/locked environment on one device (SURVEY.md 8(f) row 1).

`BatchedLockedEnv` is what `robogym.envs.dactyl.locked.make_env()` is for ONE environment, for `nenv`
environments at once, with every per-step piece a tensor op around ONE fused physics launch
(`engine.BatchedSim.step`) -- no Python loop over environments:

* action -> ctrl              RobotEnv._set_action (robogym/robot_env.py:497-504) via
                              ShadowHandCubeFacade.denormalize_position_control
* physics                     SimulationInterface.step (robogym/mujoco/simulation_interface.py:176-189)
* goal                        LockedParallelGoal (robogym/envs/dactyl/goals/locked_parallel.py:34-76):
                              goal = z-rotation x one of the 24 axis-aligned orientations, distance =
                              rotation angle of quat_difference(goal, cube)
* goal info / reward          RobotEnv._get_goal_info (robogym/robot_env.py:577-625): reward = decrease of the goal
                              distance, success = distance < success_threshold["cube_quat"] (locked.py:57)
* multi-goal bookkeeping      MultiGoalTracker.process (robogym/utils/multi_goal_tracker.py:157-241)
* drop handling (optional)    StopOnFallWrapper (robogym/wrappers/cube.py:106-150)
* reset                       CubeEnv._reset + LockedEnv._randomize_cube_initial_position
                              (robogym/envs/dactyl/common/cube_env.py:330-355, locked.py:193-224), served from a
                              pool of pre-generated initial states so that finished environments restart inside the
                              same step (vector-env auto-reset) without stalling the other environments.

The simulator is injected (`sim_factory`): the product path is `engine.BatchedSim` (CUDA, fails loudly without a
GPU); tests drive the identical host logic on a CPU simulator built from the fp64 oracle.
"""
import itertools
import math

import numpy as np

from .batched_env import ShadowHandCubeFacade


# ---------------------------------------------------------------- quaternion helpers on [..., 4] tensors (w, x, y, z)
def quat_mul(torch, a, b):
    """Hamilton product (robogym/utils/rotation.py:234-268)."""
    w0, x0, y0, z0 = a.unbind(-1)
    w1, x1, y1, z1 = b.unbind(-1)
    return torch.stack([w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1,
                        w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1,
                        w0 * y1 - x0 * z1 + y0 * w1 + z0 * x1,
                        w0 * z1 + x0 * y1 - y0 * x1 + z0 * w1], dim=-1)


def quat_conjugate(torch, q):
    return q * torch.tensor([1.0, -1.0, -1.0, -1.0], dtype=q.dtype, device=q.device)


def quat_positive(torch, q):
    """rotation.quat_normalize (rotation.py:281-286): the representative with w >= 0 (no rescaling)."""
    return torch.where(q[..., :1] < 0, -q, q)


def quat_angle_between(torch, goal, cur):
    """quat_magnitude(quat_difference(goal, cur)) (rotation.py:271-278)."""
    d = quat_positive(torch, quat_mul(torch, goal, quat_conjugate(torch, cur)))
    return 2.0 * torch.acos(torch.clamp(d[..., 0], -1.0, 1.0))


def parallel_quats():
    """The 24 orientations whose faces are parallel to the world axes (cube_utils.PARALLEL_QUATS), as w >= 0 unit
    quaternions.  Enumerated from the rotation group of the cube directly: signed permutation matrices of det +1."""
    out = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            R = np.zeros((3, 3))
            for r in range(3):
                R[r, perm[r]] = signs[r]
            if np.linalg.det(R) < 0.5:
                continue
            # rotation matrix -> quaternion (largest-component branch)
            t = np.trace(R)
            if t > 0:
                s = math.sqrt(t + 1.0) * 2
                q = [0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s]
            else:
                i = int(np.argmax(np.diag(R)))
                j, k = (i + 1) % 3, (i + 2) % 3
                s = math.sqrt(1.0 + R[i, i] - R[j, j] - R[k, k]) * 2
                q = [0.0, 0.0, 0.0, 0.0]
                q[0] = (R[k, j] - R[j, k]) / s
                q[1 + i] = 0.25 * s
                q[1 + j] = (R[j, i] + R[i, j]) / s
                q[1 + k] = (R[k, i] + R[i, k]) / s
            q = np.asarray(q)
            out.append(q if q[0] >= 0 else -q)
    assert len(out) == 24
    return np.stack(out)


class TorchRand:
    """Random draws on the device (one generator per environment batch)."""

    def __init__(self, torch, device, seed, dtype=None):
        self.torch, self.device, self.dtype = torch, device, dtype or torch.float32
        self.gen = torch.Generator(device=device)
        self.gen.manual_seed(int(seed))

    def randn(self, n, k):
        return self.torch.randn(n, k, device=self.device, generator=self.gen, dtype=self.dtype)

    def uniform(self, lo, hi, n, k):
        return lo + (hi - lo) * self.torch.rand(n, k, device=self.device, generator=self.gen, dtype=self.dtype)

    def randint(self, hi, n):
        return self.torch.randint(0, hi, (n,), device=self.device, generator=self.gen)


def track_goals(env, success, dtype):
    """MultiGoalTracker.process (robogym/utils/multi_goal_tracker.py:157-241) for every environment of `env` (a batched dactyl
    environment: its tracker tensors are updated in place).  success_pause_range_s is (0, 0) when the tracker is built, so one
    successful step counts.  Returns (sub_goal_is_successful, success reward, done, trial_success, new-goal mask)."""
    torch = env.torch
    env.steps_since_last_goal += 1
    env.consecutive_success = torch.where(success, env.consecutive_success + 1, torch.zeros_like(env.consecutive_success))
    got = (env.consecutive_success >= 1) & ~env.success_pending
    success_reward = got.to(dtype) * env.success_reward
    env.successes_so_far += got.long()
    env.success_pending |= got
    done = ~got & (env.steps_since_last_goal >= env.max_timesteps_per_goal)
    settle = env.success_pending & (env.steps_since_last_goal >= env.min_timesteps_per_goal)
    env.success_pending &= ~settle
    trial_success = settle & (env.successes_so_far >= env.successes_needed)
    done |= trial_success
    env.steps_since_last_goal[trial_success] = 0
    return got, success_reward, done, trial_success, settle & ~trial_success


class ActionLatency:
    """RandomizedActionLatency (robogym/wrappers/randomizations.py:516-556): every action COORDINATE is delayed by 0..max_delay
    env-steps, drawn per episode."""

    def __init__(self, torch, rand, nenv, nu, max_delay, dtype, device):
        self.torch, self.rand, self.max_delay = torch, rand, int(max_delay)
        self.history = torch.zeros(nenv, self.max_delay + 1, nu, dtype=dtype, device=device)
        self.delay = torch.zeros(nenv, nu, dtype=torch.long, device=device)

    def reset(self, idx):
        k = int(idx.numel())
        self.history[idx] = 0
        self.delay[idx] = self.rand.randint(self.max_delay + 1, k * self.delay.shape[1]).reshape(k, -1)

    def __call__(self, a):
        # The reference shifts its history with a tuple assignment whose right-hand side is a VIEW (randomizations.py:546-549):
        # history[0] = action is visible to the shift that follows, so the result is [a, a, old[1], old[2], ...] -- a delay of
        # d >= 1 returns the action of d - 1 steps ago (and the default max_delay = 1 delays nothing).  Reproduced as is: this
        # is a drop-in, not a correction.
        torch = self.torch
        self.history.copy_(torch.cat([a.unsqueeze(1), a.unsqueeze(1), self.history[:, 1:-1]], dim=1))
        return torch.gather(self.history, 1, self.delay.unsqueeze(1)).squeeze(1)

    def observe(self, obs):
        obs["action_history"] = self.history[:, :-1].clone()
        obs["action_delay"] = self.delay.clone()


STATE_FIELDS = ("qpos", "qvel", "ctrl", "pid", "qacc_warmstart", "time", "site_xpos", "act_force")


class InitialStatePool:
    """Pre-generated episode starts (CubeEnv._reset): qpos0 -> `reset_initial_steps` zero-action steps (deterministic,
    computed once; absolute mid-range targets) -> cube position wiggle + uniform random orientation -> `n_random_initial_steps` steps holding one
    random action -> keep the state if the cube is still on the palm (the reference re-draws until it is)."""

    def __init__(self, sim, facade, rand, reset_initial_steps=20, n_random_initial_steps=10, cube_position_wiggle_std=0.005, randomizer=None):
        self.sim, self.fac, self.rand = sim, facade, rand
        self.torch = facade.torch
        self.reset_initial_steps = reset_initial_steps
        self.n_random_initial_steps = n_random_initial_steps
        self.wiggle = cube_position_wiggle_std
        self.randomizer = randomizer        # per-episode model parameters: the settle steps then run under each episode's own
        self.params = None                  # parameters (as in the reference, whose wrappers write the model before env.reset)
        self.settled = None
        if randomizer is None:
            self._settle()
            self.settled = {k: getattr(sim, k)[:1].clone() for k in ("qpos", "qvel", "ctrl", "pid", "qacc_warmstart", "time")}
        self.store = None
        self.cursor = 0
        self.generated = 0
        self.rejected = 0

    def _settle(self):
        sim, fac = self.sim, self.fac
        sim.reset()
        zero = self.torch.zeros(sim.nenv, fac.P.shape[0], dtype=sim.qpos.dtype, device=sim.qpos.device)
        for _ in range(self.reset_initial_steps):
            sim.ctrl.copy_(self._absolute_ctrl(zero))   # locked.py:197-201 (absolute targets)
            sim.step()

    def _absolute_ctrl(self, action):
        """denormalize_position_control(relative_action=False) under the pool's own (possibly randomised) control ranges."""
        cr = None
        if self.params is not None and "actuator_ctrlrange" in self.params:
            cr = self.params["actuator_ctrlrange"].reshape(action.shape[0], -1, 2).to(action.dtype)
        return self.fac.denormalize_position_control(action, None, relative_action=False, ctrlrange=cr)

    def randomize(self, wiggle, quat, action):
        """Apply given draws to the settled state and run the random-action steps; returns the on-palm mask."""
        sim, fac, torch = self.sim, self.fac, self.torch
        if self.settled is None:
            self._settle()
        else:
            for k, v in self.settled.items():
                getattr(sim, k).copy_(v.expand_as(getattr(sim, k)))
        sim.qpos[:, fac.cube_pos_idx] += wiggle * self.wiggle
        q = quat / quat.norm(dim=1, keepdim=True)
        sim.qpos[:, fac.cube_quat_idx] = quat_positive(torch, q)      # rotation.uniform_quat (rotation.py:440-446)
        sim.forward()
        for _ in range(self.n_random_initial_steps):
            sim.ctrl.copy_(self._absolute_ctrl(action))   # locked.py:216-221 (absolute targets)
            sim.step()
        if self.n_random_initial_steps == 0:
            sim.forward()
        return fac.on_palm(sim.site_xpos)

    def refill(self):
        n = self.sim.nenv
        if self.randomizer is not None:
            self.params = self.randomizer.sample(n)
            self.randomizer.apply(self.sim, self.params)
        ok = self.randomize(self.rand.randn(n, 3), self.rand.randn(n, 4), self.rand.uniform(-1.0, 1.0, n, self.fac.P.shape[0]))
        idx = ok.nonzero().squeeze(1)
        self.generated += n
        self.rejected += n - int(idx.numel())
        if idx.numel() == 0:
            raise RuntimeError("no valid initial state: the cube fell off the palm in every environment of the pool")
        self.store = {k: getattr(self.sim, k)[idx].clone() for k in STATE_FIELDS}
        if self.params is not None:
            self.store.update({"param:" + k: v[idx].clone() for k, v in self.params.items()})
        self.cursor = 0

    def take(self, k):
        """k initial states (dict of [k, ...] tensors), refilling the pool as needed."""
        torch = self.torch
        parts = []
        while k > 0:
            if self.store is None or self.cursor >= self.store["qpos"].shape[0]:
                self.refill()
            a = self.cursor
            b = min(a + k, self.store["qpos"].shape[0])
            parts.append({f: v[a:b] for f, v in self.store.items()})
            self.cursor = b
            k -= b - a
        return {f: torch.cat([p[f] for p in parts], dim=0) for f in parts[0]}


class BatchedLockedEnv:
    REWARD_NAMES = ("env", "goal", "success", "drop")

    def __init__(self, sim_factory, model, names, nenv, device, seed=0, pool_size=None, rand=None, relative_action=True,
                 successes_needed=50, max_timesteps_per_goal=400, min_timesteps_per_goal=0, success_threshold=0.4,
                 success_reward=5.0, stop_on_fall=True, drop_reward=-20.0, reset_initial_steps=20,
                 n_random_initial_steps=10, cube_position_wiggle_std=0.005, auto_reset=True, observe_forwards=None,
                 randomize=False, action_latency=None):
        import torch

        self.torch = torch
        self.nenv = int(nenv)
        self.device = device
        self.sim = sim_factory(self.nenv)
        dtype = self.sim.qpos.dtype
        self.fac = ShadowHandCubeFacade(model, names, device, dtype=dtype)
        self.rand = rand or TorchRand(torch, device, seed, dtype)
        pool_sim = sim_factory(int(pool_size or min(self.nenv, 1184)))
        self.randomizer = None
        if randomize:
            # the randomisation stack of locked.py:263-277, sampled per environment on the device (randomization.py)
            from .randomization import LockedRandomizer

            self.randomizer = LockedRandomizer(model, names, self.rand, torch, device, dtype)
            self.ts_state = self.randomizer.timestep_state(self.nenv)
            self.wind_state = self.randomizer.wind_state(self.nenv, self.sim.n_substeps * self.randomizer.timestep0)
            self.timestep = self.sim.enable_per_env_timestep()
            self.xfrc = self.sim.enable_xfrc()
        # RandomizeObservationWrapper with the locked environment's noise levels (locked.py:233-238, randomizations.py:314-389):
        # noisy_fingertip_pos / noisy_hand_angle / noisy_cube_pos / noisy_cube_quat next to the clean observations
        self.obs_noise = None
        if randomize:
            from .obs_noise import BatchedObservationNoise

            self.obs_noise = BatchedObservationNoise(torch, self.rand, self.nenv, dict(fingertip_pos=15, hand_angle=24, cube_pos=3, cube_quat=4))
        self.pool = InitialStatePool(pool_sim, self.fac, self.rand, reset_initial_steps, n_random_initial_steps, cube_position_wiggle_std, self.randomizer)
        self.relative_action = relative_action
        self.successes_needed, self.max_timesteps_per_goal, self.min_timesteps_per_goal = successes_needed, max_timesteps_per_goal, min_timesteps_per_goal
        self.success_threshold, self.success_reward = success_threshold, success_reward
        self.stop_on_fall, self.drop_reward, self.auto_reset = stop_on_fall, drop_reward, auto_reset
        # After SimulationInterface.step() (which ends with sim.forward()) the reference calls sim.forward() again while
        # observing: RobotEnv._observe_sync (robot_env.py:677), MujocoObservationProvider.sync (observation/mujoco.py:27)
        # and, under StopOnFallWrapper, cube_utils.on_palm (cube_utils.py:19).  mujoco-py's PID state in userdata
        # advances in every one of them, so they are part of the dynamics; they are fused into the step launch.
        # observe_forwards=0 drops them (faster, not the reference's trajectory).
        if observe_forwards is None:
            observe_forwards = 2 + (1 if stop_on_fall else 0)
        self.final_forward = 1 + int(observe_forwards)
        self.parallel = torch.as_tensor(parallel_quats(), dtype=dtype, device=device)
        # MujocoQposObservation / MujocoQvelObservation blank the target cube's joints (robogym/observation/mujoco.py:36-61)
        tj = [j for j, nme in enumerate(names["joint"]) if nme is not None and nme.startswith("target:")]
        span = {0: (7, 6), 1: (4, 3), 2: (1, 1), 3: (1, 1)}   # free, ball, slide, hinge: (nq, nv) per joint
        tq, tv = [], []
        for j in tj:
            nq_j, nv_j = span[int(model["jnt_type"][j])]
            tq += list(range(int(model["jnt_qposadr"][j]), int(model["jnt_qposadr"][j]) + nq_j))
            tv += list(range(int(model["jnt_dofadr"][j]), int(model["jnt_dofadr"][j]) + nv_j))
        self.target_qpos_idx = torch.as_tensor(tq, dtype=torch.long, device=device)
        self.target_qvel_idx = torch.as_tensor(tv, dtype=torch.long, device=device)
        n = self.nenv
        z = lambda dt: torch.zeros(n, dtype=dt, device=device)
        self.goal_quat = torch.zeros(n, 4, dtype=dtype, device=device)
        self.goal_quat[:, 0] = 1.0
        self.prev_dist = torch.full((n,), float("nan"), dtype=dtype, device=device)
        self.t = z(torch.long)
        self.steps_since_last_goal = z(torch.long)
        self.consecutive_success = z(torch.long)
        self.successes_so_far = z(torch.long)
        self.goals_so_far = z(torch.long)
        self.success_pending = z(torch.bool)        # MultiGoalTracker._success_and_no_goal_reset
        self.first_drop = z(torch.long)             # StopOnFallWrapper.first_drop
        self.episodes = 0
        # RandomizedActionLatency: first entry of locked.py:265-277's stack, so it is on whenever the stack is
        if action_latency is None:
            action_latency = 1 if randomize else 0
        self.latency = ActionLatency(torch, self.rand, n, int(model["nu"]), action_latency, dtype, device)
        self.max_delay, self.action_history, self.action_delay = self.latency.max_delay, self.latency.history, self.latency.delay

    # ---------------------------------------------------------------- goals
    def sample_goals(self, n):
        """LockedParallelGoal.next_goal (locked_parallel.py:34-39)."""
        torch = self.torch
        ang = self.rand.uniform(-math.pi, math.pi, n, 1)[:, 0].to(self.goal_quat.dtype)
        zq = torch.stack([torch.cos(0.5 * ang), torch.zeros_like(ang), torch.zeros_like(ang), torch.sin(0.5 * ang)], dim=1)
        zq = quat_positive(torch, zq)
        return quat_mul(torch, zq, self.parallel[self.rand.randint(24, n)])

    def goal_distance(self):
        return quat_angle_between(self.torch, self.goal_quat, self.sim.qpos[:, self.fac.cube_quat_idx])

    def _set_new_goal(self, mask, goals=None):
        """RobotEnv.reset_goal (robot_env.py:893-904) for the environments in `mask`."""
        idx = mask.nonzero().squeeze(1)
        if idx.numel() == 0:
            return
        self.goal_quat[idx] = self.sample_goals(int(idx.numel())) if goals is None else goals
        self.goals_so_far[idx] += 1
        self.steps_since_last_goal[idx] = 0
        self.consecutive_success[idx] = 0
        # reset_goal ends with _observe_sync: two more sim.forward() for these environments (PID state), then
        # _previous_goal_distance = None -> update_goal_info sets it to the current distance
        if self.final_forward > 1:
            self.sim.forward(mask=mask, count=2)
        self.prev_dist[idx] = self.goal_distance()[idx]

    # ---------------------------------------------------------------- reset
    def _load_states(self, idx, st):
        for f in STATE_FIELDS:
            getattr(self.sim, f)[idx] = st[f]

    def _reset_envs(self, mask):
        idx = mask.nonzero().squeeze(1)
        k = int(idx.numel())
        if k == 0:
            return
        st = self.pool.take(k)
        self._load_states(idx, st)
        if self.randomizer is not None:
            self.randomizer.apply(self.sim, {f[6:]: v for f, v in st.items() if f.startswith("param:")}, idx)
            ts, ws = self.randomizer.timestep_state(k), self.randomizer.wind_state(k, self.sim.n_substeps * self.randomizer.timestep0)
            for key, v in ts.items():
                self.ts_state[key][idx] = v
            self.wind_state["hit_prob"][idx] = ws["hit_prob"]
            self.timestep[idx] = self.randomizer.timestep0
            self.xfrc[idx] = 0
        if self.obs_noise is not None:              # RandomizeObservationWrapper.reset: new per-episode biases
            self.obs_noise.reset(idx)
        if self.max_delay > 0:                      # RandomizedActionLatency.reset
            self.latency.reset(idx)
        self.t[idx] = 0
        self.successes_so_far[idx] = 0
        self.goals_so_far[idx] = 0
        self.success_pending[idx] = False
        self.first_drop[idx] = 0
        self.episodes += k
        self._set_new_goal(mask)

    def reset(self):
        """RobotEnv.reset (robot_env.py:757-792) for every environment."""
        self._reset_envs(self.torch.ones(self.nenv, dtype=self.torch.bool, device=self.device))
        return self.observe()

    # ---------------------------------------------------------------- observations
    def observe(self):
        """LockedEnv._default_observation_map (locked.py:132-146)."""
        torch = self.torch
        s = self.sim
        obs = self.fac.observe(s.qpos, s.qvel, s.site_xpos, getattr(s, "act_force", None))
        obs["qpos"] = s.qpos.clone()
        obs["qpos"][:, self.target_qpos_idx] = 0.0
        obs["qvel"] = s.qvel.clone()
        obs["qvel"][:, self.target_qvel_idx] = 0.0
        obs["goal_pos"] = torch.zeros(self.nenv, 3, dtype=s.qpos.dtype, device=self.device)
        obs["goal_quat"] = quat_positive(torch, self.goal_quat)
        qg = torch.zeros_like(s.qpos)
        qg[:, self.fac.cube_quat_idx] = self.goal_quat
        qg[:, self.fac.cube_pos_idx] = torch.tensor([0.0, 0.0, -0.025], dtype=s.qpos.dtype, device=self.device)
        obs["qpos_goal"] = qg
        obs["is_goal_achieved"] = (self.goal_distance() < self.success_threshold).to(s.qpos.dtype)
        if self.max_delay > 0:
            self.latency.observe(obs)
        if self.obs_noise is not None:
            obs = self.obs_noise(obs)
        return obs

    # ---------------------------------------------------------------- step
    def step(self, action, new_goals=None):
        """RobotEnv.step (robot_env.py:804-844) + step_finalize for every environment.
        Returns obs (dict of [nenv, ...]), reward [nenv, 4] (env, goal, success, drop), done [nenv] bool, info (dict).
        With auto_reset, finished environments are restarted before the observation is taken; `info` then describes
        the step that ended the episode.  `new_goals` ([nenv, 4], optional) overrides the sampled goals (tests)."""
        torch = self.torch
        s = self.sim
        a = torch.clamp(torch.as_tensor(action, dtype=s.qpos.dtype, device=self.device), -1.0, 1.0)
        if self.max_delay > 0:
            a = self.latency(a)                     # RandomizedActionLatency.step
        cr = None
        if self.randomizer is not None:
            cr = s._params["actuator_ctrlrange"].reshape(self.nenv, -1, 2)
        s.ctrl.copy_(self.fac.denormalize_position_control(a, s.qpos, relative_action=self.relative_action, ctrlrange=cr))
        s.step(final_forward=self.final_forward)
        if self.randomizer is not None:     # RandomizedTimestepWrapper.step / RandomizedWindWrapper.step: set up the NEXT step
            self.timestep.copy_(self.randomizer.next_timestep(self.ts_state))
            self.randomizer.next_wind(self.wind_state, self.xfrc)
        self.t += 1
        # _get_goal_info
        dist = self.goal_distance()
        prev = torch.where(torch.isnan(self.prev_dist), dist, self.prev_dist)
        goal_reward = prev - dist
        self.prev_dist = dist.clone()
        success = dist < self.success_threshold
        got, success_reward, done, trial_success, newgoal = track_goals(self, success, dist.dtype)
        info = dict(goal_dist=dist, goal_achieved=success, sub_goal_is_successful=got, trial_success=trial_success,
                    goal_reset=newgoal.clone(), successes_so_far=self.successes_so_far.clone())
        self._set_new_goal(newgoal, None if new_goals is None else torch.as_tensor(new_goals, dtype=dist.dtype, device=self.device)[newgoal])
        info["goals_so_far"] = self.goals_so_far.clone()                     # MultiGoalTracker.update_info runs after reset_goal
        info["steps_since_last_goal"] = self.steps_since_last_goal.clone()
        drop = torch.zeros_like(dist)
        fell = torch.zeros_like(done)
        if self.stop_on_fall:
            fell = ~self.fac.on_palm(s.site_xpos)
            first = fell & (self.first_drop == 0)
            drop = first.to(dist.dtype) * self.drop_reward
            self.first_drop = torch.where(first, info["successes_so_far"] + 1, self.first_drop)
            done |= fell
        info["fell_down"] = fell
        reward = torch.stack([torch.zeros_like(dist), goal_reward, success_reward, drop], dim=1)
        if self.auto_reset:
            self._reset_envs(done)
        return self.observe(), reward, done, info


def make_cuda_env(nenv, device=0, seed=0, n_substeps=10, **kw):
    """dactyl/locked on the CUDA engine (the product path; raises without a GPU)."""
    import json
    import os

    from . import engine

    here = os.path.dirname(os.path.abspath(__file__))
    blob = open(os.path.join(here, "assets", "dactyl_locked.rgm"), "rb").read()
    names = json.load(open(os.path.join(here, "assets", "dactyl_locked.names.json")))
    model = engine.DeviceModel(blob, device)
    import torch

    dev = torch.device("cuda", device)
    factory = lambda n: engine.BatchedSim(model, n, n_substeps, outputs=("site_xpos", "act_force", "ncon", "warn"))
    return BatchedLockedEnv(factory, model.host, names, nenv, dev, seed=seed, **kw)
