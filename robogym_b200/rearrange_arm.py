"""Batched dual-simulation arm controller of the rearrange environments (SURVEY 8(f) row 4).

The reference drives the UR16e of `robogym.envs.rearrange` with TWO simulations per environment
(robogym/robot/composite/ur_gripper_arm.py:104-150): a *solver* simulation -- arm + gripper only, the tool centre point welded
to a mocap body -- turns the policy's tool-space action into joint angles, and the *main* simulation, whose arm joints are
driven by mujoco-py's cascaded-PI controllers, tracks them.  Per env-step (robogym/robot_env.py:804-844):

  1. `URGripperCompositeRobot.denormalize_position_control(action, relative_action=True)`
       arm    : tool displacement = a[:3] * max_position_change, angles = a[3:] * speed_per_dof (free_dof_tcp_arm.py:161-178)
       gripper: current gripper target + a[-1] * half control range, clipped (robot_interface.py:247-278)
  2. `JointControlledTcpArm.set_position_control` (joint_controlled_tcp_arm.py:90-98)
       with `arm_reset_controller_error`: solver arm joints := main arm joints, forward (free_dof_tcp_arm.py:215-226)
       `FreeDOFTcpArm.set_position_control` (free_dof_tcp_arm.py:182-206): clip the angle mapped to joint 6 against its range
       (`constrain_quat_ctrl`, :133-155), `MocapSolver.get_tcp_quat` (mocap_solver.py:29-46), `mocap_set_action`
       (gym.envs.robotics.utils: mocap bodies re-seated on their welded body, then moved by the deltas), solver `mj_sim.step()`
       main ctrl[:6] := solver arm joint angles (joint_controlled_arm.py:180-181); main gripper ctrl := gripper target
  3. main `SimulationInterface.step()` (substeps + forward), and the forward `RobotEnv._observe_sync` adds before observing
     (robot_env.py:677) -- mujoco-py's controller state advances in each forward, so the count matters (`main_forwards`)
  4. `on_observations_updated` (joint_controlled_tcp_arm.py:129-140): the solver's gripper follows the main gripper

Here both simulations are `BatchedSim`s (one fused launch each per env-step) and steps 1-4 are one masked kernel launch
between each pair of simulation launches (rg_arm_phase, csrc/rg_arm.inl); nothing leaves the device.  The class also works on
any object with BatchedSim's attributes on the CPU: there steps 1-4 are the float tensor ops of `_step_torch`, so the CPU tier
runs it on the oracle stand-in (tests/stubs) beside the unmodified reference environment (tests/test_rearrange_arm.py), and the
GPU tests hold the kernel to that path bit for bit.

The robot's part of the reference's reset is here too: `initialize_sim_state` (RearrangeEnv._initialize_sim_state for MOCAP_IK,
rearrange/common/base.py:448-465) and `randomize_initial_position` (_randomize_robot_initial_position, :484-496: one random
action held for n_random_initial_steps env-steps, then zero actions), for the environments of a mask.
"""
import ctypes
import math

import numpy as np

# robogym/robot/ur16e/mujoco/free_dof_tcp_arm.py:13-17 and robot/control/tcp/solver.py:10-13 (euler index of each axis)
DOF_SPEED = {"roll": math.radians(200), "pitch": math.radians(600), "yaw": math.radians(300)}
EULER_INDEX = {"roll": 0, "pitch": 2, "yaw": 1}
JOINT_OF_DOF = {"pitch": 5}                      # MocapSolver.JOINT_MAPPING (mocap_solver.py:17-19)
JOINT_DRIFT_THRESHOLD = math.radians(1)         # free_dof_tcp_arm.py:26-28
EQ_WELD = 1
TABLETOP_EXPERIMENT_INITIAL_POS = np.deg2rad([135.0, -90.0, 135.0, -100.0, -240.0, 135.0])   # robot/ur16e/arm_interface.py:27


def euler2quat(t, euler):
    """robogym/utils/rotation.py:110-126"""
    ai, aj, ak = euler[..., 2] / 2, -euler[..., 1] / 2, euler[..., 0] / 2
    si, sj, sk = t.sin(ai), t.sin(aj), t.sin(ak)
    ci, cj, ck = t.cos(ai), t.cos(aj), t.cos(ak)
    cc, cs, sc, ss = ci * ck, ci * sk, si * ck, si * sk
    return t.stack([cj * cc + sj * ss, cj * cs - sj * sc, -(cj * ss + sj * cc), cj * sc - sj * cs], dim=-1)


def quat_mul(t, q0, q1):
    """robogym/utils/rotation.py:234-257"""
    w0, x0, y0, z0 = q0.unbind(-1)
    w1, x1, y1, z1 = q1.unbind(-1)
    return t.stack([w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1, w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1,
                    w0 * y1 + y0 * w1 + z0 * x1 - x0 * z1, w0 * z1 + z0 * w1 + x0 * y1 - y0 * x1], dim=-1)


def quat2mat(t, q):
    """robogym/utils/rotation.py:202-225 (unit-norm input: the degenerate branch is not needed)"""
    w, x, y, z = q.unbind(-1)
    s2 = 2.0 / (q * q).sum(-1)
    X, Y, Z = x * s2, y * s2, z * s2
    wX, wY, wZ, xX, xY, xZ, yY, yZ, zZ = w * X, w * Y, w * Z, x * X, x * Y, x * Z, y * Y, y * Z, z * Z
    return t.stack([t.stack([1.0 - (yY + zZ), xY - wZ, xZ + wY], -1), t.stack([xY + wZ, 1.0 - (xX + zZ), yZ - wX], -1),
                    t.stack([xZ - wY, yZ + wX, 1.0 - (xX + yY)], -1)], -2)


def align_axis(t, cmd_quat, axis):
    """MocapSolver.align_axis (mocap_solver.py:59-75): rotate `cmd_quat` by the shortest arc that brings its body axis closest to
    world axis `axis` exactly onto it (rotation.vectors2quat, rotation.py:469-486; the antiparallel case cannot occur: the
    chosen body axis has its largest component along the world axis, sign-flipped to be positive)."""
    mtx = quat2mat(t, cmd_quat)
    nr = mtx[:, axis, :].abs().argmax(dim=1)
    ax = mtx.gather(2, nr.view(-1, 1, 1).expand(-1, 3, 1)).squeeze(2)
    ax = ax * t.sign(ax[:, axis:axis + 1])
    e = t.zeros_like(ax)
    e[:, axis] = 1.0
    q = t.cat([((ax * ax).sum(1) * 1.0).sqrt().unsqueeze(1) + ax[:, axis:axis + 1], t.linalg.cross(ax, e)], dim=1)
    q = q / q.norm(dim=1, keepdim=True)
    q = q * t.where(q[:, :1] < 0, -t.ones_like(q[:, :1]), t.ones_like(q[:, :1]))       # quat_normalize: w >= 0
    return quat_mul(t, q, cmd_quat)


class BatchedTcpArmController:
    """`main`, `solver`: BatchedSim-like objects for the joint-actuated scene and the mocap-welded arm (the solver needs the
    outputs body_xpos / body_xquat).  `dof_dims`: the tool rotations the policy controls -- ("roll", "pitch") is
    ControlMode.TCP_ROLL_YAW's FreeRollYawTcpArm (free_dof_tcp_arm.py:243-250; no alignment axis), the reference's default and the
    mode SURVEY 8(d) row 4 names; ("pitch",) with align_axis="pitch" is ControlMode.TCP_WRIST's FreeWristTcpArm (:232-240)."""

    def __init__(self, main, solver, max_position_change, dof_dims=("roll", "pitch"), reset_controller_error=True, prefix="robot0:", main_forwards=2,
                 align_axis=None):
        assert max_position_change and max_position_change > 0.0, "Position multiplier must be a positive number"
        self.main, self.solver = main, solver
        self.t = main.torch
        self.max_position_change = float(max_position_change)
        self.dof_dims = tuple(dof_dims)
        self.reset_controller_error = bool(reset_controller_error)
        self.main_forwards = int(main_forwards)
        self.align_axis = None if align_axis is None else EULER_INDEX[align_axis]
        mm, ms = main.model.host, solver.model.host
        arm = [f"{prefix}J{i}" for i in range(1, 7)]
        self.arm_qadr_main = [int(mm["jnt_qposadr"][main.model.name2id("joint", n)]) for n in arm]
        self.arm_qadr_solver = [int(ms["jnt_qposadr"][solver.model.name2id("joint", n)]) for n in arm]
        self.arm_jnt_solver = [solver.model.name2id("joint", n) for n in arm]
        gj, ga = prefix + "r_gripper_RJ0_outer", prefix + "r_gripper_finger_joint"
        self.grip_qadr_main = int(mm["jnt_qposadr"][main.model.name2id("joint", gj)])
        self.grip_qadr_solver = int(ms["jnt_qposadr"][solver.model.name2id("joint", gj)])
        self.grip_act_main = main.model.name2id("actuator", ga)
        self.grip_act_solver = solver.model.name2id("actuator", ga)
        cr = np.asarray(mm["actuator_ctrlrange"]).reshape(-1, 2)[self.grip_act_main]
        self.grip_lo, self.grip_hi = float(cr[0]), float(cr[1])
        self.arm_act_main = [main.model.name2id("actuator", f"ur_actuator_{i}") for i in range(1, 7)]
        self.tcp_body = solver.model.name2id("body", prefix + "gripper_tcp")
        # mocap welds of the solver model: (mocap slot, welded body), as gym's reset_mocap2body_xpos pairs them
        self.welds = []
        for i in range(int(ms["neq"])):
            if int(ms["eq_type"][i]) != EQ_WELD:
                continue
            b1, b2 = int(ms["eq_obj1id"][i]), int(ms["eq_obj2id"][i])
            k, body = int(ms["body_mocapid"][b1]), b2
            if k == -1:
                k, body = int(ms["body_mocapid"][b2]), b1
            assert k != -1, "weld without a mocap body"
            self.welds.append((i, k, body))
        assert self.welds, "the solver simulation has no mocap weld"
        jr = np.asarray(ms["jnt_range"]).reshape(-1, 2)
        self.jnt_lo = [float(jr[j, 0]) for j in self.arm_jnt_solver]
        self.jnt_hi = [float(jr[j, 1]) for j in self.arm_jnt_solver]
        self.speed = [DOF_SPEED[d] * self.max_position_change for d in self.dof_dims]
        self.action_dim = 3 + len(self.dof_dims) + 1
        # CUDA simulations run steps 1-4 as the kernel of rg_arm_phase, from these tables (built once, passed with every launch)
        self.on_device = bool(getattr(main.qpos, "is_cuda", False))
        self._tables = self._arm_tables() if self.on_device else None
        # configurations whose kernel steps are bit-identical to the tensor path's (DESIGN §9): in the others an unmasked step()
        # keeps the tensor path, so what it computes does not change; masked steps and the reset run the kernel everywhere
        self.kernel_exact = self.on_device and self.align_axis is None

    def _arm_tables(self):
        from . import engine

        T = engine.ArmTables()
        T.narm = len(self.arm_qadr_main)
        for j in range(T.narm):
            T.arm_qpos_main[j], T.arm_qpos_solver[j], T.arm_act_main[j] = self.arm_qadr_main[j], self.arm_qadr_solver[j], self.arm_act_main[j]
            T.lo_lim[j] = self.jnt_lo[j] + JOINT_DRIFT_THRESHOLD           # the scalars constrain_quat_ctrl subtracts the joint from
            T.hi_lim[j] = self.jnt_hi[j] - JOINT_DRIFT_THRESHOLD
        T.grip_qpos_main, T.grip_qpos_solver, T.grip_act_main, T.grip_act_solver = self.grip_qadr_main, self.grip_qadr_solver, self.grip_act_main, self.grip_act_solver
        T.tcp_body = self.tcp_body
        T.nweld = len(self.welds)
        for w, (_, k, body) in enumerate(self.welds):
            T.weld_mocap[w], T.weld_body[w] = k, body
        T.ndof = len(self.dof_dims)
        for i, d in enumerate(self.dof_dims):
            T.euler_index[i] = EULER_INDEX[d]
            T.dof_joint[i] = JOINT_OF_DOF.get(d, -1)
            T.speed[i] = self.speed[i]
        T.align_axis = -1 if self.align_axis is None else self.align_axis
        T.max_position_change, T.grip_lo, T.grip_hi = self.max_position_change, self.grip_lo, self.grip_hi
        T.grip_half = (self.grip_hi - self.grip_lo) / 2.0
        return T

    @staticmethod
    def _arm_sim(sim):
        from . import engine

        m = sim.model.host
        return engine.ArmSim(int(m["nq"]), int(m["nu"]), int(m["nbody"]), int(m["nmocap"]), *[engine.ptr(getattr(sim, n, None)) for n in
                             ("qpos", "ctrl", "body_xpos", "body_xquat", "mocap_pos", "mocap_quat")])

    def _phase(self, phases, mask, action=None):
        """one launch of rg_arm_phase on the environments of `mask` (a device uint8 tensor, or None: all)"""
        from . import engine

        if action is not None:
            if tuple(action.shape) != (self.main.nenv, self.action_dim):
                raise ValueError(f"action: expected shape {(self.main.nenv, self.action_dim)}, got {tuple(action.shape)}")
            action = action.to(device=self.main.device, dtype=self.t.float32).contiguous()
        width = self.action_dim
        engine._check(engine.lib().rg_arm_phase(ctypes.byref(self._tables), int(phases), self.main.nenv, ctypes.byref(self._arm_sim(self.main)),
                                                ctypes.byref(self._arm_sim(self.solver)), engine.ptr(action), width, engine.ptr(mask),
                                                0 if mask is None else int(mask.numel()), engine.current_stream(self.t, self.main.device)))

    def _mask(self, mask):
        from . import engine

        if not self.on_device:
            if mask is not None:
                raise ValueError("a mask needs the CUDA simulations; the tensor path steps every environment")
            return None
        return engine.device_mask(self.t, mask, self.main.nenv, self.main.device)

    # ---- reset: JointControlledTcpArm.__init__ / reset (joint_controlled_tcp_arm.py:52-58,100-102), MocapSolver.reset (mocap_solver.py:55-57)
    def reset(self, mask=None):
        """Call after the main simulation has its initial state: the solver arm takes the main arm's joint angles and its gripper
        state, the mocap welds are re-zeroed (relative pose = identity, model-wide) and the mocap bodies seated on the tool.
        `mask` ([nenv] bool / uint8; CUDA simulations only): only those environments."""
        ms = self.solver.model.host
        data = np.array(ms["eq_data"], dtype=np.float64).reshape(int(ms["neq"]), -1)
        for i, _, _ in self.welds:
            data[i, :7] = [0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]
        self.solver.model.set_field("eq_data", data.reshape(-1))
        mask = self._mask(mask)
        if self.on_device:
            from . import engine

            self._phase(engine.ARM_SYNC | engine.ARM_GRIP, mask)
            self.solver.forward(mask)
            self._phase(engine.ARM_SEAT, mask)
            return
        self.solver.qpos[:, self.arm_qadr_solver] = self.main.qpos[:, self.arm_qadr_main].to(self.solver.qpos.dtype)
        self.solver.qpos[:, self.grip_qadr_solver] = self.main.qpos[:, self.grip_qadr_main].to(self.solver.qpos.dtype)
        self.solver.ctrl[:, self.grip_act_solver] = self.main.ctrl[:, self.grip_act_main].to(self.solver.ctrl.dtype)
        self.solver.forward()
        self._seat_mocaps()

    def _seat_mocaps(self):
        for _, k, body in self.welds:
            self.solver.mocap_pos[:, k] = self.solver.body_xpos[:, body]
            self.solver.mocap_quat[:, k] = self.solver.body_xquat[:, body]

    # ---- step 1
    def denormalize(self, action):
        """[-1, 1]^(3 + ndof + 1) -> tool displacement (m), tool angles (rad), gripper target (joint units)"""
        t = self.t
        a = action                                   # float32, like the environment's action space: the reference multiplies the
        dt = self.main.qpos.dtype                    # translations and the gripper share in float32, the angles in float64
        n = len(self.dof_dims)
        pos = (a[:, :3] * self.max_position_change).to(dt)
        ang = a[:, 3:3 + n].to(dt) * t.tensor(self.speed, dtype=dt, device=a.device)
        centre = self.main.ctrl[:, self.grip_act_main]   # MujocoRobotiqGripper.get_current_position is the current TARGET (mujoco_robotiq_gripper.py:139-140)
        grip = (centre + (a[:, 3 + n] * ((self.grip_hi - self.grip_lo) / 2.0)).to(dt)).clamp(self.grip_lo, self.grip_hi)
        return pos, ang, grip

    # ---- step 2
    def set_position_control(self, pos, ang, grip):
        t, s = self.t, self.solver
        if self.reset_controller_error:
            s.qpos[:, self.arm_qadr_solver] = self.main.qpos[:, self.arm_qadr_main].to(s.qpos.dtype)
            s.forward()
        ang = ang.to(s.qpos.dtype).clone()
        for i, d in enumerate(self.dof_dims):                       # constrain_quat_ctrl
            j = JOINT_OF_DOF.get(d)
            if j is None:
                continue
            jp = s.qpos[:, self.arm_qadr_solver[j]]
            ang[:, i] = t.minimum(t.maximum(ang[:, i], self.jnt_lo[j] + JOINT_DRIFT_THRESHOLD - jp), self.jnt_hi[j] - JOINT_DRIFT_THRESHOLD - jp)
        euler = t.zeros(ang.shape[0], 3, dtype=ang.dtype, device=ang.device)
        for i, d in enumerate(self.dof_dims):
            euler[:, EULER_INDEX[d]] = ang[:, i]
        gq = s.body_xquat[:, self.tcp_body].to(ang.dtype)
        target = quat_mul(t, gq, euler2quat(t, euler))              # MocapSolver.get_tcp_quat
        if self.align_axis is not None:
            target = align_axis(t, target, self.align_axis)
        dquat = target - gq
        self._seat_mocaps()                                          # mocap_set_action
        k = self.welds[0][1]
        s.mocap_pos[:, k] += pos.to(s.mocap_pos.dtype)
        s.mocap_quat[:, k] += dquat.to(s.mocap_quat.dtype)
        s.step(final_forward=0)                                      # mj_sim.step(): substeps only
        self.main.ctrl[:, self.arm_act_main] = s.qpos[:, self.arm_qadr_solver].to(self.main.ctrl.dtype)
        self.main.ctrl[:, self.grip_act_main] = grip.to(self.main.ctrl.dtype)

    # ---- steps 1-4
    def step(self, action, mask=None):
        """One env-step: the action ([nenv, action_dim] in [-1, 1]) through the solver simulation into the main simulation's
        controls, the main simulation's step with `main_forwards` forwards, the solver's gripper synced.  `mask` ([nenv] bool /
        uint8; CUDA simulations only): only those environments are stepped, the others are left as they are."""
        if mask is None and not self.kernel_exact:
            return self._step_torch(action, self.main_forwards)
        self._step(action, self._mask(mask), self.main_forwards, True)

    def _step(self, action, mask, main_forwards, grip_sync, main_step=True):
        if not self.on_device:
            return self._step_torch(action, main_forwards, grip_sync, main_step)
        from . import engine

        if self.reset_controller_error:
            self._phase(engine.ARM_SYNC, mask)
            self.solver.forward(mask)
        self._phase(engine.ARM_PRESOLVE, mask, action)
        self.solver.step(final_forward=0, mask=mask)
        self._phase(engine.ARM_POSTSOLVE, mask, action)
        if main_step:
            self.main.step(final_forward=main_forwards, mask=mask)
            if grip_sync:
                self._phase(engine.ARM_GRIP, mask)

    def _step_torch(self, action, main_forwards, grip_sync=True, main_step=True):
        """steps 1-4 as float tensor ops, every environment: the path of the CPU stand-ins, and the reference the GPU tests hold
        the kernel to"""
        pos, ang, grip = self.denormalize(action)
        self.set_position_control(pos, ang, grip)
        if not main_step:
            return
        self.main.step(final_forward=main_forwards)
        if grip_sync:
            self.solver.qpos[:, self.grip_qadr_solver] = self.main.qpos[:, self.grip_qadr_main].to(self.solver.qpos.dtype)
            self.solver.ctrl[:, self.grip_act_solver] = self.main.ctrl[:, self.grip_act_main].to(self.solver.ctrl.dtype)

    # ---- the robot's part of the reset (RearrangeEnv._reset, rearrange/common/base.py:897-932)
    def initialize_sim_state(self, mask=None):
        """_initialize_sim_state for TcpSolverMode.MOCAP_IK (base.py:448-465): the main simulation's welds switched off
        (model-wide), then robot.reset(): the main arm at TABLETOP_EXPERIMENT_INITIAL_POS in qpos and ctrl
        (JointControlledArm.set_simulation_start_position, joint_controlled_arm.py:123-132) and the controller's reset.  The
        reference rebuilds both simulations before this (_recreate_sim), so velocities, controller (PID) state and warm starts
        of both are cleared here; the rebuilt solver arm already stands at the start pose, which is what reset()'s copy of the
        main arm gives it.  The reference calls this before the objects are placed and settled (base.py:904-913)."""
        dev_mask = self._mask(mask)                     # refused before anything is written
        t = self.t
        keep = None if mask is None else (~t.as_tensor(mask, device=self.main.qpos.device).reshape(-1, 1).bool())
        for sim in (self.main, self.solver):            # _recreate_sim: both simulations start at rest, controller state cleared
            for name in ("qvel", "pid", "qacc_warmstart"):
                v = getattr(sim, name)
                if keep is None:
                    v.zero_()
                else:
                    v.mul_(keep.to(v.dtype))
        mm = self.main.model.host
        active = np.array(mm["eq_active"]).reshape(-1).copy()
        active[np.asarray(mm["eq_type"]).reshape(-1) == EQ_WELD] = 0
        self.main.model.set_field("eq_active", active)
        start = self.t.tensor(TABLETOP_EXPERIMENT_INITIAL_POS, dtype=self.main.qpos.dtype, device=self.main.qpos.device)
        if mask is None:
            self.main.qpos[:, self.arm_qadr_main] = start
            self.main.ctrl[:, self.arm_act_main] = start.to(self.main.ctrl.dtype)
        else:
            self.main.qpos[:, self.arm_qadr_main] = t.where(keep, self.main.qpos[:, self.arm_qadr_main], start)
            self.main.ctrl[:, self.arm_act_main] = t.where(keep, self.main.ctrl[:, self.arm_act_main], start.to(self.main.ctrl.dtype))
        self.reset(dev_mask)

    def sample_initial_action(self, seed, epoch, mask=None):
        """action_space.sample() of each environment of `mask` on the device ([nenv, action_dim] float32; rows of other
        environments are zero): Philox4x32-10 keyed by (seed, environment) under purpose 5, gym's Box.sample mapping (rg_arm_sample_actions)"""
        from . import engine

        if not self.on_device:
            raise ValueError("sample_initial_action draws on the CUDA device; on other simulations pass the action to hold_initial_action")
        t = self.t
        m = engine.device_mask(t, mask, self.main.nenv, self.main.device)
        out = t.zeros(self.main.nenv, self.action_dim, dtype=t.float32, device=self.main.device)
        engine._check(engine.lib().rg_arm_sample_actions(self.main.nenv, self.action_dim, int(seed) & 0xFFFFFFFF, int(epoch) & 0xFFFFFFFF, engine.ptr(m),
                                                         0 if m is None else int(m.numel()), engine.ptr(out), engine.current_stream(t, self.main.device)))
        return out

    def hold_initial_action(self, action, mask=None, n_random_initial_steps=10, n_zero_steps=100):
        """the step loop of _randomize_robot_initial_position (base.py:484-496) with a given action: n_random_initial_steps
        env-steps of `action`, one controller step of the zero action without a main step, then n_zero_steps env-steps of the zero
        action.  Each env-step is _set_action and mujoco_simulation.step(): ONE main forward and no gripper sync, as the
        reference has no observation between them.  With n_random_initial_steps < 1 nothing is stepped."""
        if n_random_initial_steps < 1:
            return
        mask = self._mask(mask)
        for _ in range(int(n_random_initial_steps)):
            self._step(action, mask, 1, False)
        zero = action * 0.0
        self._step(zero, mask, 1, False, main_step=False)
        for _ in range(int(n_zero_steps)):
            self._step(zero, mask, 1, False)

    def randomize_initial_position(self, mask, seed, epoch, n_random_initial_steps=10, n_zero_steps=100):
        """_randomize_robot_initial_position for the environments of `mask` (None: all): the held random action is drawn on the
        device (sample_initial_action) and returned."""
        action = self.sample_initial_action(seed, epoch, mask)
        self.hold_initial_action(action, mask, n_random_initial_steps, n_zero_steps)
        return action
