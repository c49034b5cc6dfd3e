"""The settle launch on the CUDA kernel (rg_step_settle through BatchedSim.settle and rearrange_scene.stabilize_objects).

* Byte identity: the settle equals the composition it stands for -- dof_damping bound per environment with the object dofs at
  the override in the selected environments only, a masked step of the same substeps, the rows restored, a masked forward --
  in every output, for masks of one, a few and all environments, on 2048 rearrange_blocks5_tcp environments and on
  rearrange_ycb8_tcp with per-environment object draws and empty slots.  Environments outside the mask keep their state and
  outputs.  A batch that has dof_damping bound per environment settles to the same bytes.
* The reference fixture: from the recorded resets the kernel lands on the reference's settled poses within the bound
  tests/test_settle.py derives.
* Padded slots: the active objects' settled poses do not depend on whether the empty slots' dofs are in the list.
* The ABI refuses dof ids outside [0, nv)."""
import os

import numpy as np
import pytest

import test_settle as T
from helpers import golden_model

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
OUTPUTS = ("site_xpos", "body_xpos", "body_xquat", "geom_xpos", "act_force", "qacc", "contact", "ncon", "warn", "sensordata")
STATE = ("qpos", "qvel", "pid", "qacc_warmstart", "time")
CAPS = dict(contact_capacity=64, row_capacity=160, dofs_per_contact=16)
TABLE_TOP = 0.453 + 0.03324

pytestmark = pytest.mark.gpu


def _engine():
    from robogym_b200 import build, engine

    build.build()
    return engine


def _sim(blob, nenv, nsub=40):
    engine = _engine()
    model = engine.DeviceModel(blob, 0)
    return engine.BatchedSim(model, nenv, nsub, outputs=OUTPUTS, **CAPS)


def _snapshot(sim):
    import torch

    torch.cuda.synchronize()
    return {k: getattr(sim, k).cpu().numpy().copy() for k in STATE + ("ctrl",) + OUTPUTS}


def _put(sim, snap):
    for k in STATE + ("ctrl",) + OUTPUTS:
        if k in snap:
            getattr(sim, k).copy_(sim.torch.as_tensor(snap[k], device=sim.device))


def _blocks_state(nenv, seed=0):
    """nenv copies of the first recorded reset, every block lifted by 1-4 mm, turned about z and moving a little"""
    c = T._golden()[0]
    blob, m, names = golden_model(T.ASSET, c["model"])
    e, _, dofs = T.dropped_batch(nenv, seed)
    snap = dict(qpos=e.qpos, qvel=e.qvel, ctrl=e.ctrl, pid=e.pid, qacc_warmstart=e.warm, time=e.time)
    return blob, m, dofs, snap, (e.mocap_pos, e.mocap_quat)


def _compose(sim, dofs, damping, nsub, mask, rows):
    """the per-environment-row composition: rows [nenv, nv] float64 of dof_damping are bound (set_param) on `sim`"""
    t = sim.torch
    low = rows.copy()
    on = mask.cpu().numpy().astype(bool)
    low[np.ix_(on, dofs)] = damping
    sim.set_param("dof_damping", low)
    sim.step(nsub, final_forward=0, mask=mask)
    sim.set_param("dof_damping", rows)
    sim.forward(mask=mask)
    t.cuda.synchronize()


def _assert_bytes(a, b, what, envs=None):
    for k in a:
        x, y = (a[k], b[k]) if envs is None else (a[k][envs], b[k][envs])
        if x.tobytes() != y.tobytes():
            bad = np.nonzero((x != y).reshape(len(x), -1).any(1))[0]
            raise AssertionError(f"{what}: {k} differs in {len(bad)} environments, first {bad[:5]}")


def _masks(t, nenv, device):
    rng = np.random.RandomState(3)
    one = t.zeros(nenv, dtype=t.uint8, device=device); one[nenv // 3] = 1
    few = t.zeros(nenv, dtype=t.uint8, device=device); few[t.as_tensor(rng.choice(nenv, 13, replace=False), device=device)] = 1
    return dict(one=one, few=few, all=t.ones(nenv, dtype=t.uint8, device=device))


def _identity(blob, dofs, snap, mocap, nenv, nsub, prepare=None):
    """settle against the composition on one pair of batches (`prepare(sim)` binds a scene's per-environment rows)"""
    import torch as t

    a, b = _sim(blob, nenv), _sim(blob, nenv)
    for s in (a, b):
        if prepare:
            prepare(s)
        if mocap[0] is not None:
            s.mocap_pos.copy_(t.as_tensor(mocap[0], device=s.device)); s.mocap_quat.copy_(t.as_tensor(mocap[1], device=s.device))
    _put(a, snap)
    a.forward()
    start = _snapshot(a)
    rows = np.repeat(np.asarray(b.model.host["dof_damping"], dtype=np.float64)[None], nenv, 0)
    for name, mask in _masks(t, nenv, a.device).items():
        _put(a, start); _put(b, start)
        a.settle(dofs, 1e-3, nsub, mask=mask)
        t.cuda.synchronize()
        got = _snapshot(a)
        _compose(b, dofs, 1e-3, nsub, mask, rows)
        _assert_bytes(got, _snapshot(b), f"settle vs composition, mask {name}")
        off = ~mask.cpu().numpy().astype(bool)
        _assert_bytes(got, start, f"environments outside mask {name}", off)
        on = ~off
        assert not np.array_equal(got["qpos"][on], start["qpos"][on])
        # a batch with dof_damping bound per environment (the override then goes into each environment's own row)
        _put(b, start)
        b.settle(dofs, 1e-3, nsub, mask=mask)
        _assert_bytes(got, _snapshot(b), f"settle with per-environment damping rows, mask {name}")
        print(f"settle == composition, mask {name} ({int(on.sum())} environments), launch {a.launch_info()} / {b.launch_info()}")
    return a


def test_cuda_settle_is_the_composition_on_2048_block_environments():
    blob, m, dofs, snap, mocap = _blocks_state(2048)
    sim = _identity(blob, dofs, snap, mocap, 2048, 2 * 40)
    assert int((sim.warn.cpu().numpy() & ~1).max()) == 0


def _ycb_scene(nenv, seed=7):
    from robogym_b200 import rearrange_mesh_scene as rms

    b8, bt = (open(os.path.join(ASSETS, n + ".rgm"), "rb").read() for n in ("rearrange_ycb8", "rearrange_ycb8_tcp"))
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    sb = rms.slotted_model(bt, lib)
    rng = np.random.RandomState(seed)
    draws = rng.randint(0, len(lib.entries), (nenv, 8))
    draws[rng.rand(nenv, 8) < 0.25] = -1                 # about a quarter of the slots empty
    draws[0] = -1; draws[0, 2] = 4                        # one environment with a single object
    xy = np.array([[1.25 + 0.27 * (k % 3), 0.32 + 0.36 * (k // 3)] for k in (0, 1, 2, 3, 5, 6, 7, 8)])
    yaw = rng.uniform(-np.pi, np.pi, (nenv, 8))
    return lib, sb, draws, np.broadcast_to(xy, (nenv, 8, 2)).copy(), yaw


def _ycb_prepare(lib, draws, xy, yaw):
    from robogym_b200 import rearrange_mesh_scene as rms

    def prepare(sim):
        sc = rms.BatchedMeshScene(sim, lib)
        sc.set_objects(draws)
        sc.place(xy, yaw, TABLE_TOP, clearance=2e-3)
        sim.ctrl.copy_(sim.qpos[:, :7])                    # the arm holds its pose
        return sc
    return prepare


def test_cuda_settle_is_the_composition_on_ycb_draws_with_empty_slots():
    from robogym_b200 import rearrange_scene

    nenv = 512
    lib, sb, draws, xy, yaw = _ycb_scene(nenv)
    prepare = _ycb_prepare(lib, draws, xy, yaw)
    probe = _sim(sb, 1)
    bodies = [probe.model.name2id("body", f"object{k}") for k in range(8)]
    dofs = rearrange_scene.object_dofs(probe.model.host, bodies)
    # the state the placement leaves: qpos / qvel written by place(), identical in both batches
    s = _sim(sb, nenv)
    prepare(s)
    snap = _snapshot(s)
    _identity(sb, dofs, snap, (None, None), nenv, 2 * 40, prepare)


def _reference_sim(c, nenv):
    """a batch of nenv copies of a recorded reset"""
    import torch as t

    blob, m, names = golden_model(T.ASSET, c["model"])
    sim = _sim(blob, nenv)
    st = c["state0"]
    for k, key in (("qpos", "qpos"), ("qvel", "qvel"), ("ctrl", "ctrl"), ("pid", "pid"), ("qacc_warmstart", "warm")):
        getattr(sim, k).copy_(t.as_tensor(np.asarray(st[key], dtype=np.float32), device=sim.device).expand_as(getattr(sim, k)))
    sim.mocap_pos.copy_(t.as_tensor(np.asarray(st["mocap_pos"], dtype=np.float32).reshape(1, -1, 3), device=sim.device).expand_as(sim.mocap_pos))
    sim.mocap_quat.copy_(t.as_tensor(np.asarray(st["mocap_quat"], dtype=np.float32).reshape(1, -1, 4), device=sim.device).expand_as(sim.mocap_quat))
    return sim, m, [names["body"].index(f"object{k}") for k in range(5)]


def test_cuda_padded_slots_do_not_change_the_active_objects():
    """stabilize_objects lists every slot's dofs, a parked one's too; the active blocks settle as they do with the parked slots
    left out of the list.  From each recorded reset, blocks 3 and 4 are parked on the floor away from the table, as
    BatchedBlockScene.place parks an unused block.  The parked dofs still enter the Newton solve's line search over the whole
    system, so the results agree to rounding rather than bit for bit: the bound is the one the reference comparison uses
    (tests/test_settle.py), a tenth of how far the settle moves the blocks."""
    import torch as t

    from robogym_b200 import rearrange_scene

    tol = T.tolerance()
    for c in T._golden():
        runs = []
        for listed in (5, 3):
            sim, m, bodies = _reference_sim(c, 64)
            qadr = [int(m["jnt_qposadr"][m["body_jntadr"][b]]) for b in bodies]
            half_z = np.asarray(m["geom_size"]).reshape(-1, 3)[[int(m["body_geomadr"][b]) for b in bodies], 2]
            for k in (3, 4):
                sim.qpos[:, qadr[k]:qadr[k] + 7] = t.tensor([3.0 + 0.25 * k, -1.0, half_z[k] + 1e-3, 1, 0, 0, 0], device=sim.device)
            q0 = sim.qpos.cpu().numpy().astype(np.float64)
            rearrange_scene.stabilize_objects(sim, bodies[:listed], n_steps=c["n_steps"])
            t.cuda.synchronize()
            assert int(sim.warn.max()) == 0
            runs.append(sim.qpos.cpu().numpy().astype(np.float64))
        act = np.concatenate([np.arange(qadr[k], qadr[k] + 7) for k in range(3)])
        worst = np.abs(runs[0][:, act] - runs[1][:, act]).max()
        moved = np.abs(runs[0][:, act] - q0[:, act]).max()
        same = int((runs[0][:, act] == runs[1][:, act]).all(1).sum())
        print(f"seed {c['seed']}: parked slots listed or not, active block poses differ by at most {worst:.3g} (bit-identical in "
              f"{same} of 64 environments); the settle moved them by up to {moved:.3g}")
        assert moved > 5 * tol and worst < tol, (worst, moved, tol)


def test_cuda_settle_lands_on_the_reference():
    import torch as t

    from robogym_b200 import rearrange_scene

    tol = T.tolerance()
    for c in T._golden():
        sim, m, bodies = _reference_sim(c, 4)
        rearrange_scene.stabilize_objects(sim, bodies, n_steps=c["n_steps"], damping=c["damping"])
        t.cuda.synchronize()
        q = sim.qpos.cpu().numpy()
        assert np.array_equal(q[0], q[3])
        err = T._object_error(q[0].astype(np.float64), c)
        print(f"seed {c['seed']}: settled block poses within {err.max():.3g} of the reference (bound {tol:.3g})")
        assert int(sim.warn.max()) == 0 and err.max() < tol, (err, tol)


def test_cuda_abi_refuses_dof_ids_out_of_range():
    engine = _engine()
    blob, m, dofs, snap, mocap = _blocks_state(4)
    sim = _sim(blob, 4)
    for bad in ([m["nv"]], [-1], [8, 9, 1000]):
        with pytest.raises(engine.EngineError, match="out of range"):
            sim.settle(bad, 1e-3, 10)
    with pytest.raises(engine.EngineError, match="dof list"):
        sim.settle([], 1e-3, 10)
    with pytest.raises(engine.EngineError, match="damping"):
        sim.settle([8], -1.0, 10)
