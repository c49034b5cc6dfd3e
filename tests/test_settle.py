"""The settle launch (rg_step_settle, BatchedSim.settle, rearrange_scene.stabilize_objects): the reference's stabilize_objects
(robogym/envs/rearrange/common/utils.py:76-93) with the object damping as a launch constant.  CPU tier: the emulation of the
kernel source (tests/emu, the settle build pyemu_settle) and the library's argument checks; the CUDA kernel is checked in tests/test_settle_gpu.py.

* The emulated settle equals the composition it stands for -- the object dofs' damping set in the selected environments only,
  a masked step of the same substeps, the damping restored, a masked forward -- byte for byte, and leaves the other
  environments as they were.
* Giving the override to only one of the two reads of dof_damping (the passive force, the implicit term of the Euler factor)
  changes the result: the settle has to reach both.
* From the reset states the unmodified reference recorded (tests/golden/reference_settle.json.gz, tools/make_settle_golden.py),
  the fp64 oracle reproduces the reference's settled poses and the emulated kernel lands on them within a bound derived from
  how far the settle moves the blocks."""
import gzip
import json
import os
import sys

import numpy as np
import pytest

import pyemu_settle
from helpers import golden_model
from robogym_b200 import engine, rearrange_scene

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "stubs"))
ASSET = "rearrange_blocks5_tcp"
NSUB = 40                      # bench.py's rearrange_blocks_tcp substeps per env-step
FIELDS = ("qpos", "qvel", "pid", "warm", "time", "site_xpos", "body_xpos", "body_xquat", "geom_xpos", "act_force", "qacc", "contact", "ncon",
          "warn", "sensordata")


def composed(e, mask, dofs, damping, nsub, final_forward=1):
    """the settle through the existing primitives: the damping edited (only the selected environments are stepped), a masked
    step of nsub substeps, the damping restored, a masked forward"""
    row = e.model_field("dof_damping", np.float32)
    saved = row.copy()
    row[dofs] = np.float32(damping)
    e.step(nsub, 0, mask=mask)
    row[:] = saved
    e.step(0, final_forward, mask=mask)


def _golden():
    with gzip.open(os.path.join(HERE, "golden", "reference_settle.json.gz"), "rt") as f:
        return json.load(f)["cases"]


def object_dofs(m, names):
    bodies = [names["body"].index(f"object{k}") for k in range(8) if f"object{k}" in names["body"]]
    return rearrange_scene.object_dofs(m, bodies), bodies


def load_state(e, st, rows=slice(None)):
    for k in ("qpos", "qvel", "ctrl", "pid", "warm"):
        getattr(e, k)[rows] = np.asarray(st[k], dtype=np.float32)
    e.mocap_pos[rows] = np.asarray(st["mocap_pos"], dtype=np.float32).reshape(-1, 3)
    e.mocap_quat[rows] = np.asarray(st["mocap_quat"], dtype=np.float32).reshape(-1, 4)


def dropped_batch(nenv, seed=0):
    """nenv copies of a reset the reference recorded, each block lifted by a few millimetres, turned and moving a little: a
    placement that has not settled.  Returns the batch, the model and the object dofs."""
    c = _golden()[0]
    blob, m, names = golden_model(ASSET, c["model"])
    e = pyemu_settle.SettleBatch(blob, m, nenv, 64, 160, 16)
    load_state(e, c["state0"])
    rng = np.random.RandomState(seed)
    dofs, bodies = object_dofs(m, names)
    for b in bodies:
        j = int(m["body_jntadr"][b])
        a, d = int(m["jnt_qposadr"][j]), int(m["jnt_dofadr"][j])
        e.qpos[:, a + 2] += rng.uniform(1e-3, 4e-3, nenv).astype(np.float32)
        q = e.qpos[:, a + 3:a + 7].astype(np.float64)
        half = rng.uniform(-0.3, 0.3, nenv)
        turn = np.stack([np.cos(half), 0 * half, 0 * half, np.sin(half)], 1)          # about z, applied in the world frame
        w = turn[:, :1] * q[:, :1] - turn[:, 3:] * q[:, 3:]
        x = turn[:, :1] * q[:, 1:2] - turn[:, 3:] * q[:, 2:3]
        y = turn[:, :1] * q[:, 2:3] + turn[:, 3:] * q[:, 1:2]
        z = turn[:, :1] * q[:, 3:] + turn[:, 3:] * q[:, :1]
        e.qpos[:, a + 3:a + 7] = np.concatenate([w, x, y, z], 1).astype(np.float32)
        e.qvel[:, d:d + 6] = rng.uniform(-0.05, 0.05, (nenv, 6)).astype(np.float32)
    return e, m, dofs


def snapshot(e):
    return {k: getattr(e, k).copy() for k in FIELDS}


MASK = np.array([1, 0, 1, 1, 0, 1], dtype=np.uint8)


@pytest.fixture(scope="module")
def runs():
    a, m, dofs = dropped_batch(len(MASK))
    b, _, _ = dropped_batch(len(MASK))
    before = snapshot(a)
    a.settle(dofs, 1e-3, 2 * NSUB, mask=MASK)
    composed(b, MASK, dofs, 1e-3, 2 * NSUB)
    return before, snapshot(a), snapshot(b), dofs


def test_emulated_settle_is_the_composition_byte_for_byte(runs):
    before, a, b, _ = runs
    for k in FIELDS:
        assert a[k].tobytes() == b[k].tobytes(), k
    off = MASK == 0
    for k in FIELDS:
        assert a[k][off].tobytes() == before[k][off].tobytes(), k       # environments outside the mask are untouched
    on = MASK == 1
    assert not np.array_equal(a["qpos"][on], before["qpos"][on])
    assert int(a["warn"].max()) == 0


def test_override_has_to_reach_both_reads_of_the_damping(runs):
    _, settled, _, dofs = runs
    out = {}
    for reads in (1, 2):
        e, _, _ = dropped_batch(len(MASK))
        e.settle(dofs, 1e-3, 2 * NSUB, mask=MASK, reads=reads)
        out[reads] = e.qpos.copy()
    plain, _, _ = dropped_batch(len(MASK))
    plain.step(2 * NSUB, 1, mask=MASK)
    on = MASK == 1
    for reads, q in out.items():
        assert not np.array_equal(q[on], settled["qpos"][on]), f"the override on read {reads} alone gives the settle's result"
        assert not np.array_equal(q[on], plain.qpos[on]), f"the override on read {reads} alone changes nothing"
    assert not np.array_equal(out[1][on], out[2][on])


# ---------------------------------------------------------------------------------------------- against the reference
def _object_moves(c):
    """per block: how far the reference's settle moved its position"""
    q0, q1 = np.array(c["state0"]["qpos"]), np.array(c["qpos"])
    return np.array([np.abs(q1[a:a + 3] - q0[a:a + 3]).max() for a in c["qposadr"]])


def tolerance():
    """Every block of every recorded seed sinks by the same few hundredths of a millimetre (the seeds place the blocks
    differently, but each starts the same height above its resting depth).  A settle that lands within a tenth of the smallest
    move on every seed has settled the blocks, and one that did nothing (or stopped short) misses by the whole move.  The bound
    is that tenth, taken from the fixture itself."""
    moves = np.concatenate([_object_moves(c) for c in _golden()])
    assert moves.min() > 1e-5 and moves.max() - moves.min() < 0.1 * moves.min(), moves
    return 0.1 * moves.min()


def _object_error(q, c):
    ref = np.array(c["qpos"])
    err = []
    for a in c["qposadr"]:
        qe = q[a + 3:a + 7] * np.sign(np.dot(q[a + 3:a + 7], ref[a + 3:a + 7]))
        err.append(max(np.abs(q[a:a + 3] - ref[a:a + 3]).max(), np.abs(qe - ref[a + 3:a + 7]).max()))
    return np.array(err)


def test_fixture_records_the_reference_settle():
    cases = _golden()
    assert len(cases) >= 3 and len({c["seed"] for c in cases}) == len(cases)
    for c in cases:
        blob, m, names = golden_model(ASSET, c["model"])
        dofs, _ = object_dofs(m, names)
        assert c["dofs"] == dofs and c["n_steps"] == 100 and c["nsub"] == NSUB and c["damping"] == 1e-3


def test_oracle_settle_reproduces_the_reference():
    """the fp64 oracle, stepped as stabilize_objects steps it (100 x (nsub mj_step + forward) at damping 1e-3, then a forward
    with the damping restored), reproduces the recorded poses"""
    from oracle_generic_sim import OracleGenericSim
    from test_rearrange_arm import _load_state

    for c in _golden()[:2]:
        blob, m, _ = golden_model(ASSET, c["model"])
        sim = OracleGenericSim(blob, 1, c["nsub"])
        _load_state(sim, c["state0"])
        damp = np.array(m["dof_damping"], dtype=np.float64)
        low = damp.copy()
        low[c["dofs"]] = c["damping"]
        sim.model.set_field("dof_damping", low)
        for _ in range(c["n_steps"]):
            sim.step(c["nsub"], 1)
        sim.model.set_field("dof_damping", damp)
        sim.forward()
        err = _object_error(sim.qpos[0].numpy(), c)
        assert err.max() < 1e-9, err


def test_emulated_settle_lands_on_the_reference():
    tol = tolerance()
    for c in _golden():
        blob, m, _ = golden_model(ASSET, c["model"])
        e = pyemu_settle.SettleBatch(blob, m, 1, 64, 160, 16)
        load_state(e, c["state0"])
        e.settle(c["dofs"], c["damping"], c["n_steps"] * c["nsub"])
        err = _object_error(e.qpos[0].astype(np.float64), c)
        assert int(e.warn[0]) == 0
        assert err.max() < tol, (c["seed"], err, tol)


# ---------------------------------------------------------------------------------------------- the C ABI's checks
def _settle_rc(dofs, damping, nsub=10, final_forward=1):
    L = engine.lib()
    d = np.ascontiguousarray(dofs, dtype=np.int32)
    rc = L.rg_step_settle(None, None, d.ctypes.data if d.size else None, int(d.size), float(damping), nsub, final_forward, None)
    return rc, L.rg_last_error().decode()


@pytest.mark.skipif(not os.path.exists(engine.LIB_PATH), reason="needs the built library")
def test_abi_refuses_bad_dof_lists_and_damping():
    rc, msg = _settle_rc([], 1e-3)
    assert rc != 0 and "dof list" in msg
    rc, msg = _settle_rc(np.arange(65), 1e-3)
    assert rc != 0 and "dof list" in msg
    for bad in (-1e-3, float("nan"), float("inf"), 1e39):
        rc, msg = _settle_rc([8, 9], bad)
        assert rc != 0 and "damping" in msg, bad
    rc, msg = _settle_rc([8, 9], 1e-3, nsub=-1)
    assert rc != 0
    rc, msg = _settle_rc([8, 9], 1e-3, final_forward=5)
    assert rc != 0
    rc, msg = _settle_rc([8, 9], 1e-3)
    assert rc != 0 and "null" in msg                        # the arguments are fine; there is no batch
