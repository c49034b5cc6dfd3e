"""Per-environment mesh scale in the narrow phase (`mesh_scale`, include/robogym_b200.h) and the full cube's size randomisation
built on it (FullCubeRandomizer(cube_size_range=...), the reference's RandomizedPerpendicularCubeSizeWrapper).

The oracle carries the reference's literal edits: mesh_vert x s, geom_rbound x s, cubelet body_pos x s.  The engine keeps the
vertices and scales the support point (and its own OBB cull box) by mesh_scale instead."""
import copy
import gzip
import json
import os

import numpy as np
import pytest

import pyemu
from helpers import full_cube_states, oracle_pair
from robogym_b200 import mjcf, modelblob

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
CAPS = dict(contact_capacity=64, row_capacity=256, dofs_per_contact=32)
CONSTS = ("dof_invweight0", "body_invweight0", "tendon_invweight0", "tendon_length0", "body_subtreemass", "opt_meaninertia")


# ---------------------------------------------------------------------------------------------- small model with hulls
def _clouds():
    rng = np.random.RandomState(11)
    out = {}
    for name, n, ext in (("ma.stl", 40, (0.05, 0.045, 0.04)), ("mb.stl", 30, (0.04, 0.04, 0.035))):
        p = rng.randn(n, 3)
        p /= np.linalg.norm(p, axis=1, keepdims=True)
        out[name] = p * np.array(ext) * rng.uniform(0.8, 1.0, (n, 1))
    return out


# a convex hull resting on the plane, a second hull on top of it (mesh-mesh) and a capsule on that one (capsule-mesh)
STACK = """<mujoco><compiler angle="radian" coordinate="local"/><option timestep="0.002"/><size nuserdata="0" njmax="400" nconmax="60"/>
<asset><mesh name="ma" file="ma.stl"/><mesh name="mb" file="mb.stl"/></asset>
<worldbody><body name="floor" pos="0 0 0"><geom name="floor" type="plane" size="2 2 1" condim="3"/></body>
<body name="ha" pos="0 0 0.09" euler="0.2 -0.1 0.4"><joint type="free"/><geom name="ha" type="mesh" mesh="ma" density="800" condim="3"/></body>
<body name="hb" pos="0.01 0.005 0.22" euler="-0.3 0.2 1.0"><joint type="free"/><geom name="hb" type="mesh" mesh="mb" density="600" condim="3"/></body>
<body name="cap" pos="-0.005 0.0 0.34" euler="1.45 0.1 0"><joint type="free"/><geom name="cap" type="capsule" size="0.02 0.04" density="500" condim="3"/></body>
</worldbody></mujoco>"""


def _stack():
    clouds = _clouds()
    cm = mjcf.compile_mjcf(STACK, asset_loader=lambda p: clouds[p.split("/")[-1]])
    return cm.blob(), cm.m


def _mesh_geoms(m):
    return np.nonzero(np.asarray(m["geom_type"]) == mjcf.GEOM_MESH)[0]


def _scale_oracle(om, m, s):
    """the reference's edits on the oracle model: every hull's vertices and every mesh geom's bounding sphere times s"""
    om.field("mesh_vert")[:] *= s
    om.field("geom_rbound")[_mesh_geoms(m)] *= s


def _scale_emu(e, m, s):
    e.model_field("mesh_scale", np.float32)[:] = s
    e.model_field("geom_rbound", np.float32)[_mesh_geoms(m)] *= np.float32(s)


def _teacher_forced(blob, m, s, scale_emu=True, windows=25):
    om, d = oracle_pair(blob)
    if s != 1.0:
        _scale_oracle(om, m, s)
    e = pyemu.EmuBatch(blob, {k: m[k] for k in modelblob.DIMS}, 1)
    if scale_emu:
        _scale_emu(e, m, s)
    errs, same, ncon, qs = [], 0, [], []
    for _ in range(windows):
        for _ in range(20):
            d.step()
        d.forward()
        e.qpos[0], e.qvel[0], e.warm[0] = d.qpos, d.qvel, d.qacc_warmstart
        e.step(5, 1)
        for _ in range(5):
            d.step()
        d.forward()
        same += int(e.ncon[0]) == int(d.ncon[0])
        ncon.append(int(d.ncon[0]))
        errs.append(float(np.abs(e.qpos[0] - d.qpos).max()))
        qs.append(e.qpos[0].copy())
    return errs, same, ncon, int(e.warn[0]), np.array(qs), d.qpos.copy()


@pytest.mark.parametrize("s", [0.8, 1.25])
def test_emulated_mesh_scale_matches_oracle_with_scaled_vertices(s):
    """mesh_scale = s model-wide in the emulated kernel against mesh_vert x s (and rbound x s) in the oracle: a hull on the plane,
    a hull on that hull, a capsule on top.  Teacher-forced every 20 substeps: same contact counts, fp32 round-off once resting."""
    blob, m = _stack()
    assert m["nmesh"] == 2
    errs, same, ncon, warn, _, q_end = _teacher_forced(blob, m, s)
    assert warn == 0 and same >= 23 and min(ncon[-8:]) >= 3, ncon
    assert np.median(errs) < 2e-6 and max(errs) < 5e-3 and np.median(errs[-8:]) < 1e-6, errs
    # and the scale mattered: the resting stack's height follows it
    _, _, _, _, _, q_one = _teacher_forced(blob, m, 1.0)
    assert abs(q_end[2] - q_one[2]) > 0.005


def test_explicit_unit_mesh_scale_is_bit_identical():
    blob, m = _stack()
    dims = {k: m[k] for k in modelblob.DIMS}
    om, d = oracle_pair(blob)
    for _ in range(60):
        d.step()
    d.forward()
    runs = []
    for explicit in (False, True):
        e = pyemu.EmuBatch(blob, dims, 1)
        if explicit:
            e.model_field("mesh_scale", np.float32)[:] = 1.0
        e.qpos[0], e.qvel[0], e.warm[0] = d.qpos, d.qvel, d.qacc_warmstart
        for _ in range(10):
            e.step(5, 1)
        runs.append((e.qpos.copy(), e.qvel.copy(), e.ncon.copy()))
    for a, b in zip(*runs):
        assert np.array_equal(a, b)


# hull cube (8 corners) next to a box: between the two, at s = 1.05, lies a contact that the UNSCALED geom box of the hull culls
PAIR = """<mujoco><compiler angle="radian" coordinate="local"/><option timestep="0.002" gravity="0 0 0"/><size nuserdata="0" njmax="100" nconmax="20"/>
<asset><mesh name="cube" file="cube.stl"/></asset>
<worldbody>
<body name="hull" pos="0 0 0.5"><joint type="free"/><geom name="hull" type="mesh" mesh="cube" density="500"/></body>
<body name="box" pos="{x:.6f} 0 0.5"><joint type="free"/><geom name="box" type="box" size="0.05 0.05 0.05" density="500"/></body>
</worldbody></mujoco>"""


def test_obb_cull_scales_with_the_hull():
    """A contact between the unscaled and the scaled box of the hull at s = 1.05: the oracle (which has no box cull) finds it, the
    kernel must too.  The same kernel with the hull's box shrunk by 1/s -- what an OBB that ignores mesh_scale would test -- drops it."""
    s, h = 1.05, 0.05
    corners = np.array([[sx, sy, sz] for sx in (-h, h) for sy in (-h, h) for sz in (-h, h)])
    x = h + 0.5 * (h + s * h)                     # box face at 0.5 (h + s h) from the hull centre: 1.25 mm inside the scaled hull
    cm = mjcf.compile_mjcf(PAIR.format(x=x), asset_loader=lambda p: corners)
    blob, m = cm.blob(), cm.m
    g = cm.name2id("geom", "hull")
    aabb = np.asarray(m["geom_aabb"]).reshape(-1, 6)[g]
    assert np.allclose(aabb, [0, 0, 0, h, h, h]) and np.allclose(m["geom_quat"].reshape(-1, 4)[g], [1, 0, 0, 0])
    om, d = oracle_pair(blob)
    _scale_oracle(om, m, s)
    d.forward()
    assert int(d.ncon[0]) >= 1
    want = sorted(d.contact.reshape(-1, 24)[:int(d.ncon[0]), 0])
    dims = {k: m[k] for k in modelblob.DIMS}
    got = []
    for shrink in (False, True):
        e = pyemu.EmuBatch(blob, dims, 1)
        _scale_emu(e, m, s)
        if shrink:
            e.model_field("geom_aabb", np.float32)[6 * g:6 * g + 6] /= np.float32(s)
        e.qpos[0] = d.qpos
        e.forward()
        got.append((int(e.ncon[0]), e.dbg_view(0)["con"][:int(e.ncon[0]), 0] if e.ncon[0] else []))
    assert got[0][0] == int(d.ncon[0]), (got, want)
    assert np.allclose(sorted(got[0][1]), want, atol=2e-6)
    assert np.allclose(want, -0.5 * (s - 1) * h, atol=2e-4)       # penetration 1.25 mm
    assert got[1][0] == 0


# ---------------------------------------------------------------------------------------------- the full cube
def _full():
    blob = open(os.path.join(ROOT, "robogym_b200", "assets", "dactyl_full_perpendicular.rgm"), "rb").read()
    names = json.load(open(os.path.join(ROOT, "robogym_b200", "assets", "dactyl_full_perpendicular.names.json")))
    return blob, names, modelblob.unpack(blob)


def _cube_edits(m, names, s):
    """PerpendicularCubeSizeModifier(s) on a copy of the host model, then mj_setConst (cube_env._reset: set_constants())"""
    m = copy.deepcopy(m)
    cb = [i for i, n in enumerate(names["body"]) if n and n.startswith("cube:cubelet:")]
    cg = [i for i, n in enumerate(names["geom"]) if n and n.startswith("cube:cubelet:")]
    mid = names["mesh"].index("cube:rounded_cube")
    a, nv = int(m["mesh_vertadr"][mid]), int(m["mesh_vertnum"][mid])
    bp = m["body_pos"].reshape(-1, 3)
    bp[cb] *= s
    mv = m["mesh_vert"].reshape(-1, 3)
    mv[a:a + nv] *= s
    m["geom_rbound"][cg] *= s
    mjcf.set_const(m, spatial_tendon_eval=lambda q: mjcf.tendon_eval(m, q))
    return m, cb, cg, mid


@pytest.fixture(scope="module")
def full_states():
    """teacher-forcing states built like tests/test_full_cube.py's fixture"""
    return full_cube_states(_full()[0])


def check(qpos, ncon, warn, after):
    """the thresholds of tests/test_full_cube.py"""
    eq = np.array([np.abs(qpos[k] - after[k][0]).max() for k in range(len(after))])
    dn = np.array([abs(int(ncon[k]) - after[k][2]) for k in range(len(after))])
    assert int(np.max(warn)) == 0
    assert (m_ := np.median(eq)) < 2e-3, m_
    assert eq.max() < 3e-2
    assert dn.max() <= 5 and np.median(dn) <= 2


def _oracle_after(blob, edited, states, nsub=10):
    after = []
    for st in states:
        om, d = oracle_pair(blob)
        for name in ("body_pos", "mesh_vert", "geom_rbound") + CONSTS:
            om.field(name)[:] = np.asarray(edited[name]).reshape(-1)
        nu = edited["nu"]
        d.qpos[:], d.qvel[:], d.ctrl[:] = st[0], st[1], st[2]
        d.userdata[:3 * nu] = st[3]
        d.qacc_warmstart[:] = st[4]
        d.env_step(nsub)
        after.append((d.qpos.copy(), d.qvel.copy(), int(d.ncon[0])))
    return after


def _host_shifted_body_pos(blob, body_pos):
    """body_pos rows as the engine stores them (bodies attached to the world relative to the model's fp32 origin)"""
    m = modelblob.unpack(blob)
    bp = np.asarray(body_pos, dtype=np.float64).reshape(-1, 3).copy()
    roots = [b for b in range(1, m["nbody"]) if m["body_parentid"][b] == 0]
    origin = np.float32(m["body_pos"].reshape(-1, 3)[roots].mean(0))
    bp[roots] = (bp[roots] - origin.astype(np.float64)).astype(np.float32)
    return bp.reshape(-1)


def test_emulated_set_const_on_the_scaled_full_cube():
    """rg_set_const's kernel code on the nv = 168 layout with the cubelet offsets scaled: within 2e-4 of the host mj_setConst."""
    blob, names, m = _full()
    edited, cb, cg, mid = _cube_edits(m, names, 1.05)
    e = pyemu.EmuBatch(blob, {k: m[k] for k in modelblob.DIMS}, 1, **CAPS)
    e.model_field("body_pos", np.float32)[:] = _host_shifted_body_pos(blob, edited["body_pos"])
    got = e.set_const()
    for k in ("dof_invweight0", "body_invweight0", "tendon_invweight0", "opt_meaninertia"):
        want = np.asarray(edited[k], dtype=np.float64).reshape(-1)
        err = np.abs(got[k] - want) / np.maximum(np.abs(want), 1e-12)
        assert err.max() < 2e-4, (k, float(err.max()))
    # the scaled offsets moved the constants of the cube's bodies
    assert np.abs(edited["body_invweight0"] - m["body_invweight0"]).max() > 1e-3 * np.abs(m["body_invweight0"]).max()


def test_emulated_full_cube_at_scale_1_05(full_states):
    """The full cube in emulation at s = 1.05 (mesh_scale of cube:rounded_cube, scaled cubelet offsets and bounding spheres, the
    constants of the scaled model), teacher-forced against an oracle carrying the modifier's literal edits."""
    blob, names, m = _full()
    states, after0 = full_states
    n = 6
    states, after0 = states[:n], after0[:n]
    edited, cb, cg, mid = _cube_edits(m, names, 1.05)
    want = _oracle_after(blob, edited, states)
    e = pyemu.EmuBatch(blob, {k: m[k] for k in modelblob.DIMS}, n, **CAPS)
    e.model_field("body_pos", np.float32)[:] = _host_shifted_body_pos(blob, edited["body_pos"])
    e.model_field("geom_rbound", np.float32)[:] = edited["geom_rbound"]
    e.model_field("mesh_scale", np.float32)[mid] = 1.05
    for k in CONSTS:
        if np.asarray(edited[k]).size:
            e.model_field(k, np.float32)[:] = np.asarray(edited[k]).reshape(-1)
    for k, st in enumerate(states):
        e.qpos[k], e.qvel[k], e.ctrl[k], e.pid[k], e.warm[k] = st
    e.step(10, 1)
    check(e.qpos, e.ncon, e.warn, want)
    assert np.abs(np.array([w[0] for w in want]) - np.array([a[0] for a in after0])).max() > 1e-3


# ---------------------------------------------------------------------------------------------- the randomiser
def _randomizer(names, m, seed, cube_size_range):
    import torch

    from robogym_b200.locked_env import TorchRand
    from robogym_b200.randomization import FullCubeRandomizer

    return FullCubeRandomizer(m, names, TorchRand(torch, "cpu", seed, torch.float64), torch, torch.device("cpu"), torch.float64,
                              cube_size_range=cube_size_range)


def test_randomizer_rows_reproduce_the_reference_modifier():
    """FullCubeRandomizer(cube_size_range=...) against what the unmodified PerpendicularCubeSizeModifier did to the model
    (tests/golden/reference_cube_size.json.gz, tools/make_cube_size_golden.py) for s = 0.95, 1.0, 1.05."""
    import torch

    blob, names, m = _full()
    rec = json.load(gzip.open(os.path.join(ROOT, "tests", "golden", "reference_cube_size.json.gz")))
    R = _randomizer(names, m, 0, (0.95, 1.05))
    svals = torch.tensor([[r["s"]] for r in rec["runs"]], dtype=torch.float64)
    p = R.sample(len(svals), noises={"cube_size": svals})
    mid = names["mesh"].index("cube:rounded_cube")
    a, nvt = int(m["mesh_vertadr"][mid]), int(m["mesh_vertnum"][mid])
    bp0, rb0, mv0 = m["body_pos"].reshape(-1, 3), np.asarray(m["geom_rbound"]), m["mesh_vert"].reshape(-1, 3)
    assert names["geom"][18] is None and names["body"][int(m["geom_bodyid"][18])].startswith("cube:cubelet:")
    for k, r in enumerate(rec["runs"]):
        s = r["s"]
        bp = p["body_pos"][k].numpy().reshape(-1, 3)
        rb = p["geom_rbound"][k].numpy()
        ms = p["mesh_scale"][k].numpy()
        assert list(np.nonzero(np.any(bp != bp0, axis=1))[0]) == r["bodies"]
        assert np.array_equal(bp[r["bodies"]].ravel(), np.array(r["body_pos"]))
        assert list(np.nonzero(rb != rb0)[0]) == r["geoms"]
        assert np.array_equal(rb[r["geoms"]], np.array(r["geom_rbound"]))
        assert rb[18] == rb0[18]                                            # the unnamed cubelet geom keeps its bounding sphere
        # the reference scales the vertex rows of one mesh; the engine's row scales that mesh
        assert list(np.nonzero(ms != 1.0)[0]) == ([mid] if s != 1.0 else [])
        assert ms[mid] == s
        if s != 1.0:
            assert r["mesh_vert_rows"] == [a, a + nvt] and r["n_mesh_vert_rows"] == nvt
            assert np.array_equal(mv0[a:a + nvt].ravel() * ms[mid], np.array(r["mesh_vert"]))
        else:
            assert r["bodies"] == [] and r["geoms"] == [] and r["n_mesh_vert_rows"] == 0


def test_randomizer_draws_last_and_leaves_the_other_rows_alone():
    blob, names, m = _full()
    n = 256
    base = _randomizer(names, m, 7, None).sample(n)
    R = _randomizer(names, m, 7, (0.95, 1.05))
    p = R.sample(n)
    added = {"body_pos", "geom_rbound", "mesh_scale"}
    assert set(p) == set(base) | added and not added & set(base)
    for k in base:
        assert np.array_equal(p[k].numpy(), base[k].numpy()), k
    mid = names["mesh"].index("cube:rounded_cube")
    s = p["mesh_scale"][:, mid].numpy()
    assert s.min() >= 0.95 and s.max() <= 1.05 and s.std() > 0.02
    cg = R.cubelet_geoms.numpy()
    assert len(cg) == 25 and 18 not in cg and len(R.cubelet_bodies) == 26
    other = np.setdiff1d(np.arange(m["ngeom"]), cg)
    assert np.array_equal(p["geom_rbound"].numpy()[:, other], np.broadcast_to(np.asarray(m["geom_rbound"])[other], (n, len(other))))
    assert np.allclose(p["geom_rbound"].numpy()[:, cg], np.asarray(m["geom_rbound"])[cg] * s[:, None], rtol=1e-15)
    assert np.array_equal(np.delete(p["mesh_scale"].numpy(), mid, axis=1), np.ones((n, m["nmesh"] - 1)))


def test_mesh_scale_must_be_finite_and_positive():
    from robogym_b200 import engine

    for bad in ([1.0, 0.0], [1.0, -2.0], [np.nan, 1.0], [np.inf, 1.0]):
        with pytest.raises(ValueError):
            engine.check_mesh_scale(np.array(bad))
    engine.check_mesh_scale(np.array([0.5, 2.0]))
    with pytest.raises(ValueError):
        _randomizer(*_full()[1:], 0, (0.0, 1.05))


# ---------------------------------------------------------------------------------------------- CUDA
def _cuda_sim(blob, n, **kw):
    from robogym_b200 import build, engine

    build.build()
    model = engine.DeviceModel(blob, 0)
    return model, engine.BatchedSim(model, n, 10, outputs=("site_xpos", "ncon", "warn"), **kw)


def _load_states(sim, states):
    import torch

    f = lambda i: torch.tensor(np.stack([s[i] for s in states]), dtype=torch.float32, device=sim.device)
    sim.qpos.copy_(f(0)); sim.qvel.copy_(f(1)); sim.ctrl.copy_(f(2)); sim.pid.copy_(f(3)); sim.qacc_warmstart.copy_(f(4))


def _stack_states(blob, m, scales):
    """per scale: a state of the settling stack on the oracle with that scale, and the oracle one env-step (10 substeps) later"""
    states, after = [], []
    for s in scales:
        om, d = oracle_pair(blob)
        _scale_oracle(om, m, s)
        for _ in range(150):
            d.step()
        d.forward()
        states.append((d.qpos.copy(), d.qvel.copy(), np.zeros(0), np.zeros(0), d.qacc_warmstart.copy()))
        d.env_step(10)
        after.append((d.qpos.copy(), d.qvel.copy(), int(d.ncon[0])))
    return states, after


@pytest.mark.gpu
def test_cuda_per_environment_mesh_scale_on_the_hull_stack():
    import torch

    blob, m = _stack()
    scales = np.linspace(0.8, 1.25, 8)
    states, want = _stack_states(blob, m, scales)
    model, sim = _cuda_sim(blob, len(scales))
    ms = np.repeat(scales[:, None], m["nmesh"], axis=1)
    sim.set_param("mesh_scale", ms)
    rb = np.repeat(np.asarray(m["geom_rbound"])[None], len(scales), axis=0)
    rb[:, _mesh_geoms(m)] *= scales[:, None]
    sim.set_param("geom_rbound", rb)
    _load_states(sim, states)
    sim.step()
    torch.cuda.synchronize()
    q, ncon = sim.qpos.cpu().numpy(), sim.ncon.cpu().numpy()
    eq = np.array([np.abs(q[k] - want[k][0]).max() for k in range(len(scales))])
    assert int(sim.warn.max()) == 0 and all(int(ncon[k]) == want[k][2] for k in range(len(scales))), (ncon, [w[2] for w in want])
    assert np.median(eq) < 1e-5 and eq.max() < 1e-3, eq
    # without the scale the same states land elsewhere
    sim.set_param("mesh_scale", np.ones_like(ms))
    sim.set_param("geom_rbound", np.repeat(np.asarray(m["geom_rbound"])[None], len(scales), axis=0))
    _load_states(sim, states)
    sim.step()
    torch.cuda.synchronize()
    q1 = sim.qpos.cpu().numpy()
    assert np.abs(q1 - np.array([w[0] for w in want])).max() > 1e-3


@pytest.mark.gpu
def test_cuda_mesh_vert_edit_agrees_with_mesh_scale():
    """rg_model_set_field("mesh_vert", v s) -- what the mujoco_py shim forwards for the reference modifier's in-place edit -- reaches
    the narrow phase, and agrees with mesh_scale = s to fp32 round-off."""
    import torch

    blob, m = _stack()
    s = 1.25
    states, want = _stack_states(blob, m, [s] * 4)
    rb = np.asarray(m["geom_rbound"]).copy()
    rb[_mesh_geoms(m)] *= s
    out = []
    for how in ("mesh_vert", "mesh_scale"):
        model, sim = _cuda_sim(blob, len(states))
        model.set_field("geom_rbound", rb)
        if how == "mesh_vert":
            model.set_field("mesh_vert", np.asarray(m["mesh_vert"]) * s)
        else:
            model.set_field("mesh_scale", np.full(m["nmesh"], s))
        _load_states(sim, states)
        sim.step()
        torch.cuda.synchronize()
        out.append((sim.qpos.cpu().numpy(), sim.ncon.cpu().numpy(), int(sim.warn.max())))
    (qa, na, wa), (qb, nb, wb) = out
    assert wa == 0 and wb == 0 and np.array_equal(na, nb)
    assert np.abs(qa - qb).max() < 1e-5
    assert np.abs(qa - np.array([w[0] for w in want])).max() < 1e-3 and all(int(na[k]) == want[k][2] for k in range(len(states)))
    with pytest.raises(Exception):
        model.set_field("mesh_scale", np.zeros(m["nmesh"]))


@pytest.mark.gpu
def test_cuda_full_cube_with_its_own_scale_per_environment(full_states):
    """16 environments of the full cube, s from 0.95 to 1.05, each against an oracle with that environment's edits; the constants
    come from rg_set_const on the device (each environment's own cubelet offsets)."""
    import torch

    blob, names, m = _full()
    states, after0 = full_states
    n = len(states)
    scales = np.linspace(0.95, 1.05, n)
    edits = [_cube_edits(m, names, s) for s in scales]
    want = [_oracle_after(blob, e[0], [st])[0] for e, st in zip(edits, states)]
    model, sim = _cuda_sim(blob, n, **CAPS)
    mid = edits[0][3]
    ms = np.ones((n, m["nmesh"]))
    ms[:, mid] = scales
    sim.set_param("body_pos", np.stack([e[0]["body_pos"] for e in edits]))
    sim.set_param("geom_rbound", np.stack([e[0]["geom_rbound"] for e in edits]))
    sim.set_param("mesh_scale", ms)
    sim.set_const()
    _load_states(sim, states)
    sim.step()
    torch.cuda.synchronize()
    check(sim.qpos.cpu().numpy(), sim.ncon.cpu().numpy(), sim.warn.cpu().numpy(), want)
    far = np.array([k for k in range(n) if abs(scales[k] - 1) > 0.02])
    assert np.abs(np.array([want[k][0] for k in far]) - np.array([after0[k][0] for k in far])).max() > 1e-3


@pytest.mark.gpu
def test_cuda_full_cube_randomizer_with_cube_size_at_batch_4096(full_states):
    """BASELINE.json configs[2] at its batch size with FullCubeRandomizer(cube_size_range=(0.95, 1.05)) applied: 16 parameter rows and
    16 states tiled over the batch reproduce themselves bit for bit in every slot, no warning bits, and the constants rg_set_const
    derived on the device match the host mj_setConst of each environment's scaled model."""
    import torch

    from robogym_b200.locked_env import TorchRand
    from robogym_b200.randomization import FullCubeRandomizer

    blob, names, m = _full()
    states, _ = full_states
    n, N = len(states), 4096
    model, sim = _cuda_sim(blob, N, **CAPS)
    R = FullCubeRandomizer(m, names, TorchRand(torch, sim.device, 5), torch, sim.device, torch.float32, cube_size_range=(0.95, 1.05))
    p = R.sample(n)
    idx = torch.as_tensor(np.arange(N) % n, device=sim.device)
    R.apply(sim, {k: v[idx] for k, v in p.items()})
    idx = idx.cpu().numpy()
    _load_states(sim, [states[k] for k in idx])
    sim.step()
    torch.cuda.synchronize()
    q = sim.qpos.cpu().numpy()
    assert int(sim.warn.max()) == 0
    assert sim.launch_info()["warps_per_cta"] >= 1
    assert np.array_equal(q.reshape(N // n, n, -1), np.broadcast_to(q[:n], (N // n, n, q.shape[1])))
    for k in range(4):
        host = copy.deepcopy(m)
        host["body_inertia"] = p["body_inertia"][k].double().cpu().numpy()
        host["body_pos"] = p["body_pos"][k].double().cpu().numpy()
        mjcf.set_const(host, spatial_tendon_eval=lambda qq: mjcf.tendon_eval(host, qq))
        for name in ("dof_invweight0", "body_invweight0", "tendon_invweight0", "opt_meaninertia"):
            got = sim._params[name][k].double().cpu().numpy()
            w = np.asarray(host[name], dtype=np.float64).reshape(-1)
            err = np.abs(got - w) / np.maximum(np.abs(w), 1e-12)
            assert err.max() < 2e-4, (k, name, float(err.max()))
