"""Per-slot object scale in the YCB mesh scene: the engine's per-environment `geom_mesh_scale` row (include/robogym_b200.h), and
on top of it `BatchedMeshScene.set_objects(draw, scale)`, `compact_model(..., scale)` and the reference's scale rules
(`ObjectLibrary.object_scales`, `sample_object_size_scales`).

The ground truth of what the reference compiles for a scaled object is tests/golden/reference_ycb_scale.json.gz, written by
tools/make_ycb_scale_golden.py from the reference's own make_mesh_object documents and STL files."""
import gzip
import json
import os

import numpy as np
import pytest

import pyemu
import test_mesh_scene as tms
from helpers import oracle_pair
from robogym_b200 import engine, modelblob
from robogym_b200 import rearrange_mesh_scene as rms

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_ycb_scale.json.gz")
TABLE_TOP, CAPS, ARM_INIT = tms.TABLE_TOP, tms.CAPS, tms.ARM_INIT


@pytest.fixture(scope="module")
def scene():
    b8, bt = tms._blob("rearrange_ycb8"), tms._blob("rearrange_ycb8_tcp")
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    return b8, lib, rms.slotted_model(b8, lib)


@pytest.fixture(scope="module")
def golden():
    return json.loads(gzip.decompress(open(GOLDEN, "rb").read()))


def _scene_rows(sb, lib, draw, scale):
    sim = tms._RecordingSim(sb, len(draw))
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draw, scale)
    return sim.params, sc


def _inertia_tensor(I, q):
    R = rms._quat2mat(np.asarray(q, dtype=np.float64))
    return R @ np.diag(I) @ R.T


def _close(a, b, rtol=1e-9, atol=1e-12):
    return np.allclose(np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64), rtol=rtol, atol=atol)


def _hull_digest(v):
    v = np.asarray(v, dtype=np.float64).reshape(-1, 3)
    return dict(n=len(v), mean=v.mean(0), lo=v.min(0), hi=v.max(0), r2=(v * v).sum(1).mean())


def _object_rows(blob, k):
    """part geom rows, body rows and hull vertices of object<k> of a compiled model"""
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    b = names["body"].index(f"object{k}")
    g = np.nonzero(m["geom_bodyid"] == b)[0]
    hulls = [rms.Hull.of(m, int(m["geom_dataid"][j])).vert for j in g]
    return ({f: rms._rows(m, f, "ngeom")[g] for f in rms.SCENE_GEOM_FIELDS}, {f: rms._rows(m, f, "nbody")[b] for f in rms.BODY_FIELDS}, hulls)


# ---------------------------------------------------------------------------------------------- validation
def test_geom_mesh_scale_values_and_width_are_checked():
    """set_param refuses a wrong width and values that are not finite and > 0; DeviceModel.set_field refuses the array (it
    exists per environment only).  Both checks run before anything reaches the engine."""
    import torch

    sim = object.__new__(engine.BatchedSim)
    sim.torch, sim.nenv = torch, 2
    sim.model = type("M", (), {})()
    sim.model.host = {"ngeom": 5, "nmesh": 3}
    for bad in (0.0, -1.0, np.nan, np.inf):
        rows = np.ones((2, 5))
        rows[1, 3] = bad
        with pytest.raises(ValueError, match="geom_mesh_scale must be finite and positive"):
            sim.set_param("geom_mesh_scale", rows)
    with pytest.raises(engine.EngineError, match="expected 5 values"):
        sim.set_param("geom_mesh_scale", np.ones((2, 3)))
    model = object.__new__(engine.DeviceModel)
    with pytest.raises(ValueError, match="per-environment.*mesh_scale"):
        model.set_field("geom_mesh_scale", np.ones(5))


def test_scene_and_compact_model_refuse_bad_scales(scene):
    b8, lib, sb = scene
    for bad in (0.0, -0.5, np.nan, np.inf):
        scale = np.ones((2, 8))
        scale[1, 4] = bad
        with pytest.raises(ValueError, match="scale"):
            _scene_rows(sb, lib, np.array([lib.identity[0]] * 2), scale)
        with pytest.raises(ValueError, match="scale"):
            rms.compact_model(b8, lib, lib.identity[0], scale[1])


# ---------------------------------------------------------------------------------------------- against the reference
def test_compact_model_and_scene_rows_match_the_reference_compiled_objects(scene, golden):
    """At every recorded scale s: compact_model's part rows, body rows and hulls are what the model compiler makes of the
    reference's make_mesh_object(files, s); the scene writes the same rows per environment except geom_aabb, which it keeps
    unscaled for the engine to scale, plus geom_mesh_scale = s on the slot's part geoms."""
    b8, lib, sb = scene
    ms = modelblob.unpack(sb)
    for o in golden["objects"]:
        k = o["slot"]
        assert lib.entries[lib.identity[0][k]].nparts == o["nparts"]
        draw = np.array([lib.identity[0]] * len(o["runs"]))
        scale = np.ones(draw.shape)
        scale[:, k] = [r["s"] for r in o["runs"]]
        rows, sc = _scene_rows(sb, lib, draw, scale)
        gs, bs = sc.geoms[k], sc.bodies[k]
        for i, r in enumerate(o["runs"]):
            s = r["s"]
            parts, body, hulls = _object_rows(rms.compact_model(b8, lib, draw[i], scale[i]), k)
            for f in rms.SCENE_GEOM_FIELDS:
                want = np.asarray(r[f])
                assert _close(parts[f], want), (o["name"], s, f)
                w = want.shape[1]
                got = rows[f][i].reshape(-1, w)[gs[:o["nparts"]]]
                assert _close(got, want / s if f == "geom_aabb" else want), (o["name"], s, f, "scene")
            for src in (body, {f: rows[f][i].reshape(ms["nbody"], -1)[bs] for f in rms.BODY_FIELDS}):
                assert _close(src["body_mass"], r["body_mass"]) and _close(src["body_ipos"], r["body_ipos"], atol=1e-11), (o["name"], s)
                # principal axes of a near-degenerate inertia may come out in another order: compare the full tensor
                assert _close(_inertia_tensor(src["body_inertia"], src["body_iquat"]), _inertia_tensor(r["body_inertia"], r["body_iquat"]),
                              rtol=1e-8, atol=1e-9 * max(r["body_inertia"])), (o["name"], s)
            assert np.array_equal(rows["geom_mesh_scale"][i][gs], np.full(len(gs), s))
            for h, d in zip(hulls, r["hulls"]):
                got = _hull_digest(h)
                assert got["n"] == d["n"]
                for key in ("mean", "lo", "hi", "r2"):
                    assert _close(got[key], d[key], atol=1e-11), (o["name"], s, key)
        others = np.delete(np.arange(ms["ngeom"]), gs)
        assert np.array_equal(rows["geom_mesh_scale"][:, others], np.ones((len(o["runs"]), len(others))))


def test_library_extents_are_the_reference_mesh_extents(scene, golden):
    _, lib, _ = scene
    for o in golden["objects"]:
        assert _close(lib.entries[lib.identity[0][o["slot"]]].extents, o["extents"], atol=1e-9), o["name"]


def _reference_object_scales(extents, draw, size_scale, mesh_scale, normalize_mesh, normalized_mesh_size):
    """MeshRearrangeEnv._recreate_sim (robogym/envs/rearrange/common/mesh.py:66-102) then make_objects_xml's
    `obj_group.scale * simulation_params.mesh_scale` (simulation/mesh.py:59), one object group per drawn slot (an empty slot is
    an object the environment does not have), written out loop by loop"""
    nenv, nslot = draw.shape
    out = np.ones(draw.shape)
    for i in range(nenv):
        num_objects = int((draw[i] >= 0).sum())
        global_scale = 1.0 if num_objects < 10 else (10.0 / num_objects) ** 0.5
        if normalize_mesh:
            new_scales = [normalized_mesh_size / (np.max(extents[e]) / 2.0) if e >= 0 else 1.0 for e in draw[i]]
        else:
            new_scales = np.ones(nslot)
        for k in range(nslot):
            orig = size_scale[i, k]
            if num_objects >= 10:
                orig = min(orig, 1.0)
            if draw[i, k] >= 0:
                out[i, k] = orig * new_scales[k] * global_scale * mesh_scale
    return out


@pytest.mark.parametrize("nslot", [8, 12])
def test_object_scales_follow_the_reference_rules(scene, nslot):
    _, lib, _ = scene
    rng = np.random.RandomState(nslot)
    draw = rng.randint(-1, len(lib.entries), (6, nslot))
    draw[0, :4] = -1                                   # an environment with 4 objects fewer than slots
    size = np.exp(rng.uniform(-0.5, 1.8, draw.shape))
    ext = [e.extents for e in lib.entries]
    for kw in (dict(), dict(mesh_scale=1.3), dict(normalize_mesh=True), dict(normalize_mesh=True, normalized_mesh_size=0.08, mesh_scale=0.9)):
        full = dict(dict(mesh_scale=1.0, normalize_mesh=False, normalized_mesh_size=0.05), **kw)
        want = _reference_object_scales(ext, draw, size, **full)
        assert np.allclose(lib.object_scales(draw, size, **kw), want, rtol=1e-14), kw
    n = (draw >= 0).sum(1)
    big = np.repeat(n >= 10, nslot).reshape(draw.shape) & (draw >= 0)
    if nslot >= 10:   # with 10 or more objects no object is scaled up by its size scale, and all of them shrink by sqrt(10 / n)
        assert big.any() and (~big & (draw >= 0)).any()
        assert np.all(lib.object_scales(draw, size)[big] <= np.repeat(np.sqrt(10.0 / np.maximum(n, 1)), nslot).reshape(draw.shape)[big] + 1e-15)
    # 12 slots, 3 of them empty: 9 objects, so nothing shrinks
    d9 = np.array([[0, 1, 2, 3, -1, 5, 6, -1, 8, 9, -1, 11]])
    assert np.allclose(lib.object_scales(d9, np.full(d9.shape, 1.3))[d9 >= 0], 1.3, rtol=1e-15)


def test_sample_object_size_scales_is_exp_of_a_uniform_draw():
    import torch

    g = torch.Generator().manual_seed(3)
    s = rms.sample_object_size_scales(4000, 8, 0.5, 1.8, generator=g)
    assert s.shape == (4000, 8) and s.dtype == torch.float64
    u = torch.log(s)
    assert float(u.min()) >= -0.5 and float(u.max()) <= 1.8
    assert abs(float(u.mean()) - 0.65) < 0.02                      # mean of U(-0.5, 1.8)
    again = rms.sample_object_size_scales(4000, 8, 0.5, 1.8, generator=torch.Generator().manual_seed(3))
    assert torch.equal(s, again)


def test_rebuilding_the_identity_draw_gives_the_base_arrays(scene):
    """compact_model returns the base blob itself for the identity draw at scale 1; the rebuild it skips still reproduces every
    array of the base exactly (only its geom names, object<k>-<j>, differ)"""
    b8, lib, _ = scene
    rebuilt = rms._build(b8, lib, [(e, lib.entries[e].nparts, 1.0) for e in lib.identity[0]], set_const=False)
    m0, m1 = modelblob.unpack(b8), modelblob.unpack(rebuilt)
    assert all(m0[k] == m1[k] for k in modelblob.DIMS)
    for _, name, _ in modelblob.ARRAYS:
        assert np.array_equal(m0[name], m1[name]), name


def test_identity_draw_at_scale_one_is_the_base_blob_byte_for_byte(scene):
    b8, lib, _ = scene
    assert rms.compact_model(b8, lib, lib.identity[0], np.ones(8)) == b8
    assert rms.compact_model(b8, lib, lib.identity[0]) == b8
    # a scale on an empty slot has nothing to scale
    draw = list(lib.identity[0])
    draw[3] = -1
    assert rms.compact_model(b8, lib, draw, [1, 1, 1, 2.0, 1, 1, 1, 1]) == rms.compact_model(b8, lib, draw)


def test_same_object_in_two_slots_at_two_scales(scene):
    """Two slots of one environment draw the 29-part object at 0.7 and 1.45: the batch keeps both on the library's hulls and
    tells them apart by geom_mesh_scale; the compact model gives each its own scaled hulls."""
    b8, lib, sb = scene
    draw = np.array([[2, 1, 2, 3, 4, 5, 6, 7]])
    scale = np.array([[0.7, 1.0, 1.45, 1.0, 1.0, 1.0, 1.0, 1.0]])
    rows, sc = _scene_rows(sb, lib, draw, scale)
    g0, g2 = sc.geoms[0][:29], sc.geoms[2][:29]
    assert np.array_equal(rows["geom_dataid"][0][g0], rows["geom_dataid"][0][g2])
    assert np.all(rows["geom_mesh_scale"][0][g0] == 0.7) and np.all(rows["geom_mesh_scale"][0][g2] == 1.45)
    mass = rows["body_mass"][0]
    assert np.isclose(mass[sc.bodies[2]] / mass[sc.bodies[0]], (1.45 / 0.7) ** 3, rtol=1e-12)
    pos = rows["geom_pos"][0].reshape(-1, 3)
    assert np.allclose(pos[g2] * 0.7, pos[g0] * 1.45, rtol=1e-12, atol=1e-15)
    c = rms.compact_model(b8, lib, draw[0], scale[0])
    p0, _, h0 = _object_rows(c, 0)
    p2, _, h2 = _object_rows(c, 2)
    mc = modelblob.unpack(c)
    assert mc["nmesh"] == modelblob.unpack(b8)["nmesh"] + 2 * 29         # two scaled copies of the 29 hulls, after the base's meshes
    for a, b, h in zip(h0, h2, lib.entries[2].hulls):
        assert np.allclose(a, 0.7 * h.vert, rtol=1e-15) and np.allclose(b, 1.45 * h.vert, rtol=1e-15)
    assert np.allclose(p2["geom_aabb"] * 0.7, p0["geom_aabb"] * 1.45, rtol=1e-12, atol=1e-15)


def test_place_rests_objects_by_their_scaled_lowest_point(scene):
    _, lib, sb = scene
    import torch

    draw = np.array([[0, 1, 2, 3, 4, 5, 6, -1]] * 2)
    scale = np.array([[1.5] * 8, [0.6] * 8])
    _, sc = _scene_rows(sb, lib, draw, scale)
    sc.place(torch.zeros(2, 8, 2), torch.zeros(2, 8), TABLE_TOP, clearance=0.0)
    for k in range(7):
        z = sc.sim.qpos[:, sc.qadr[k] + 2].numpy()
        assert np.allclose(z, TABLE_TOP - scale[:, k] * lib.entries[k].lowest_point(), atol=1e-6), k


# ---------------------------------------------------------------------------------------------- emulation against the oracle
def _reset(om, d, m, names, lib, draw, scale, lift=0.002):
    """test_mesh_scene's reset with each drawn object resting by its scaled lowest hull point"""
    tms._reset(om, d, m, names, lib, draw)
    adr = lambda i: int(m["jnt_qposadr"][names["joint"].index(f"object{i}:joint")])
    for i in range(8):
        if draw[i] >= 0:
            d.qpos[adr(i) + 2] = TABLE_TOP - scale[i] * lib.entries[draw[i]].lowest_point() + lift
    d.warning[:] = 0


def _rollout(blob, lib, draw, scale, n, settle):
    """test_mesh_scene's oracle rollout (settle, then n teacher-forcing states of 20 substeps each) from the scaled reset"""
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    om, d = oracle_pair(blob)
    _reset(om, d, m, names, lib, draw, scale)
    eqd = om.field("eq_data").copy()
    for _ in range(settle):
        d.step()
    p0 = d.mocap_pos[:3].copy()
    lo, hi = m["actuator_ctrlrange"].reshape(-1, 2)[0]
    rng = np.random.RandomState(0)
    states, after = [], []
    for k in range(n):
        a = 0.15 * k
        d.mocap_pos[:3] = p0 + [0.03 * np.sin(a), 0.04 * (1 - np.cos(a)), -0.03 * np.sin(0.5 * a)]
        d.ctrl[0] = rng.uniform(lo, hi)
        states.append((d.qpos.copy(), d.qvel.copy(), d.ctrl.copy(), d.userdata[:3].copy(), d.qacc_warmstart.copy(),
                       d.mocap_pos[:3].copy(), d.mocap_quat[:4].copy()))
        for _ in range(20):
            d.step()
        d.forward()
        after.append((d.qpos.copy(), d.qvel.copy(), int(d.ncon[0])))
    assert d.warning[0] == 0
    return states, after, eqd


def _emu_scene(sb, lib, draw, scale, nenv, bind=True):
    """tms._emu_scene with the draw's scaled rows and (bind=True) its geom_mesh_scale row"""
    e = tms._emu_scene(sb, lib, draw, nenv)
    rows, _ = _scene_rows(sb, lib, np.array([draw]), np.array([scale]))
    for f in rms.SCENE_GEOM_FIELDS + rms.BODY_FIELDS:
        e.model_field(f, np.float32)[:] = rows[f][0]
    for k, v in e.set_const().items():
        if k in rms.SET_CONST_FIELDS:
            e.model_field(k, np.float32)[:] = v
    row = rows["geom_mesh_scale"][0]
    assert e.use_geom_scale(row if bind else None) == len(row)
    return e


DRAW = [None, 1, 2, 3, 2, 5, 6, 7]                  # slot 0: the 41-part object; the 29-part object twice, at two scales
SCALE = [0.8, 1.25, 0.7, 1.15, 1.3, 0.9, 1.2, 0.75]


def test_emulated_scaled_slots_match_oracle_on_the_compact_model(scene):
    b8, lib, sb = scene
    draw = list(DRAW)
    draw[0] = lib.identity[1][0]
    c = rms.compact_model(b8, lib, draw, SCALE)
    mc, nc = modelblob.unpack(c), modelblob.unpack_names(c)
    states, after, eqd = _rollout(c, lib, draw, SCALE, 4, settle=300)
    e = _emu_scene(sb, lib, draw, SCALE, len(states))
    e.model_field("eq_data", np.float32)[:] = eqd
    for k, st in enumerate(states):
        e.qpos[k], e.qvel[k], e.ctrl[k], e.pid[k], e.warm[k] = st[:5]
        e.mocap_pos[k, 0], e.mocap_quat[k, 0] = st[5], st[6]
    e.step(20, 1)
    arm, obj = tms._errors(e.qpos, after, mc, nc)
    assert e.warn.max() == 0
    assert arm.max() < 1e-4 and np.median(obj) < 1e-4, (arm.max(), np.median(obj), obj.max())
    assert np.mean(np.abs(e.ncon - np.array([a[2] for a in after])) <= 2) > 0.8


def test_contact_that_only_the_scaled_hull_makes(scene):
    """The cracker box (slot 0) at s = 1.2, 1 mm into the table: its scaled hull touches the table box, the unscaled one --
    and the unscaled geom box that an OBB cull ignoring geom_mesh_scale would test -- are 2 cm above it.  The kernel finds the
    contacts the oracle finds on the compact model; without the geom_mesh_scale row it finds none."""
    b8, lib, sb = scene
    draw, scale = list(lib.identity[0]), [1.2] + [1.0] * 7
    assert lib.entries[draw[0]].nparts == 1
    c = rms.compact_model(b8, lib, draw, scale)
    mc, nc = modelblob.unpack(c), modelblob.unpack_names(c)
    om, d = oracle_pair(c)
    _reset(om, d, mc, nc, lib, draw, scale)
    a0 = int(mc["jnt_qposadr"][nc["joint"].index("object0:joint")])
    d.qpos[a0 + 2] = TABLE_TOP - 1.2 * lib.entries[draw[0]].lowest_point() - 0.001
    d.forward()
    obj_c = set(np.nonzero(mc["geom_bodyid"] == nc["body"].index("object0"))[0])
    table_c = nc["geom"].index("table")
    con = d.contact.reshape(-1, 24)[:int(d.ncon[0])]
    want = sorted(r[0] for r in con if {int(r[20]), int(r[21])} in ({g, table_c} for g in obj_c))
    assert want and np.allclose(want, -0.001, atol=2e-4)
    ms, ns = modelblob.unpack(sb), modelblob.unpack_names(sb)
    part, table = int(np.nonzero(ms["geom_bodyid"] == ns["body"].index("object0"))[0][0]), ns["geom"].index("table")
    # the pair's boxes in the world (object upright, unrotated): the scaled one reaches into the table top, the unscaled one not
    rows, _ = _scene_rows(sb, lib, np.array([draw]), np.array([scale]))
    A = rms._quat2mat(rows["geom_quat"][0].reshape(-1, 4)[part])
    gpos = np.array([0, 0, d.qpos[a0 + 2]]) + rows["geom_pos"][0].reshape(-1, 3)[part]
    ab = rows["geom_aabb"][0].reshape(-1, 6)[part]
    zmin = lambda s: (gpos + A @ (s * ab[:3]))[2] - np.abs(A[2]) @ (s * ab[3:])
    assert zmin(1.2) < TABLE_TOP < TABLE_TOP + 0.015 < zmin(1.0)
    got = []
    for bind in (True, False):
        e = _emu_scene(sb, lib, draw, scale, 1, bind=bind)
        e.qpos[0] = d.qpos
        e.mocap_pos[0, 0], e.mocap_quat[0, 0] = d.mocap_pos[:3], d.mocap_quat[:4]
        e.forward()
        n = int(e.ncon[0])
        got.append(sorted(float(r[2]) for r in e.contact[0, :n] if {int(r[0]), int(r[1])} == {part, table}))
    assert len(got[0]) == len(want) and np.allclose(got[0], want, atol=2e-5), (got[0], want)
    assert got[1] == []


# ---------------------------------------------------------------------------------------------- resting on the table
# A 3 x 3 grid on the table with the cell below the arm (x 1.22, y 0.20: the elbow link reaches down to 0.54 m and the gripper
# hangs at x 1.32, y 0.45) left empty.  Objects up to 1.65 x their size stay apart and clear of the arm there; in the cell below
# the arm the cracker box at 1.5 (0.32 m tall) starts inside the elbow link and is knocked over, on the oracle as on the GPU.
REST_XY = [[1.22 + 0.32 * (k % 3), 0.20 + 0.57 * (k // 3)] for k in range(1, 9)]
REST_STEPS = 50
# the base draw at 1.5, at 0.6, and with both scales side by side (the rearrange_ycb8_tcp draw is left out: its round one-part
# objects rock in place at any scale, by up to 0.1 rad on the oracle)
REST_SCALES = ([1.5] * 8, [0.6] * 8, [1.5, 0.6] * 4)


def _oracle_rest(blob, lib, draw, scale, n=REST_STEPS):
    """the resting reset (_rest_reset) on the oracle: poses of the object bodies [8, 7] at the start and after n env-steps"""
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    om, d = oracle_pair(blob)
    d.reset()
    om.field("eq_data")[:7] = [0, 0, 0, 1, 0, 0, 0]
    d.qpos[:6] = ARM_INIT
    adr = [int(m["jnt_qposadr"][names["joint"].index(f"object{i}:joint")]) for i in range(8)]
    for i in range(8):
        d.qpos[adr[i]:adr[i] + 7] = [*REST_XY[i], TABLE_TOP - scale[i] * lib.entries[draw[i]].lowest_point() + 1e-3, 1, 0, 0, 0]
    d.forward()
    tcp = names["body"].index("robot0:gripper_tcp")
    d.mocap_pos[:3] = d.xpos[3 * tcp:3 * tcp + 3]
    d.mocap_quat[:4] = d.xquat[4 * tcp:4 * tcp + 4]
    d.ctrl[:] = m["actuator_ctrlrange"].reshape(-1, 2)[:, 1]
    pose = lambda: np.array([d.qpos[a:a + 7] for a in adr])
    p0 = pose()
    for _ in range(n):
        for _ in range(20):
            d.step()
    d.forward()
    assert d.warning[0] == 0
    return p0, pose()


def _at_rest(p0, p1):
    """largest displacement and rotation angle of the objects between two poses ([..., 7]: position, quaternion)"""
    dq = np.clip(np.abs((p0[..., 3:] * p1[..., 3:]).sum(-1)), 0.0, 1.0)
    return np.abs(p1[..., :3] - p0[..., :3]).max(), float((2 * np.arccos(dq)).max())


def test_oracle_rests_scaled_objects_placed_clear_of_the_arm(scene):
    """The resting reset of the GPU test below on the oracle, on compact models with literally scaled hulls: after 50 env-steps
    every object is where it was put, less the 1 mm clearance it falls, and unrotated.  (The objects' velocities do not settle
    to zero: contact jitter leaves up to about 0.5 rad/s on some of them at every scale, 1 included.)"""
    b8, lib, _ = scene
    for scale in REST_SCALES:
        dx, da = _at_rest(*_oracle_rest(rms.compact_model(b8, lib, lib.identity[0], scale), lib, lib.identity[0], scale))
        assert dx < 3e-3 and da < 0.02, (scale, dx, da)


# ---------------------------------------------------------------------------------------------- GPU
def _scaled_place(sc, sim, rng=None):
    import torch

    xy = torch.tensor([[1.25 + 0.27 * (k % 3), 0.32 + 0.36 * (k // 3)] for k in (0, 1, 2, 3, 5, 6, 7, 8)], device=sim.device).expand(sim.nenv, 8, 2)
    yaw = torch.zeros(sim.nenv, 8, device=sim.device) if rng is None else torch.as_tensor(rng.uniform(-np.pi, np.pi, (sim.nenv, 8)), device=sim.device)
    sc.place(xy, yaw, TABLE_TOP)


def _rest_reset(model, sim, sc):
    """tools/mesh_scene_bench.py's reset: mocap weld at identity, the arm at its start pose holding still on the mocap body, the
    gripper command at its upper limit, and the objects resting on the table by their scaled lowest hull points, unrotated, on
    REST_XY"""
    import torch

    m, names = model.host, modelblob.unpack_names(model.blob)
    eq = np.array(m["eq_data"], dtype=np.float64).reshape(-1, 7)
    eq[0] = [0, 0, 0, 1, 0, 0, 0]
    model.set_field("eq_data", eq.reshape(-1))
    sim.qpos[:, :6] = torch.tensor(ARM_INIT, dtype=torch.float32, device=sim.device)
    sc.place(torch.tensor(REST_XY, device=sim.device).expand(sim.nenv, 8, 2), torch.zeros(sim.nenv, 8, device=sim.device), TABLE_TOP)
    sim.forward()
    tcp = names["body"].index("robot0:gripper_tcp")
    sim.mocap_pos[:, 0].copy_(sim.body_xpos[:, tcp]); sim.mocap_quat[:, 0].copy_(sim.body_xquat[:, tcp])
    sim.ctrl.copy_(torch.tensor(m["actuator_ctrlrange"].reshape(-1, 2)[:, 1], dtype=torch.float32, device=sim.device).expand_as(sim.ctrl))
    sim.qvel.zero_(); sim.pid.zero_(); sim.qacc_warmstart.zero_(); sim.warn.zero_()


@pytest.mark.gpu
def test_cuda_sixteen_scaled_draws_match_sixteen_compact_oracles(scene):
    import torch

    b8, lib, sb = scene
    rng = np.random.RandomState(7)
    draws = rng.randint(0, len(lib.entries), (16, 8))
    scales = rng.uniform(0.6, 1.6, (16, 8))
    draws[3, 2] = -1
    draws[5, 1] = draws[5, 6] = 2                  # one object twice in one environment, at two scales
    scales[5, 1], scales[5, 6] = 0.65, 1.5
    states, after = [], []
    for draw, scale in zip(draws, scales):
        st, af, eqd = _rollout(rms.compact_model(b8, lib, draw, scale), lib, draw, scale, 1, settle=300)
        states += st; after += af
    _, model, sim = tms._gpu_batch(sb, 16, outputs=("ncon", "warn"), **CAPS)
    model.set_field("eq_data", eqd)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draws, scales)
    tms._load_states(sim, states)
    sim.step()
    torch.cuda.synchronize()
    q = sim.qpos.cpu().numpy()
    ms, ns = modelblob.unpack(sb), modelblob.unpack_names(sb)
    arm = np.array([np.abs(q[i][:8] - after[i][0][:8]).max() for i in range(16)])
    obj = np.concatenate([tms._errors(q[i:i + 1], after[i:i + 1], ms, ns, [k for k in range(8) if draws[i, k] >= 0])[1] for i in range(16)])
    assert int(sim.warn.max()) == 0
    assert arm.max() < 1e-4 and np.median(obj) < 1e-4, (arm.max(), np.median(obj), obj.max())
    assert np.mean(np.abs(sim.ncon.cpu().numpy() - np.array([a[2] for a in after])) <= 2) > 0.8


@pytest.mark.gpu
def test_cuda_unit_geom_mesh_scale_row_is_bit_identical(scene):
    import torch

    b8, lib, sb = scene
    rng = np.random.RandomState(11)
    draws = rng.randint(0, len(lib.entries), (32, 8))
    out = []
    for bind in (False, True):
        _, model, sim = tms._gpu_batch(sb, 32, outputs=("ncon", "warn", "contact"), **CAPS)
        sc = rms.BatchedMeshScene(sim, lib)
        sc.set_objects(draws)
        if bind:
            sim.set_param("geom_mesh_scale", np.ones((32, model.host["ngeom"])))
        sim.qpos[:, :6] = torch.tensor(ARM_INIT, dtype=torch.float32, device=sim.device)
        _scaled_place(sc, sim, np.random.RandomState(1))
        for _ in range(3):
            sim.step()
        torch.cuda.synchronize()
        out.append([t.cpu().numpy().copy() for t in (sim.qpos, sim.qvel, sim.contact, sim.ncon)])
    for a, b in zip(*out):
        assert np.array_equal(a, b)


def test_emulated_scale_path_sees_the_oracle_contacts_along_the_resting_run(scene):
    """Along the oracle's 50 env-steps of the resting reset at 1.5, a forward of the emulated kernel from the oracle's state finds
    the same contacts with geom_mesh_scale rows on the slotted model as with literally scaled hulls on the compact model: same
    count, same distances to fp32 round-off."""
    b8, lib, sb = scene
    draw, scale = lib.identity[0], REST_SCALES[0]
    c = rms.compact_model(b8, lib, draw, scale)
    mc = modelblob.unpack(c)
    om, d = oracle_pair(c)
    slotted = _emu_scene(sb, lib, draw, scale, 1)
    compact = pyemu.EmuBatch(c, {k: mc[k] for k in modelblob.DIMS}, 1, **CAPS)
    p0, _ = _oracle_rest(c, lib, draw, scale, n=0)
    # replay the oracle's run: _oracle_rest's reset, then env-steps, forwarding both emulated models from every state
    m, names = modelblob.unpack(c), modelblob.unpack_names(c)
    d.reset()
    om.field("eq_data")[:7] = [0, 0, 0, 1, 0, 0, 0]
    d.qpos[:6] = ARM_INIT
    adr = [int(m["jnt_qposadr"][names["joint"].index(f"object{i}:joint")]) for i in range(8)]
    for i in range(8):
        d.qpos[adr[i]:adr[i] + 7] = p0[i]
    for e in (slotted, compact):
        e.model_field("eq_data", np.float32)[:7] = [0, 0, 0, 1, 0, 0, 0]
    for k in range(REST_STEPS):
        got = []
        for e in (slotted, compact):
            e.qpos[0], e.qvel[0] = d.qpos, d.qvel
            e.forward()
            got.append(np.sort(e.contact[0, :int(e.ncon[0]), 2]))
        assert len(got[0]) == len(got[1]) and np.allclose(got[0], got[1], atol=2e-6), (k, got)
        for _ in range(20):
            d.step()


@pytest.mark.gpu
@pytest.mark.xfail(strict=False, reason="open: the fp32 engine does not hold the 8-object ycb scene at rest for 50 env-steps. "
                   "The oracle does (test_oracle_rests_scaled_objects_placed_clear_of_the_arm), and the scale path finds the "
                   "oracle's contacts (test_emulated_scale_path_sees_the_oracle_contacts_along_the_resting_run), but in "
                   "emulation the free run drifts by centimetres from the oracle even on compact models without "
                   "geom_mesh_scale, and at 1.5 a relative change of 5e-8 in the derived constants decides whether objects "
                   "stay within 3 cm or are thrown off the table (DESIGN.md section 8)")
def test_cuda_scaled_objects_rest_on_the_table(scene):
    """The base draw at 1.5, at 0.6 and at both, placed by place(), stays at rest on the table for 50 env-steps, where the
    oracle on the compact models leaves it"""
    import torch

    b8, lib, sb = scene
    draws = np.array([lib.identity[0]] * len(REST_SCALES))
    scales = np.array(REST_SCALES)
    _, model, sim = tms._gpu_batch(sb, len(draws), outputs=("ncon", "warn", "body_xpos", "body_xquat"), **CAPS)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draws, scales)
    _rest_reset(model, sim, sc)
    pose = lambda: torch.stack([sim.qpos[:, a:a + 7] for a in sc.qadr], 1).double().cpu().numpy()
    p0 = pose()
    for _ in range(REST_STEPS):
        sim.step()
    torch.cuda.synchronize()
    p1 = pose()
    assert int(sim.warn.max()) == 0
    for i in range(len(draws)):
        dx, da = _at_rest(p0[i], p1[i])
        assert dx < 3e-3 and da < 0.02, (i, dx, da)
        _, want = _oracle_rest(rms.compact_model(b8, lib, draws[i], scales[i]), lib, draws[i], scales[i])
        assert np.abs(p1[i, :, :3] - want[:, :3]).max() < 1e-3, (i, p1[i, :, :3] - want[:, :3])


def _diverged(sim):
    """environments whose state is no longer finite or that the engine flagged as a bad state (warning bit 2)"""
    return int((~sim.qpos.isfinite().all(1) | ((sim.warn & 4) != 0)).sum())


@pytest.mark.gpu
def test_cuda_batch_1024_scaled_random_draws_runs(scene):
    """1024 random draws resting on the table for 65 env-steps, with and without the reference's randomised object scales: no
    more environments diverge with scales than without"""
    import torch

    b8, lib, sb = scene
    rng = np.random.RandomState(9)
    draws = rng.randint(-1, len(lib.entries), (1024, 8))
    scales = lib.object_scales(draws, rms.sample_object_size_scales(1024, 8, 0.5, 0.5, generator=torch.Generator(device="cuda:0").manual_seed(2)))
    counts = {}
    for arm, scale in (("unscaled", None), ("scaled", scales)):
        _, model, sim = tms._gpu_batch(sb, 1024, outputs=("ncon", "warn", "body_xpos", "body_xquat"), **dict(CAPS, contact_capacity=256))
        sc = rms.BatchedMeshScene(sim, lib)
        sc.set_objects(draws, scale)
        _rest_reset(model, sim, sc)
        for _ in range(65):
            sim.step()
        torch.cuda.synchronize()
        assert int((sim.warn & ~(1 | 4)).max()) == 0
        counts[arm] = _diverged(sim)
        print("slotted ycb, 1024 random draws, %s: launch %s, mean active pairs %.0f, diverged %d"
              % (arm, sim.launch_info(), float(sim.pair_counts().float().mean()), counts[arm]))
    assert counts["scaled"] <= counts["unscaled"], counts
