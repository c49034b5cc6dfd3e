"""Per-environment YCB object draws (robogym_b200.rearrange_mesh_scene): the object library of the two committed ycb scenes, the
padded "slotted" model a batch shares, the per-draw "compact" model the reference would build, and on the engine the
per-environment geom_dataid rows and pair lists (rg_batch_update_pairs) that make a slotted batch step what the compact models
step."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import pyemu
from helpers import oracle_pair
from robogym_b200 import modelblob
from robogym_b200 import rearrange_mesh_scene as rms

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
ARM_INIT = np.deg2rad(np.array([135.0, -90.0, 135.0, -100.0, -240.0, 135.0]))   # robogym/robot/ur16e/arm_interface.py:27
TABLE_TOP = 0.453 + 0.03324
CAPS = dict(contact_capacity=64, row_capacity=128)
_mesh_lib = None


def _blob(name):
    return open(os.path.join(ASSETS, name + ".rgm"), "rb").read()


@pytest.fixture(scope="module")
def scene():
    b8, bt = _blob("rearrange_ycb8"), _blob("rearrange_ycb8_tcp")
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    return b8, lib, rms.slotted_model(b8, lib)


def emu_pairs_lib():
    """tests/emu_mesh: the device code's pair-list compaction, and per-environment lists on an emulation handle"""
    global _mesh_lib
    if _mesh_lib is None:
        here = os.path.join(ROOT, "tests", "emu_mesh")
        subprocess.check_call(["make", "-C", here, "-s"])
        L = ctypes.CDLL(os.path.join(here, "_build", "librg_emu_mesh.so"))
        L.rge_pairs.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_int)]
        L.rge_use_pairs.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        _mesh_lib = L
    return _mesh_lib


def _active_pairs(m, dataid):
    """the static pairs whose geoms are both enabled in a geom_dataid row (what rg_batch_update_pairs keeps), in order"""
    on = (np.asarray(m["geom_type"]) != rms.GEOM_MESH) | (np.asarray(dataid) >= 0)
    keep = on[m["pair_geom1"]] & on[m["pair_geom2"]]
    return m["pair_geom1"][keep], m["pair_geom2"][keep]


def _geom_labels(m, names):
    """geom -> label that survives the slot expansion: object<k>-<j> for the j-th part of object k, else the rank among the others"""
    out, other = [], 0
    part = {}
    for g in range(m["ngeom"]):
        b = names["body"][m["geom_bodyid"][g]] or ""
        if b.startswith("object"):
            j = part.get(b, 0)
            part[b] = j + 1
            out.append(f"{b}-{j}")
        else:
            out.append(("other", other))
            other += 1
    return out


# ---------------------------------------------------------------------------------------------- host: library and models
def test_library_holds_both_scenes_objects_once(scene):
    _, lib, _ = scene
    assert lib.part_counts[:8] == [1, 3, 29, 5, 6, 1, 13, 1]                 # rearrange_ycb8, in slot order
    assert [lib.part_counts[e] for e in lib.identity[1]] == [41, 1, 1, 1, 1, 1, 1, 6]   # rearrange_ycb8_tcp
    assert lib.identity[0] == list(range(8))
    # the tcp scene's five one-part objects are one object, and it has nothing in common with the ycb8 draw
    assert len(set(lib.identity[1][1:6])) == 1 and len(lib.entries) == 12 and lib.max_parts == 41
    assert not set(lib.identity[0]) & set(lib.identity[1])


def test_compact_model_of_the_identity_draw_is_the_base_scene(scene):
    b8, lib, _ = scene
    m0, m1 = modelblob.unpack(b8), modelblob.unpack(rms.compact_model(b8, lib, lib.identity[0]))
    assert all(m0[k] == m1[k] for k in modelblob.DIMS)
    for kind, name, _ in modelblob.ARRAYS:
        if kind == "I":
            assert np.array_equal(m0[name], m1[name]), name
        else:
            assert np.all(np.abs(m0[name] - m1[name]) <= 1e-7 * np.abs(m0[name])), name


def test_slotted_model_pairs_of_the_identity_draw_are_the_base_pairs(scene):
    b8, lib, sb = scene
    ms, ns = modelblob.unpack(sb), modelblob.unpack_names(sb)
    m0, n0 = modelblob.unpack(b8), modelblob.unpack_names(b8)
    P = lib.max_parts
    assert ms["ngeom"] == m0["ngeom"] - 59 + 8 * P
    for k in range(8):     # P contiguous parts per slot, named object<k>-<j>; the base object's parts enabled, the rest not
        b = ns["body"].index(f"object{k}")
        g = np.nonzero(ms["geom_bodyid"] == b)[0]
        assert len(g) == P and g[-1] - g[0] == P - 1 and ns["geom"][g[0]] == f"object{k}-0"
        assert ((ms["geom_dataid"][g] >= 0).sum(), (ms["geom_dataid"][g] < 0).sum()) == (lib.part_counts[k], P - lib.part_counts[k])
    p1, p2 = _active_pairs(ms, ms["geom_dataid"])
    ls, l0 = _geom_labels(ms, ns), _geom_labels(m0, n0)
    assert [(ls[a], ls[b]) for a, b in zip(p1, p2)] == [(l0[a], l0[b]) for a, b in zip(m0["pair_geom1"], m0["pair_geom2"])]
    # every pair of a disabled part is dropped, every other candidate pair of the padded model is in the list
    assert ms["npair"] > 10 * len(p1)


def test_emulated_pair_compaction_matches_the_host_rule(scene):
    b8, lib, sb = scene
    ms = modelblob.unpack(sb)
    e = pyemu.EmuBatch(sb, {k: ms[k] for k in modelblob.DIMS}, 1)
    L = emu_pairs_lib()
    rng = np.random.RandomState(3)
    for draw in ([2] * 8, list(rng.randint(0, len(lib.entries), 8))):
        rows, _ = _scene_rows(sb, lib, np.array([draw]))
        did = rows["geom_dataid"][0].astype(np.int32)
        out = np.zeros(ms["npair"], np.uint32)
        w = ctypes.c_int()
        n = L.rge_pairs(e.h, did.ctypes.data, out.ctypes.data, len(out), ctypes.byref(w))
        p1, p2 = _active_pairs(ms, did)
        assert w.value == 0 and n == len(p1)
        assert np.array_equal(out[:n] & 0xffff, p1) and np.array_equal(out[:n] >> 16, p2)
        small = np.zeros(100, np.uint32)                  # a list that is too short: truncated in order, warning bit 6
        assert L.rge_pairs(e.h, did.ctypes.data, small.ctypes.data, 100, ctypes.byref(w)) == 100 and w.value == 64
        assert np.array_equal(small, out[:100])
    did[0] = 7                                            # an id on a geom that is not a mesh: disabled, warning bit 7
    n = L.rge_pairs(e.h, did.ctypes.data, out.ctypes.data, len(out), ctypes.byref(w))
    assert w.value == 128 and not np.any((out[:n] & 0xffff) == 0) and not np.any((out[:n] >> 16) == 0)


# ---------------------------------------------------------------------------------------------- BatchedMeshScene on the host
class _RecordingSim:
    """what BatchedMeshScene needs of a BatchedSim, recording the rows it writes"""

    def __init__(self, blob, nenv):
        import torch

        self.torch, self.nenv = torch, nenv
        self.model = type("M", (), {})()
        self.model.host = modelblob.unpack(blob)
        names = modelblob.unpack_names(blob)

        def name2id(typ, name):
            if name not in names[typ]:
                raise ValueError(name)
            return names[typ].index(name)
        self.model.name2id = name2id
        self.params, self.calls = {}, []
        self.qpos = torch.zeros(nenv, self.model.host["nq"], dtype=torch.float32)
        self.qvel = torch.zeros(nenv, self.model.host["nv"], dtype=torch.float32)

    def set_param(self, name, v):
        self.params[name] = np.array(v)

    def set_const(self, fields=()):
        self.calls.append(("set_const", tuple(fields)))

    def update_pairs(self, mask=None):
        self.calls.append(("update_pairs", mask))


def _scene_rows(sb, lib, draw):
    sim = _RecordingSim(sb, len(draw))
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draw)
    return sim.params, sc


def _draws(lib):
    t = lib.identity[1]
    return np.array([lib.identity[0], [2, 2, 2, 2, 2, 2, 2, 2], [t[0], 1, -1, 3, t[7], 5, t[6], 2],
                     [11, 10, 9, 8, 7, 6, 5, 4]])


def test_scene_rows_are_the_compact_models_rows(scene):
    b8, lib, sb = scene
    draws = _draws(lib)
    rows, sc = _scene_rows(sb, lib, draws)
    assert sc.sim.calls == [("set_const", rms.SET_CONST_FIELDS), ("update_pairs", None)]
    ms = modelblob.unpack(sb)
    for i, draw in enumerate(draws):
        mc, nc = modelblob.unpack(c := rms.compact_model(b8, lib, draw)), modelblob.unpack_names(c)
        for k in range(8):
            b = nc["body"].index(f"object{k}")
            gc = np.nonzero(mc["geom_bodyid"] == b)[0]
            gs = sc.geoms[k]
            n = lib.entries[draw[k]].nparts if draw[k] >= 0 else 0
            assert len(gc) == n
            did = rows["geom_dataid"][i, gs]
            assert np.all(did[n:] == -1) and np.all(did[:n] >= 0)
            for j in range(n):
                assert rms.Hull.of(ms, did[j]).key == rms.Hull.of(mc, mc["geom_dataid"][gc[j]]).key
            for f in rms.SCENE_GEOM_FIELDS:
                w = rms._rows(ms, f, "ngeom").shape[1]
                assert np.array_equal(rows[f][i].reshape(-1, w)[gs[:n]], rms._rows(mc, f, "ngeom")[gc]), (i, k, f)
            if n:
                for f in rms.BODY_FIELDS:
                    w = rms._rows(ms, f, "nbody").shape[1]
                    assert np.array_equal(rows[f][i].reshape(-1, w)[sc.bodies[k]], rms._rows(mc, f, "nbody")[b]), (i, k, f)


def test_empty_slot_keeps_the_shared_body_rows_after_a_redraw(scene):
    b8, lib, sb = scene
    sim = _RecordingSim(sb, 2)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(np.array([[11] * 8, [2] * 8]))
    sc.set_objects(np.array([[-1] * 8, [2, -1, 2, -1, 2, -1, 2, -1]]))
    ms = modelblob.unpack(sb)
    for f in rms.BODY_FIELDS:
        rows = sim.params[f].reshape(2, ms["nbody"], -1)
        for k in range(8):
            shared = rms._rows(ms, f, "nbody")[sc.bodies[k]]
            assert np.array_equal(rows[0, sc.bodies[k]], shared), (f, k)       # all empty after a draw of object 11
            if k % 2:
                assert np.array_equal(rows[1, sc.bodies[k]], shared), (f, k)   # emptied after holding object 2


def test_library_refuses_objects_whose_shared_rows_differ(scene):
    b8, _, _ = scene
    m, names = modelblob.unpack(b8), modelblob.unpack_names(b8)
    g = int(np.nonzero(m["geom_bodyid"] == names["body"].index("object3"))[0][0])
    m["geom_friction"].reshape(-1, 3)[g, 0] = 0.5           # a material a draw would not carry into the environment's rows
    with pytest.raises(ValueError, match="geom_friction"):
        rms.ObjectLibrary.from_blobs(b8, modelblob.pack(m, names))


# ---------------------------------------------------------------------------------------------- oracle and emulation
def _reset(om, d, m, names, lib, draw):
    """test_rearrange_ycb's reset for any draw: arm at its initial pose, the drawn objects on the table by their lowest hull
    point, the empty slots parked on the floor"""
    adr = lambda i: int(m["jnt_qposadr"][names["joint"].index(f"object{i}:joint")])
    d.reset()
    d.qpos[:6] = ARM_INIT
    for i in range(8):
        d.qpos[adr(i):adr(i) + 3] = [1.0 + 0.25 * (i % 4), 1.1 + 0.3 * (i // 4), 0.8]
    d.forward()
    tcp = names["body"].index("robot0:gripper_tcp")
    om.field("eq_data")[:7] = [0, 0, 0, 1, 0, 0, 0]
    d.mocap_pos[:3] = d.xpos[3 * tcp:3 * tcp + 3]
    d.mocap_quat[:4] = d.xquat[4 * tcp:4 * tcp + 4]
    for i in range(8):
        k = i if i < 4 else i + 1
        if draw[i] >= 0:
            d.qpos[adr(i):adr(i) + 3] = [1.25 + 0.27 * (k % 3), 0.32 + 0.36 * (k // 3), TABLE_TOP - lib.entries[draw[i]].lowest_point() + 0.002]
        else:
            d.qpos[adr(i):adr(i) + 3] = [3.0 + 0.25 * (i % 4), -1.0 + 0.25 * (i // 4), 0.0]
    d.warning[:] = 0


def _rollout(blob, lib, draw, n, settle):
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    om, d = oracle_pair(blob)
    _reset(om, d, m, names, lib, draw)
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
    return states, after, eqd, d


def _errors(q, after, m, names, slots=range(8)):
    adr = lambda i: int(m["jnt_qposadr"][names["joint"].index(f"object{i}:joint")])
    arm = np.array([np.abs(q[k][:8] - after[k][0][:8]).max() for k in range(len(after))])
    obj = np.array([max(np.abs(q[k][adr(i):adr(i) + 3] - after[k][0][adr(i):adr(i) + 3]).max() for i in slots) for k in range(len(after))])
    return arm, obj


def test_oracle_rests_the_29_part_object_in_several_slots_on_the_table(scene):
    b8, lib, _ = scene
    draw = [2, 1, 2, 3, 2, 5, 6, 7]
    c = rms.compact_model(b8, lib, draw)
    m, names = modelblob.unpack(c), modelblob.unpack_names(c)
    _, after, _, d = _rollout(c, lib, draw, 2, settle=800)
    for i in range(8):
        z = d.qpos[int(m["jnt_qposadr"][names["joint"].index(f"object{i}:joint")]) + 2]
        assert TABLE_TOP < z < TABLE_TOP + 0.12, (i, z)
    assert after[-1][2] >= 15


def _emu_scene(sb, lib, draw, nenv):
    """an emulation batch of the slotted model holding one draw: the scene's rows written into the model, the derived
    constants recomputed through the kernel code, and the draw's own pair list"""
    ms = modelblob.unpack(sb)
    e = pyemu.EmuBatch(sb, {k: ms[k] for k in modelblob.DIMS}, nenv, **CAPS)
    rows, _ = _scene_rows(sb, lib, np.array([draw]))
    e.model_field("geom_dataid", np.int32)[:] = rows["geom_dataid"][0]
    for f in rms.SCENE_GEOM_FIELDS + rms.BODY_FIELDS:
        e.model_field(f, np.float32)[:] = rows[f][0]
    for k, v in e.set_const().items():
        if k in rms.SET_CONST_FIELDS:
            e.model_field(k, np.float32)[:] = v
    L = emu_pairs_lib()
    lst = np.zeros(ms["npair"], np.uint32)
    w = ctypes.c_int()
    did = rows["geom_dataid"][0].astype(np.int32)
    n = L.rge_pairs(e.h, did.ctypes.data, lst.ctypes.data, len(lst), ctypes.byref(w))
    assert w.value == 0
    L.rge_use_pairs(e.h, lst.ctypes.data, n)
    e._pairs = lst                                         # alive as long as the batch
    return e


def test_emulated_slotted_kernel_matches_oracle_on_the_compact_model(scene):
    b8, lib, sb = scene
    draw = [lib.identity[1][0], 1, 2, 3, lib.identity[1][7], 5, 6, 2]
    c = rms.compact_model(b8, lib, draw)
    mc, nc = modelblob.unpack(c), modelblob.unpack_names(c)
    states, after, eqd, _ = _rollout(c, lib, draw, 6, settle=300)
    e = _emu_scene(sb, lib, draw, len(states))
    e.model_field("eq_data", np.float32)[:] = eqd
    for k, st in enumerate(states):
        e.qpos[k], e.qvel[k], e.ctrl[k], e.pid[k], e.warm[k] = st[:5]
        e.mocap_pos[k, 0], e.mocap_quat[k, 0] = st[5], st[6]
    e.step(20, 1)
    arm, obj = _errors(e.qpos, after, mc, nc)
    assert e.warn.max() == 0
    assert arm.max() < 1e-4 and np.median(obj) < 1e-4, (arm.max(), np.median(obj), obj.max())
    assert np.mean(np.abs(e.ncon - np.array([a[2] for a in after])) <= 2) > 0.8


# ---------------------------------------------------------------------------------------------- GPU
def _gpu_batch(sb, nenv, **kw):
    from robogym_b200 import build, engine

    build.build()
    model = engine.DeviceModel(sb, 0)
    return engine, model, engine.BatchedSim(model, nenv, 20, **kw)


def _load_states(sim, states):
    import torch

    f = lambda i: torch.tensor(np.stack([s[i] for s in states]), dtype=torch.float32, device=sim.device)
    sim.qpos.copy_(f(0)); sim.qvel.copy_(f(1)); sim.ctrl.copy_(f(2)); sim.pid.copy_(f(3)); sim.qacc_warmstart.copy_(f(4))
    sim.mocap_pos[:, 0].copy_(f(5)); sim.mocap_quat[:, 0].copy_(f(6))


@pytest.mark.gpu
def test_cuda_sixteen_draws_match_sixteen_compact_oracles(scene):
    import torch

    b8, lib, sb = scene
    rng = np.random.RandomState(5)
    draws = rng.randint(0, len(lib.entries), (16, 8))
    draws[3, 2] = -1
    states, after = [], []
    for draw in draws:
        st, af, eqd, _ = _rollout(rms.compact_model(b8, lib, draw), lib, draw, 1, settle=300)
        states += st; after += af
    _, model, sim = _gpu_batch(sb, 16, outputs=("ncon", "warn"), **CAPS)
    model.set_field("eq_data", eqd)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draws)
    _load_states(sim, states)
    sim.step()
    torch.cuda.synchronize()
    q = sim.qpos.cpu().numpy()
    ms, ns = modelblob.unpack(sb), modelblob.unpack_names(sb)
    arm = np.array([np.abs(q[i][:8] - after[i][0][:8]).max() for i in range(16)])
    obj = np.concatenate([_errors(q[i:i + 1], after[i:i + 1], ms, ns, [k for k in range(8) if draws[i, k] >= 0])[1] for i in range(16)])
    assert int(sim.warn.max()) == 0
    assert arm.max() < 1e-4 and np.median(obj) < 1e-4, (arm.max(), np.median(obj), obj.max())
    assert np.mean(np.abs(sim.ncon.cpu().numpy() - np.array([a[2] for a in after])) <= 2) > 0.8


@pytest.mark.gpu
def test_cuda_identity_draw_on_the_slotted_model_steps_like_the_plain_scene(scene):
    import torch

    b8, lib, sb = scene
    states, after, eqd, _ = _rollout(b8, lib, lib.identity[0], 8, settle=200)
    engine, model, sim = _gpu_batch(sb, 8, outputs=("ncon", "warn"), **CAPS)
    model.set_field("eq_data", eqd)
    rms.BatchedMeshScene(sim, lib).set_objects(np.array([lib.identity[0]] * 8))
    plain_model = engine.DeviceModel(b8, 0)
    plain_model.set_field("eq_data", eqd)
    plain = engine.BatchedSim(plain_model, 8, 20, outputs=("ncon", "warn"), **CAPS)
    for s in (sim, plain):
        _load_states(s, states)
        s.step()
    torch.cuda.synchronize()
    assert int(sim.warn.max()) == 0 and int(plain.warn.max()) == 0
    # the same pairs in the same order; the constants differ in the last bits (recomputed in fp32 on the device), so both are
    # held to the oracle's tolerance rather than to each other's bits
    m, names = modelblob.unpack(b8), modelblob.unpack_names(b8)
    for s in (sim, plain):
        arm, obj = _errors(s.qpos.cpu().numpy(), after, m, names)
        assert arm.max() < 1e-4 and np.median(obj) < 1e-4, (arm.max(), np.median(obj), obj.max())
    assert np.mean(np.abs(sim.ncon.cpu().numpy() - plain.ncon.cpu().numpy()) <= 2) > 0.8
    counts = sim.pair_counts().cpu().numpy()
    assert np.all(counts == modelblob.unpack(b8)["npair"])


@pytest.mark.gpu
def test_cuda_redraw_and_masked_update_leave_other_environments_alone(scene):
    import torch

    b8, lib, sb = scene
    states, _, eqd, _ = _rollout(b8, lib, lib.identity[0], 1, settle=200)
    _, model, sim = _gpu_batch(sb, 8, outputs=("ncon", "warn", "contact"), **CAPS)
    model.set_field("eq_data", eqd)
    sc = rms.BatchedMeshScene(sim, lib)
    draws = np.array([lib.identity[0]] * 8)
    sc.set_objects(draws)
    # rows written through set_param without update_pairs: the next step rederives the lists of exactly those rows, so no list
    # ever names a part its row has disabled
    ms = modelblob.unpack(sb)
    _, _, other = _gpu_batch(sb, 2, **CAPS)
    shared = np.asarray(ms["geom_dataid"])
    rows29 = _scene_rows(sb, lib, np.array([[2] * 8]))[0]["geom_dataid"][0]
    n_base, n29 = len(_active_pairs(ms, shared)[0]), len(_active_pairs(ms, rows29)[0])
    other.set_param("geom_dataid", np.stack([shared, rows29]))
    other.step()
    assert list(other.pair_counts().cpu().numpy()) == [n_base, n29]
    other.set_param("geom_dataid", shared[None], idx=[1])
    other.step()
    torch.cuda.synchronize()
    assert list(other.pair_counts().cpu().numpy()) == [n_base, n_base]
    assert int((other.warn & 192).max()) == 0              # no list overflow, no bad geom_dataid (qpos0 overfills the contacts)

    def run():
        _load_states(sim, states * 8)
        sim.step()
        torch.cuda.synchronize()
        return sim.qpos.cpu().numpy().copy(), sim.contact.cpu().numpy().copy(), sim.ncon.cpu().numpy().copy()

    q0, c0, n0 = run()
    # redraw environments 2 and 5 only, rows and pair lists
    draws2 = draws.copy()
    draws2[2] = draws2[5] = [2] * 8
    sc.set_objects(draws2)                                 # all rows rewritten; every list rederived
    q1, c1, n1 = run()
    keep = [0, 1, 3, 4, 6, 7]
    assert np.array_equal(q1[keep], q0[keep]) and np.array_equal(c1[keep], c0[keep]) and np.array_equal(n1[keep], n0[keep])
    counts = sim.pair_counts().cpu().numpy()
    assert counts[2] == counts[5] > counts[0]
    # environment 2's geom_dataid row back to the shared one and only its list rederived (masked): the others keep theirs
    sim.set_param("geom_dataid", np.asarray(modelblob.unpack(sb)["geom_dataid"])[None], idx=[2])
    mask = torch.zeros(8, dtype=torch.uint8, device=sim.device)
    mask[2] = 1
    sim.update_pairs(mask)
    counts2 = sim.pair_counts().cpu().numpy()
    assert counts2[2] == counts[0] and counts2[5] == counts[5] and np.array_equal(counts2[keep], counts[keep])
    q2, c2, n2 = run()
    keep5 = keep + [5]
    assert np.array_equal(q2[keep5], q1[keep5]) and np.array_equal(c2[keep5], c1[keep5]) and np.array_equal(n2[keep5], n1[keep5])


@pytest.mark.gpu
def test_cuda_object_gripper_contact_on_the_slotted_model(scene):
    import torch

    from robogym_b200.rearrange_contacts import BatchedRearrangeContacts

    b8, lib, sb = scene
    _, model, sim = _gpu_batch(sb, 4, outputs=("ncon", "warn", "contact"), **CAPS)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(np.array([lib.identity[0], [2] * 8, lib.identity[1], [11] * 8]))
    sim.qpos[:, :6] = torch.tensor(ARM_INIT, dtype=torch.float32, device=sim.device)
    xy = torch.tensor([[1.25 + 0.27 * (k % 3), 0.32 + 0.36 * (k // 3)] for k in (0, 1, 2, 3, 5, 6, 7, 8)], device=sim.device).expand(4, 8, 2)
    sc.place(xy, torch.zeros(4, 8, device=sim.device), TABLE_TOP)
    sim.forward()
    con = BatchedRearrangeContacts(sim, 8)
    out = con.object_gripper_contact()
    torch.cuda.synchronize()
    assert out.shape == (4, 8, 2) and not bool(out.any())   # objects on the table, gripper up in the air
    assert int(sim.warn.max()) == 0 and int(sim.ncon.min()) > 0
    # every one of the P part geoms of a slot belongs to that slot's object, drawn or not
    for k in range(8):
        assert bool((con.geom_object[torch.as_tensor(sc.geoms[k], device=sim.device)] == k).all())
    # a contact of the left pad with the last part of environment 1's 29-part object in slot 3 counts for object 3
    g = int(sc.geoms[3][lib.entries[2].nparts - 1])
    sim.contact[1, 0] = torch.tensor([float(con.pads[0]), float(g), 0.0, 3.0], device=sim.device)
    sim.ncon[1] = 1
    out = con.object_gripper_contact()
    assert bool(out[1, 3, 0]) and int(out.sum()) == 1


@pytest.mark.gpu
def test_cuda_batch_1024_random_draws_runs(scene):
    import torch

    b8, lib, sb = scene
    _, model, sim = _gpu_batch(sb, 1024, outputs=("ncon", "warn"), **CAPS)
    rng = np.random.RandomState(9)
    draws = rng.randint(-1, len(lib.entries), (1024, 8))
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draws)
    sim.qpos[:, :6] = torch.tensor(ARM_INIT, dtype=torch.float32, device=sim.device)
    xy = torch.tensor([[1.25 + 0.27 * (k % 3), 0.32 + 0.36 * (k // 3)] for k in (0, 1, 2, 3, 5, 6, 7, 8)], device=sim.device).expand(1024, 8, 2)
    sc.place(xy, torch.as_tensor(rng.uniform(-np.pi, np.pi, (1024, 8)), device=sim.device), TABLE_TOP)
    for _ in range(5):
        sim.step()
    torch.cuda.synchronize()
    assert int((sim.warn & ~1).max()) == 0
    info = sim.launch_info()
    counts = sim.pair_counts().float()
    print("slotted ycb, 1024 random draws: launch %s, mean active pairs %.0f" % (info, float(counts.mean())))
