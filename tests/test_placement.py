"""Reset-time placement of rearrange objects (robogym_b200/rearrange_placement.py, csrc/rg_place.inl): rotated bounding boxes of
object bodies (rg_batch_body_aabb) and the reference's grid, rejection and goal-distance placement (rg_place_objects).

The fixture tests/golden/reference_placement.json.gz holds the reference's own results (tools/make_placement_golden.py), drawn
from the same Philox counters as the kernel through a replay RandomState (tests/placement_rng.py).  The CPU tier runs the
kernel's code on the emulation build (tests/emu); the GPU tier runs it on the device."""
import gzip
import json
import os

import numpy as np
import pytest

import pyemu
import test_mesh_scene as tms
from placement_rng import ReplayRandomState, philox
from robogym_b200 import modelblob
from robogym_b200 import rearrange_mesh_scene as rms
from robogym_b200 import rearrange_placement as rp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_placement.json.gz")
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
MODES = rp.MODES


def _ptr(a):
    return None if a is None else a.ctypes.data


def emulated_place(bbox, active, table, area, mode, seed, epoch, anchor=None, ratio=1.0, dmin=0.06, mask=None, pos=None, max_trials=100, max_per_object=20):
    """the kernel's code on the emulation build: (pos [nenv, nobj, 3], status [nenv]; -1 where mask is 0)"""
    bbox = np.ascontiguousarray(bbox, dtype=np.float64)
    nenv, nobj = bbox.shape[:2]
    active = np.ascontiguousarray(np.broadcast_to(active, (nenv, nobj)), dtype=np.uint8)
    area = np.ascontiguousarray(np.broadcast_to(area, (nenv, 6)), dtype=np.float64)
    table = np.ascontiguousarray(table, dtype=np.float64)
    anchor = None if anchor is None else np.ascontiguousarray(anchor, dtype=np.float64)
    mask = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
    pos = np.zeros((nenv, nobj, 3)) if pos is None else pos
    status = np.full(nenv, -1, np.int32)
    pyemu.lib().rge_place(nenv, nobj, _ptr(bbox), _ptr(active), _ptr(table), _ptr(area), MODES[mode], max_trials, max_per_object, ratio, dmin,
                          _ptr(anchor), seed, epoch, _ptr(mask), _ptr(pos), _ptr(status))
    return pos, status


@pytest.fixture(scope="module")
def golden():
    return json.loads(gzip.decompress(open(GOLDEN, "rb").read()))


@pytest.fixture(scope="module")
def ycb():
    b8, bt = tms._blob("rearrange_ycb8"), tms._blob("rearrange_ycb8_tcp")
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    return b8, lib, rms.slotted_model(b8, lib)


def _case_inputs(c):
    """one fixture case as a batch: environment c["env"] of a batch holding it alone at that index"""
    n = c["env"] + 1
    nobj = len(c["bbox"])
    bbox = np.zeros((n, nobj, 2, 3)); bbox[-1] = c["bbox"]
    active = np.zeros((n, nobj), np.uint8); active[-1] = c["active"]
    area = np.zeros((n, 6)); area[-1] = c["area"]
    anchor = None
    if c["anchor"] is not None:
        anchor = np.zeros((n, nobj, 3)); anchor[-1] = c["anchor"]
    mask = np.zeros(n, np.uint8); mask[-1] = 1
    return bbox, active, area, anchor, mask


def _random_boxes(rng, nenv, nobj, lo=0.01, hi=0.1):
    size = rng.uniform(lo, hi, (nenv, nobj, 3))
    center = rng.uniform(-0.02, 0.02, (nenv, nobj, 3))
    return np.stack([center, size], axis=2)


# ---------------------------------------------------------------------------------------------- CPU
def test_philox_known_answers_and_replay_equals_emulated_device_philox():
    # Random123's known-answer vectors for Philox4x32-10
    kat = [((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
           ((0xFFFFFFFF,) * 4, (0xFFFFFFFF, 0xFFFFFFFF), (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
           ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))]
    for c, k, want in kat:
        assert tuple(int(x) for x in philox(c, *k)) == want
    rng = np.random.RandomState(3)
    ctr = rng.randint(0, 1 << 32, (4096, 4), dtype=np.uint64).astype(np.uint32)
    for k0, k1 in ((0, 0), (12345, 77), (0xFFFFFFFF, 4095)):
        out = np.zeros_like(ctr)
        pyemu.lib().rge_philox(len(ctr), _ptr(ctr), k0, k1, _ptr(out))
        assert np.array_equal(out, philox(ctr, k0, k1))


def test_replay_random_state_draws_what_it_documents():
    rs = ReplayRandomState(9, 4, 2)
    x = rs.uniform((0.1, 0.2), (0.5, 0.25))
    r = philox((0, 0, 1, 2), 9, 4)
    u0 = ((int(r[0]) >> 5) * 67108864.0 + (int(r[1]) >> 6)) / 2.0 ** 53
    assert x[0] == 0.1 + (0.5 - 0.1) * u0 and 0.2 <= x[1] < 0.25 and rs.proposals == 1
    a = np.arange(10)
    rs.shuffle(a)
    assert sorted(a.tolist()) == list(range(10)) and rs.shuffles == 1


def test_emulated_kernel_reproduces_every_reference_case(golden):
    modes = set()
    for i, c in enumerate(golden["cases"]):
        bbox, active, area, anchor, mask = _case_inputs(c)
        pos, st = emulated_place(bbox, active, golden["table"], area, c["mode"], c["seed"], c["epoch"], anchor, c["ratio"], c["dmin"], mask)
        assert st[-1] == c["status"], (i, c["mode"], st[-1], c["status"])
        assert np.abs(pos[-1] - np.array(c["pos"])).max() <= 1e-12, (i, pos[-1] - np.array(c["pos"]))
        assert (st[:-1] == -1).all() and not pos[:-1].any()
        modes.add((c["mode"], c["status"]))
    # every algorithm succeeds somewhere, the fallback engages, and a crowded case fails outright
    assert {("grid_then_uniform", 1), ("grid_then_uniform", 2), ("grid_then_uniform", 0), ("grid", 1), ("uniform", 2), ("goal_distance_ratio", 3)} <= modes


def test_placement_area_matches_the_reference(golden):
    table = rp.table_dimensions(open(os.path.join(ASSETS, "rearrange_blocks5.rgm"), "rb").read())
    assert np.allclose(np.concatenate(table[:2]), golden["table"], rtol=0, atol=0) and table[2] == golden["table_height"]
    for a in golden["areas"]:
        assert np.array_equal(rp.placement_area(table, a["num_objects"], a["portion"])[0], a["area"]), a
    n = np.array([a["num_objects"] for a in golden["areas"]])
    por = np.array([a["portion"] for a in golden["areas"]])
    assert np.array_equal(rp.placement_area(table, n, por), np.array([a["area"] for a in golden["areas"]]))
    # the reference's own literal areas for the blocks environment (envs/rearrange/tests/test_placement.py)
    literal = {1.0: ((0.3038, 0.38275, 0.06648), (0.6075, 0.58178, 0.26)), 0.8: ((0.3645, 0.44093, 0.06648), (0.486, 0.46542, 0.26)),
               0.6: ((0.4253, 0.49911, 0.06648), (0.3645, 0.3491, 0.26)), 0.4: ((0.486, 0.55728, 0.06648), (0.243, 0.23271, 0.26))}
    for portion, (off, size) in literal.items():
        a = rp.placement_area(table, 1, portion)[0]
        assert np.allclose(a[:3], off, atol=1e-4) and np.allclose(a[3:], size, atol=1e-4)


def test_emulated_boxes_match_the_reference_boxes(golden, ycb):
    b8, lib, sb = ycb
    L = pyemu.lib()
    yawq = lambda a: np.array([np.cos(0.5 * a), 0.0, 0.0, np.sin(0.5 * a)])
    nmesh = 0
    for b in golden["boxes"]:
        if b["kind"] == "block":
            blob = open(os.path.join(ASSETS, "rearrange_blocks5.rgm"), "rb").read()
            e = pyemu.EmuBatch(blob, {k: modelblob.unpack(blob)[k] for k in modelblob.DIMS}, 1)
            body = modelblob.unpack_names(blob)["body"].index(b["body"])
            out = np.zeros(6)
            L.rge_body_aabb(e.h, body, _ptr(yawq(b["yaw"])), None, None, None, None, None, None, _ptr(out))
            assert np.abs(out.reshape(2, 3) - np.array(b["bbox"])).max() < 1e-6, (b, out)
            continue
        nmesh += 1
        draw, scale, yaw = np.array(b["draw"]), np.array(b["scale"]), np.array(b["yaw"])
        # the compact model (literally scaled hulls) and the slotted model with the scene's per-environment rows
        c = rms.compact_model(b8, lib, draw, scale)
        mc, nc = modelblob.unpack(c), modelblob.unpack_names(c)
        ec = pyemu.EmuBatch(c, {k: mc[k] for k in modelblob.DIMS}, 1)
        ms, ns = modelblob.unpack(sb), modelblob.unpack_names(sb)
        es = pyemu.EmuBatch(sb, {k: ms[k] for k in modelblob.DIMS}, 1)
        rec = tms._RecordingSim(sb, 1)
        rms.BatchedMeshScene(rec, lib).set_objects(draw[None], scale[None])
        rows = rec.params
        did = np.ascontiguousarray(rows["geom_dataid"][0], dtype=np.int32)
        r = {f: np.ascontiguousarray(rows[f][0], dtype=np.float32) for f in ("geom_pos", "geom_quat", "geom_size", "geom_mesh_scale")}
        for k in range(8):
            want = np.array(b["bbox"][k])
            out = np.zeros(6)
            L.rge_body_aabb(ec.h, nc["body"].index(f"object{k}"), _ptr(yawq(yaw[k])), None, None, None, None, None, None, _ptr(out))
            assert np.abs(out.reshape(2, 3) - want).max() < 1e-6, (k, out.reshape(2, 3) - want)
            out2 = np.zeros(6)
            L.rge_body_aabb(es.h, ns["body"].index(f"object{k}"), _ptr(yawq(yaw[k])), _ptr(did), _ptr(r["geom_pos"]), _ptr(r["geom_quat"]),
                            _ptr(r["geom_size"]), None, _ptr(r["geom_mesh_scale"]), _ptr(out2))
            assert np.abs(out2.reshape(2, 3) - want).max() < 1e-6, (k, out2.reshape(2, 3) - want)
    assert nmesh >= 2


@pytest.mark.parametrize("mode", ["grid_then_uniform", "grid", "uniform", "goal_distance_ratio"])
def test_emulated_placements_hold_the_reference_invariants(mode):
    """over many seeds: no two active objects overlap under the reference's predicate, every object lies inside the area, each
    box's bottom sits on the table top, and inactive slots are untouched"""
    rng = np.random.RandomState({"grid_then_uniform": 1, "grid": 2, "uniform": 3, "goal_distance_ratio": 4}[mode])
    nenv, nobj = 256, 6
    table = np.array([1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2])          # table pos, half size (rearrange scenes)
    top = table[2] + table[5]
    bbox = _random_boxes(rng, nenv, nobj, 0.01, 0.07)
    active = rng.rand(nenv, nobj) < 0.75
    area = rp.placement_area((table[:3], table[3:], top), active.sum(1), rng.uniform(0.4, 1.0, nenv))
    anchor = None
    if mode == "goal_distance_ratio":
        anchor, st0 = emulated_place(bbox, active, table, area, "uniform", 5, 0)
    init = np.full((nenv, nobj, 3), 7.0)
    pos, st = emulated_place(bbox, active, table, area, mode, int(rng.randint(1 << 31)), 3, anchor, 0.5, 0.06, pos=init.copy())
    assert (st >= 0).all() and (st > 0).mean() > 0.5
    assert np.array_equal(pos[~active], init[~active])
    for e in np.nonzero(st > 0)[0]:
        idx = np.nonzero(active[e])[0]
        b = bbox[e, idx]
        c = pos[e, idx] + b[:, 0]                                        # box centers in the world
        lo = table[:2] - table[3:5] + area[e, :2]
        assert (c[:, :2] - b[:, 1, :2] >= lo - 1e-12).all() and (c[:, :2] + b[:, 1, :2] <= lo + area[e, 3:5] + 1e-12).all()
        assert np.allclose(c[:, 2] - b[:, 1, 2], top, atol=1e-12, rtol=0)
        for i in range(len(idx)):
            for j in range(i):
                d = np.abs(c[i, :2] - c[j, :2]) * 2.0
                assert not ((d < 2 * (b[i, 1, :2] + b[j, 1, :2])).all()), (e, i, j)
    bad = np.nonzero(st == 0)[0]
    assert not pos[bad][active[bad]].any()


def test_emulated_masked_call_changes_only_the_masked_environments():
    rng = np.random.RandomState(8)
    nenv, nobj = 64, 5
    table = np.array([1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2])
    bbox = _random_boxes(rng, nenv, nobj, 0.02, 0.05)
    area = rp.placement_area((table[:3], table[3:], 0.4), nobj, 1.0)
    full, st = emulated_place(bbox, 1, table, area, "grid_then_uniform", 11, 4)
    mask = rng.rand(nenv) < 0.3
    before = rng.uniform(size=(nenv, nobj, 3))
    part, st2 = emulated_place(bbox, 1, table, area, "grid_then_uniform", 11, 4, mask=mask, pos=before.copy())
    assert np.array_equal(part[mask], full[mask]) and np.array_equal(part[~mask], before[~mask])
    assert np.array_equal(st2[mask], st[mask]) and (st2[~mask] == -1).all()


def test_inputs_are_validated():
    with pytest.raises(ValueError):
        rp.object_placements(np.zeros((2, 3, 2, 3)), 1, ((0, 0, 0), (1, 1, 1), 1), np.zeros(6), 0, 0)   # not on the device
    with pytest.raises(ValueError):
        rp.object_placements(np.zeros((2, 3, 2, 3)), 1, ((0, 0, 0), (1, 1, 1), 1), np.zeros(6), 0, 0, mode="spiral")
    with pytest.raises(ValueError):
        rp.goal_placements(np.zeros((2, 3, 2, 3)), 1, ((0, 0, 0), (1, 1, 1), 1), np.zeros(6), 0, 0, mode="uniform")
    s = rp.PlacementSeed(5)
    assert s.next() == (5, 0) and s.next() == (5, 1)


# ---------------------------------------------------------------------------------------------- GPU
def _gpu_place(bbox, active, table, area, mode, seed, epoch, anchor=None, ratio=1.0, mask=None, out=None):
    import torch

    f = lambda x: None if x is None else torch.as_tensor(np.asarray(x), device="cuda:0")
    fn = rp.goal_placements if mode == "goal_distance_ratio" else rp.object_placements
    kw = dict(anchor=f(anchor), goal_distance_ratio=ratio) if mode == "goal_distance_ratio" else {}
    pos, st = fn(f(np.asarray(bbox, dtype=np.float64)), f(active), (table[:3], table[3:], 0.0), f(area), seed, epoch, mode=mode,
                 mask=f(mask), out=None if out is None else f(out).clone(), **kw)
    torch.cuda.synchronize()
    return pos.cpu().numpy(), st.cpu().numpy()


@pytest.mark.gpu
def test_cuda_philox_equals_curand_on_a_million_counters():
    L = pyemu.philox_check()
    for k0, k1 in ((0, 0), (20261016, 1023), (0xFFFFFFFF, 0xDEADBEEF)):
        assert L.rg_philox_mismatches(1 << 20, k0, k1) == 0


@pytest.mark.gpu
def test_cuda_kernel_reproduces_every_reference_case(golden):
    table = np.array(golden["table"])
    for i, c in enumerate(golden["cases"]):
        bbox, active, area, anchor, mask = _case_inputs(c)
        pos, st = _gpu_place(bbox, active, table, area, c["mode"], c["seed"], c["epoch"], anchor, c["ratio"], mask)
        assert st[-1] == c["status"] and np.array_equal(pos[-1], np.array(c["pos"])), (i, c["mode"])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["grid_then_uniform", "grid", "uniform", "goal_distance_ratio"])
def test_cuda_kernel_equals_emulation_and_masked_calls_touch_only_the_masked(mode):
    rng = np.random.RandomState(21)
    nenv, nobj = 1024, 8
    table = np.array([1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2])
    bbox = _random_boxes(rng, nenv, nobj, 0.01, 0.08)
    active = rng.rand(nenv, nobj) < 0.8
    area = rp.placement_area((table[:3], table[3:], 0.4), active.sum(1), rng.uniform(0.4, 1.0, nenv))
    anchor = emulated_place(bbox, active, table, area, "uniform", 2, 0)[0] if mode == "goal_distance_ratio" else None
    want, wst = emulated_place(bbox, active, table, area, mode, 99, 7, anchor, 0.5)
    got, gst = _gpu_place(bbox, active, table, area, mode, 99, 7, anchor, 0.5)
    assert np.array_equal(gst, wst) and np.array_equal(got, want)
    assert len(set(wst.tolist())) >= 1 and (wst > 0).mean() > 0.3
    mask = rng.rand(nenv) < 0.05
    before = rng.uniform(size=(nenv, nobj, 3))
    part, pst = _gpu_place(bbox, active, table, area, mode, 99, 7, anchor, 0.5, mask=mask, out=before)
    keep = np.where(active[..., None], got, before)                    # inactive slots are not written
    assert np.array_equal(part[mask], keep[mask]) and np.array_equal(part[~mask], before[~mask])
    assert np.array_equal(pst[mask], gst[mask]) and (pst[~mask] == -1).all()


def _quat2mat(q):
    w, x, y, z = q
    s = 2.0 / (q @ q)
    return np.array([[1 - s * (y * y + z * z), s * (x * y - w * z), s * (x * z + w * y)],
                     [s * (x * y + w * z), 1 - s * (x * x + z * z), s * (y * z - w * x)],
                     [s * (x * z - w * y), s * (y * z + w * x), 1 - s * (x * x + y * y)]])


@pytest.mark.gpu
def test_cuda_boxes_of_random_scaled_draws_match_numpy_boxes(ycb):
    import torch

    b8, lib, sb = ycb
    rng = np.random.RandomState(5)
    nenv = 1024
    draws = rng.randint(0, len(lib.entries), (nenv, 8))
    draws[rng.rand(nenv, 8) < 0.05] = -1
    scales = rng.uniform(0.6, 1.6, (nenv, 8))
    yaw = rng.uniform(-np.pi, np.pi, (nenv, 8))
    quat = np.stack([np.cos(0.5 * yaw), 0 * yaw, 0 * yaw, np.sin(0.5 * yaw)], -1)
    quat[:, :4] = rng.normal(size=(nenv, 4, 4))                        # some full rotations too
    _, model, sim = tms._gpu_batch(sb, nenv, outputs=("ncon", "warn"), **tms.CAPS)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draws, scales)
    got = sc.bounding_boxes(torch.as_tensor(quat)).cpu().numpy()
    worst = 0.0
    for e in range(nenv):
        for k in range(8):
            d = draws[e, k]
            if d < 0:
                assert not got[e, k].any()
                continue
            ent = lib.entries[d]
            R = _quat2mat(quat[e, k])
            pts = []
            for j, h in enumerate(ent.hulls):
                Rg = _quat2mat(np.asarray(ent.parts["geom_quat"][j], dtype=np.float64))
                pts.append((np.asarray(ent.parts["geom_pos"][j]) * scales[e, k] + (h.vert * scales[e, k]) @ Rg.T) @ R.T)
            p = np.concatenate(pts)
            lo, hi = p.min(0), p.max(0)
            want = np.stack([lo + (hi - lo) / 2, (hi - lo) / 2])
            worst = max(worst, np.abs(got[e, k] - want).max())
    assert worst < 1e-5, worst


@pytest.mark.gpu
def test_cuda_lowest_hull_point_is_the_reference_resting_height(ycb):
    """place() rests an object by its scaled lowest hull point; for yaw-only rotations that is the reference's z,
    size_z - center_z + table top"""
    import torch

    b8, lib, sb = ycb
    rng = np.random.RandomState(6)
    nenv = 64
    draws = rng.randint(0, len(lib.entries), (nenv, 8))
    scales = rng.uniform(0.6, 1.6, (nenv, 8))
    yaw = rng.uniform(-np.pi, np.pi, (nenv, 8))
    _, model, sim = tms._gpu_batch(sb, nenv, outputs=("ncon", "warn"), **tms.CAPS)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draws, scales)
    q = torch.as_tensor(np.stack([np.cos(0.5 * yaw), 0 * yaw, 0 * yaw, np.sin(0.5 * yaw)], -1))
    bb = sc.bounding_boxes(q).cpu().numpy()
    sc.place(torch.zeros(nenv, 8, 2), torch.as_tensor(yaw), tms.TABLE_TOP, clearance=0.0)
    z = torch.stack([sim.qpos[:, a + 2] for a in sc.qadr], 1).double().cpu().numpy()
    ref = bb[:, :, 1, 2] - bb[:, :, 0, 2] + tms.TABLE_TOP
    assert np.abs(z - ref).max() < 2e-6, np.abs(z - ref).max()                # fp32 qpos


def _cross_object_penetrations(sim, geom_obj):
    c = sim.contact.cpu().numpy()
    n = sim.ncon.cpu().numpy()
    bad = np.zeros(sim.nenv, bool)
    for e in range(sim.nenv):
        cc = c[e, :n[e]]
        g1, g2 = cc[:, 0].astype(int), cc[:, 1].astype(int)
        o1, o2 = geom_obj[g1], geom_obj[g2]
        bad[e] = ((o1 >= 0) & (o2 >= 0) & (o1 != o2) & (cc[:, 2] < 0)).any()
    return bad


@pytest.mark.gpu
def test_cuda_end_to_end_placed_objects_do_not_touch(ycb):
    """1024 ycb environments (random draws, scales, yaws) and 2048 block environments: boxes, grid_then_uniform, forward();
    in every valid environment no contact with negative distance between parts of two different objects"""
    import torch
    from robogym_b200 import engine
    from robogym_b200.rearrange_scene import BatchedBlockScene

    b8, lib, sb = ycb
    rng = np.random.RandomState(12)
    nenv = 1024
    draws = rng.randint(0, len(lib.entries), (nenv, 8))
    draws[rng.rand(nenv, 8) < 0.1] = -1
    scales = rng.uniform(0.7, 1.3, (nenv, 8))
    yaw = rng.uniform(-np.pi, np.pi, (nenv, 8))
    _, model, sim = tms._gpu_batch(sb, nenv, outputs=("ncon", "warn", "contact"), **tms.CAPS)
    sc = rms.BatchedMeshScene(sim, lib)
    sc.set_objects(draws, scales)
    q = torch.as_tensor(np.stack([np.cos(0.5 * yaw), 0 * yaw, 0 * yaw, np.sin(0.5 * yaw)], -1))
    bbox = sc.bounding_boxes(q)
    table = rp.table_dimensions(model)
    active = torch.as_tensor(draws >= 0)
    area = rp.placement_area(table, active.sum(1), 1.0)
    pos, st = rp.object_placements(bbox, active, table, area, *rp.PlacementSeed(1).next())
    sc.place(pos[..., :2], torch.as_tensor(yaw), table[2])
    sim.forward()
    torch.cuda.synchronize()
    st = st.cpu().numpy()
    m = model.host
    geom_obj = np.full(m["ngeom"], -1)
    for k, g in enumerate(sc.geoms):
        geom_obj[g] = k
    bad = _cross_object_penetrations(sim, geom_obj)
    assert (st > 0).mean() > 0.5 and not bad[st > 0].any(), (np.bincount(st, minlength=3), np.nonzero(bad & (st > 0))[0][:10])

    blob = open(os.path.join(ASSETS, "rearrange_blocks5.rgm"), "rb").read()
    bmodel = engine.DeviceModel(blob, 0)
    bsim = engine.BatchedSim(bmodel, 2048, 10, outputs=("ncon", "warn", "contact"))
    bs = BatchedBlockScene(bsim)
    bs.set_blocks(rng.uniform(0.02, 0.05, (2048, bs.nobj)))
    yaw = rng.uniform(-np.pi, np.pi, (2048, bs.nobj))
    q = torch.as_tensor(np.stack([np.cos(0.5 * yaw), 0 * yaw, 0 * yaw, np.sin(0.5 * yaw)], -1))
    active = torch.as_tensor(rng.rand(2048, bs.nobj) < 0.8)
    table = rp.table_dimensions(bmodel)
    area = rp.placement_area(table, active.sum(1), rng.uniform(0.4, 1.0, 2048))
    pos, st = rp.object_placements(bs.bounding_boxes(q), active, table, area, *rp.PlacementSeed(2).next())
    bs.place(pos[..., :2], torch.as_tensor(yaw), pos[..., 2], active=active)
    bsim.forward()
    torch.cuda.synchronize()
    st = st.cpu().numpy()
    geom_obj = np.full(bmodel.host["ngeom"], -1)
    for k, g in enumerate(bs.geoms):
        geom_obj[g] = k
    bad = _cross_object_penetrations(bsim, geom_obj)
    assert (st > 0).mean() > 0.5 and not bad[st > 0].any(), (np.bincount(st, minlength=3), np.nonzero(bad & (st > 0))[0][:10])
