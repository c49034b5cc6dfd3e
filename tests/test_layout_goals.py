"""The reference's layout goal generators (rg_layout_goals; robogym_b200/rearrange_placement.py domino_goals / attached_goals /
fixed_goals): DominoStateGoal, AttachedBlockStateGoal and ObjectFixedStateGoal.

The fixture tests/golden/reference_layout_goals.json.gz holds the reference's own results (tools/make_layout_goals_golden.py),
drawn from the same Philox counters as the kernel through the replay RandomState of tests/layout_goals_rng.py.  The CPU tier
runs the kernel's code on the emulation build (tests/emu/rg_emu_layout.cpp); the GPU tier runs it on the device and compares
with the emulation.  Domino positions and rotations go through cos / sin, whose last bits differ between libraries, so they
are compared within a tolerance; everything else, the angles and the choice of retry included, is exact."""
import gzip
import json
import os

import numpy as np
import pytest

import pyemu_layout
from layout_goals_rng import LayoutReplayRandomState
from placement_rng import bounded, philox, u53
from robogym_b200 import rearrange_placement as rp

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_layout_goals.json.gz")
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
TABLE = np.array([1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2])


def _p(a):
    return None if a is None else a.ctypes.data


def emulated_layout(kind, bbox, active, area, seed=0, epoch=0, object_size=None, distance_mul=None, rel=None, max_retry=1000, mask=None, out=None,
                    table=TABLE):
    """rg_layout_goals' code on the emulation build: (pos, quat, status, angle, retry); status and retry -1 where mask is 0"""
    bbox = np.ascontiguousarray(bbox, dtype=np.float64)
    nenv, nobj = bbox.shape[:2]
    c = lambda v, shape, dt=np.float64: None if v is None else np.ascontiguousarray(np.broadcast_to(v, shape), dtype=dt)
    act, ar, osz, mul = c(active, (nenv, nobj), np.uint8), c(area, (nenv, 6)), c(object_size, (nenv,)), c(distance_mul, (nenv,))
    rl, mk, tab = c(rel, (nenv, nobj, 2)), c(mask, (nenv,), np.uint8), c(table, (6,))
    if out is None:
        pos, quat = np.zeros((nenv, nobj, 3)), np.zeros((nenv, nobj, 4))
        quat[..., 0] = 1.0
    else:
        pos, quat = out
    status, angle, retry = np.full(nenv, -1, np.int32), np.zeros((nenv, nobj)), np.full(nenv, -1, np.int32)
    rc = pyemu_layout.lib().rge_layout_goals(nenv, nobj, rp.LAYOUT[kind], _p(bbox), _p(act), _p(tab), _p(ar), _p(osz), _p(mul), _p(rl), max_retry, seed, epoch,
                                             _p(mk), _p(pos), _p(quat), _p(status), _p(angle), _p(retry))
    if rc != 0:
        raise ValueError(pyemu_layout.lib().rge_layout_error().decode())
    return pos, quat, status, angle, retry


@pytest.fixture(scope="module")
def golden():
    return json.loads(gzip.decompress(open(GOLDEN, "rb").read()))


def _case(c, max_retry, table):
    """one fixture case as environment c["env"] of a batch holding it alone there"""
    n, nobj = c["env"] + 1, len(c["bbox"])
    bbox = np.zeros((n, nobj, 2, 3)); bbox[-1] = c["bbox"]
    active = np.zeros((n, nobj), np.uint8); active[-1] = c["active"]
    area = np.zeros((n, 6)); area[-1] = c["area"]
    rel = None
    if c["rel"] is not None:
        rel = np.zeros((n, nobj, 2)); rel[-1] = c["rel"]
    mask = np.zeros(n, np.uint8); mask[-1] = 1
    return emulated_layout(c["kind"], bbox, active, area, c["seed"], c["epoch"], c["object_size"], c["distance_mul"], rel, max_retry, mask, table=table)


# ---------------------------------------------------------------------------------------------- CPU
def test_replay_layout_draws_read_their_documented_counters():
    rs = LayoutReplayRandomState(9, 4, 2)
    r = [philox((d, 0, 4, 2), 9, 4) for d in range(10)]
    assert rs.random() == u53(r[0][0], r[0][1])
    lo, hi = np.array([0.1, 0.2]), np.array([0.5, 0.3])
    assert np.array_equal(rs.uniform(lo, hi), lo + (hi - lo) * np.array([u53(r[1][0], r[1][1]), u53(r[2][0], r[2][1])]))
    idx = list(range(8))
    for s in range(7):
        i = 7 - s
        j = bounded(r[3 + s][0], i)
        idx[i], idx[j] = idx[j], idx[i]
    rows = np.arange(16).reshape(8, 2)
    assert np.array_equal(rs.permutation(rows), rows[idx]) and rs.modifier_draws == 10 and rs.proposals == 0


def test_emulated_kernel_reproduces_every_reference_case(golden):
    table, seen = np.array(golden["table"]), set()
    for i, c in enumerate(golden["cases"]):
        pos, quat, st, ang, retry = _case(c, golden["max_retry"], table)
        assert (st[:-1] == -1).all() and not pos[:-1].any() and (retry[:-1] == -1).all()
        assert st[-1] == c["status"], (i, c["kind"], st[-1], c["status"])
        act = np.array(c["active"], bool)
        want_pos, want_quat = np.array(c["pos"]), np.array(c["quat"])
        if c["kind"] == "domino":
            assert retry[-1] == c["retry"], (i, retry[-1], c["retry"])
            assert np.array_equal(ang[-1], np.array(c["angle"])), (i, ang[-1] - np.array(c["angle"]))
            assert np.abs(pos[-1] - want_pos).max() <= 1e-12, (i, np.abs(pos[-1] - want_pos).max())
            assert np.abs(quat[-1] - want_quat).max() <= 1e-12, (i, np.abs(quat[-1] - want_quat).max())
            seen.add(("domino", int(act.sum()), c["retry"] if c["retry"] < 1 else 1 + (c["retry"] >= 20)))
        else:
            assert np.array_equal(pos[-1], want_pos), (i, c["kind"], pos[-1] - want_pos)
            assert np.array_equal(quat[-1][act], np.tile([1.0, 0.0, 0.0, 0.0], (act.sum(), 1))), i
            seen.add((c["kind"], int(act.sum()), len(act) > act.sum()))
        assert np.array_equal(quat[-1][~act], np.tile([1.0, 0.0, 0.0, 0.0], ((~act).sum(), 1))) and not pos[-1][~act].any()
    assert {1, 2, 5, 8} <= {n for k, n, _ in seen if k == "domino"}
    assert {r for k, _, r in seen if k == "domino"} == {-1, 0, 1, 2}            # failed, first try, a few retries, 20 or more
    assert ("attached", 8, True) in seen and ("attached", 8, False) in seen and any(k == "fixed" for k, *_ in seen)


def test_fixture_covers_the_requested_shapes(golden):
    dom = [c for c in golden["cases"] if c["kind"] == "domino"]
    ecc = {round(c["bbox"][0][1][2] / c["bbox"][0][1][1], 6) for c in dom}
    assert {1.0, 1.5, 4.5} <= ecc and {2.0, 5.0} <= {c["distance_mul"] for c in dom}
    att = [c for c in golden["cases"] if c["kind"] == "attached"]
    assert len({c["object_size"] for c in att}) == 2 and len({tuple(c["area"]) for c in att}) == 2
    rel = [np.array(c["rel"]) for c in golden["cases"] if c["kind"] == "fixed"]
    assert any(((r < 0) | (r > 1)).any() for r in rel) and any(r.shape == (5, 2) for r in rel) and any(r.shape == (6, 2) for r in rel)


def test_fixed_goals_keep_the_reference_rotations(golden):
    """table_setting's turned spoon: fixed_goals hands back the init_quat the reference writes with set_target_quat"""
    c = next(c for c in golden["cases"] if c["kind"] == "fixed" and len(c["active"]) == 5)
    assert np.array_equal(np.array(c["quat"]), np.array(c["init_quat"])) and c["quat"][4][3] != 0.0


def _batch(seed, nenv=96, nobj=8):
    rng = np.random.RandomState(seed)
    size = rng.uniform(0.015, 0.035, nenv)
    ecc = rng.uniform(1.0, 4.5, nenv)
    hs = (size[:, None] * np.stack([1.0 / ecc, np.ones(nenv), ecc], 1))[:, None].repeat(nobj, 1)
    bbox = np.stack([rng.uniform(-0.003, 0.003, (nenv, nobj, 3)), hs], 2)
    active = rng.rand(nenv, nobj) < 0.6
    active[np.arange(nenv), rng.randint(nobj, size=nenv)] = True
    eight = np.zeros((nenv, nobj), bool)
    for e in range(nenv):
        eight[e, np.sort(rng.choice(nobj, min(8, nobj), replace=False))] = True
    area = rp.placement_area((TABLE[:3], TABLE[3:], 0.4), active.sum(1), rng.uniform(0.7, 1.0, nenv))
    return rng, bbox, active, eight, area, size, rng.uniform(2.0, 5.0, nenv)


def test_emulated_masked_calls_equal_full_ones():
    rng, bbox, active, eight, area, size, mul = _batch(5, nobj=10)
    nenv, nobj = active.shape
    mask = rng.rand(nenv) < 0.3
    rel = rng.uniform(-0.2, 1.2, (nenv, nobj, 2))
    for kind, act, kw in (("domino", active, dict(object_size=size, distance_mul=mul)), ("attached", eight, dict(object_size=size)),
                          ("fixed", active, dict(rel=rel))):
        full = emulated_layout(kind, bbox, act, area, 17, 5, **kw)
        before = (rng.uniform(size=(nenv, nobj, 3)), rng.uniform(size=(nenv, nobj, 4)))
        part = emulated_layout(kind, bbox, act, area, 17, 5, mask=mask, out=(before[0].copy(), before[1].copy()), **kw)
        for k, w in ((0, 3), (1, 4)):
            keep = np.where(act[..., None], full[k], before[k])
            assert np.array_equal(part[k][mask], keep[mask]) and np.array_equal(part[k][~mask], before[k][~mask]), (kind, k)
        assert np.array_equal(part[2][mask], full[2][mask]) and (part[2][~mask] == -1).all(), kind
        if kind == "domino":
            assert np.array_equal(part[4][mask], full[4][mask]) and np.array_equal(part[3][mask], full[3][mask])
            assert (full[2] == 1).mean() > 0.5 and (full[4] > 0).any(), np.bincount(full[4] + 1)
        else:
            assert (full[2] == 1).all()


def test_bad_inputs_are_refused():
    bb = np.zeros((2, 8, 2, 3))
    for kind, kw, msg in (("domino", dict(object_size=0.02), "distance_mul"), ("domino", dict(distance_mul=2.0), "object_size"),
                          ("domino", dict(object_size=0.02, distance_mul=2.0, max_retry=0), "max_retry"), ("attached", {}, "object_size"),
                          ("fixed", {}, "relative placements")):
        with pytest.raises(ValueError, match=msg):
            emulated_layout(kind, bb, 1, np.zeros(6), **kw)
    keep = [np.zeros(s) for s in ((2, 8, 2, 3), (6,), (2, 6), (2, 8, 3), (2, 8, 4))]
    act, st = np.ones((2, 8), np.uint8), np.zeros(2, np.int32)
    assert pyemu_layout.lib().rge_layout_goals(2, 8, 4, _p(keep[0]), _p(act), _p(keep[1]), _p(keep[2]), None, None, None, 1, 0, 0, None, _p(keep[3]),
                                               _p(keep[4]), _p(st), None, None) == -1
    assert "kind" in pyemu_layout.lib().rge_layout_error().decode()
    # the Python layer refuses host tensors before anything else
    table = (TABLE[:3], TABLE[3:], 0.4)
    for fn, args in ((rp.domino_goals, (0.02, 2.0)), (rp.attached_goals, (0.02,))):
        with pytest.raises(ValueError, match="CUDA"):
            fn(bb, 1, table, np.zeros(6), 0, 0, *args)
    with pytest.raises(ValueError, match="CUDA"):
        rp.fixed_goals(bb, 1, table, np.zeros(6), np.zeros((8, 2)))


# ---------------------------------------------------------------------------------------------- GPU
def _cuda(x):
    import torch

    return None if x is None else torch.as_tensor(np.asarray(x), device="cuda:0")


def _gpu(kind, bbox, active, area, seed=0, epoch=0, object_size=None, distance_mul=None, rel=None, mask=None, out=None, max_retry=1000):
    import torch

    table = (TABLE[:3], TABLE[3:], TABLE[2] + TABLE[5])
    a = (_cuda(np.asarray(bbox, dtype=np.float64)), _cuda(active), table, _cuda(area))
    o = None if out is None else (_cuda(out[0]).clone(), _cuda(out[1]).clone())
    angle = retry = None
    if kind == "domino":
        pos, quat, st, angle, retry = rp.domino_goals(*a, seed, epoch, _cuda(object_size), _cuda(distance_mul), max_retry=max_retry, mask=_cuda(mask), out=o,
                                                      details=True)
        angle, retry = angle.cpu().numpy(), retry.cpu().numpy()
    elif kind == "attached":
        pos, quat, st = rp.attached_goals(*a, seed, epoch, _cuda(object_size), mask=_cuda(mask), out=o)
    else:
        pos, quat, st = rp.fixed_goals(*a, _cuda(rel), mask=_cuda(mask), out=o)
    torch.cuda.synchronize()
    return pos.cpu().numpy(), quat.cpu().numpy(), st.cpu().numpy(), angle, retry


def fit_margins(bbox, active, area, seed, epoch, object_size, distance_mul, last):
    """per environment, the smallest |area side - arc extent| over retries 0..last[e] (numpy's own cos / sin and the boxes'
    plain rotated extents): how close the fit test that decided its retry came to the other outcome"""
    nenv, nobj = active.shape
    R = int(last.max()) + 1
    d = np.arange(2 * R)
    ctr = np.stack([d, 0 * d, 0 * d + 4, 0 * d + epoch], -1)
    words = np.stack([philox(ctr, seed, e) for e in range(nenv)])      # the key's second word is the environment
    u = ((words[..., 0] >> 5).astype(np.float64) * 67108864.0 + (words[..., 1] >> 6)) / 9007199254740992.0
    offset, delta = u[:, 0::2] * np.pi, u[:, 1::2] * (np.pi / 4.0) - np.pi / 8.0          # [nenv, R]
    margin = np.full(nenv, np.inf)
    for e in range(nenv):
        idx = np.nonzero(active[e])[0]
        n = len(idx)
        r = np.arange(last[e] + 1)
        ang = np.arange(n)[None] * delta[e, r, None] + (offset[e, r, None] + delta[e, r, None] / 2)
        between = np.arange(1, n + 1)[None] * delta[e, r, None] + offset[e, r, None]
        dist = object_size[e] * distance_mul[e]
        px = np.concatenate([np.zeros((len(r), 1)), np.cumsum(np.cos(between), 1)[:, :-1] * dist], 1)
        py = np.concatenate([np.zeros((len(r), 1)), np.cumsum(np.sin(between), 1)[:, :-1] * dist], 1)
        hx, hy = bbox[e, idx, 1, 0], bbox[e, idx, 1, 1]
        ex = np.abs(np.cos(ang)) * hx + np.abs(np.sin(ang)) * hy
        ey = np.abs(np.sin(ang)) * hx + np.abs(np.cos(ang)) * hy
        sx = (px + ex).max(1) - (px - ex).min(1)
        sy = (py + ey).max(1) - (py - ey).min(1)
        margin[e] = np.minimum(np.abs(area[e, 3] - sx), np.abs(area[e, 4] - sy)).min()
    return margin


@pytest.mark.gpu
def test_cuda_layout_goals_equal_emulation_and_masked_calls_touch_only_the_masked():
    rng, bbox, active, eight, area, size, mul = _batch(31, nenv=2048, nobj=8)
    nenv, nobj = active.shape
    rel = rng.uniform(-0.2, 1.2, (nenv, nobj, 2))
    # attached and fixed: bit for bit
    for kind, act, kw in (("attached", eight, dict(object_size=size)), ("fixed", active, dict(rel=rel))):
        want = emulated_layout(kind, bbox, act, area, 77, 9, **kw)
        got = _gpu(kind, bbox, act, area, 77, 9, **kw)
        for k in range(3):
            assert np.array_equal(got[k], want[k]), (kind, k)
        mask = rng.rand(nenv) < 0.1
        before = (rng.uniform(size=(nenv, nobj, 3)), rng.uniform(size=(nenv, nobj, 4)))
        part = _gpu(kind, bbox, act, area, 77, 9, mask=mask, out=before, **kw)
        assert np.array_equal(part[0][mask], np.where(act[..., None], got[0], before[0])[mask]) and np.array_equal(part[0][~mask], before[0][~mask])
        assert np.array_equal(part[2][mask], got[2][mask]) and (part[2][~mask] == -1).all()
    # dominoes: the same statuses, retries and angles except where the deciding fit test is within 1e-9 of flipping
    kw = dict(object_size=size, distance_mul=mul)
    want = emulated_layout("domino", bbox, active, area, 77, 9, **kw)
    got = _gpu("domino", bbox, active, area, 77, 9, **kw)
    last = np.where(want[4] >= 0, want[4], 999)
    margin = fit_margins(bbox, active, area, 77, 9, size, mul, np.maximum(last, np.where(got[4] >= 0, got[4], 999)))
    close = margin < 1e-9
    print(f"dominoes: {close.sum()} of {nenv} environments decided within 1e-9 (smallest margin {margin.min():.3g}); "
          f"statuses {np.bincount(want[2])}, retries up to {want[4].max()}")
    ok = ~close
    assert close.mean() < 0.01
    assert np.array_equal(got[2][ok], want[2][ok]) and np.array_equal(got[4][ok], want[4][ok])
    assert np.array_equal(got[3][ok], want[3][ok])
    assert np.abs(got[0][ok] - want[0][ok]).max() <= 1e-9 and np.abs(got[1][ok] - want[1][ok]).max() <= 1e-9
    assert (want[2] == 1).mean() > 0.5 and (want[4] >= 32).any(), "the batch needs environments past the first round of retries"
    mask = rng.rand(nenv) < 0.1
    before = (rng.uniform(size=(nenv, nobj, 3)), rng.uniform(size=(nenv, nobj, 4)))
    part = _gpu("domino", bbox, active, area, 77, 9, mask=mask, out=before, **kw)
    assert np.array_equal(part[0][mask], np.where(active[..., None], got[0], before[0])[mask]) and np.array_equal(part[0][~mask], before[0][~mask])
    assert np.array_equal(part[1][mask], np.where(active[..., None], got[1], before[1])[mask]) and np.array_equal(part[1][~mask], before[1][~mask])
    assert np.array_equal(part[2][mask], got[2][mask]) and (part[2][~mask] == -1).all() and np.array_equal(part[4][mask], got[4][mask])


@pytest.mark.gpu
def test_cuda_wrappers_refuse_what_the_reference_cannot_take():
    import torch

    table = (TABLE[:3], TABLE[3:], TABLE[2] + TABLE[5])
    bb = torch.zeros(3, 8, 2, 3, dtype=torch.float64, device="cuda:0")
    bb[..., 1, :] = 0.02
    area = rp.placement_area(table, 8, 1.0)
    seven = torch.ones(3, 8, dtype=torch.uint8, device="cuda:0")
    seven[1, 3] = 0
    with pytest.raises(ValueError, match="exactly 8"):
        rp.attached_goals(bb, seven, table, area, 0, 0, 0.02)
    rp.attached_goals(bb, seven, table, area, 0, 0, 0.02, mask=_cuda(np.array([1, 0, 1], bool)))     # the masked-out one is not checked
    for size, mul in ((0.0, 2.0), (0.02, -1.0), (float("nan"), 2.0)):
        with pytest.raises(ValueError, match="> 0"):
            rp.domino_goals(bb, seven, table, area, 0, 0, size, mul)
    with pytest.raises(ValueError, match="> 0"):
        rp.attached_goals(bb, 1, table, area, 0, 0, -0.02)
    with pytest.raises(ValueError, match="active object"):
        rp.domino_goals(bb, torch.zeros(3, 8, dtype=torch.uint8, device="cuda:0"), table, area, 0, 0, 0.02, 2.0)
    with pytest.raises(ValueError, match="relative_placements"):
        rp.fixed_goals(bb, 1, table, area, np.zeros((7, 2)))
    with pytest.raises(ValueError, match="init_quat"):
        rp.fixed_goals(bb, 1, table, area, np.zeros((8, 2)), init_quat=np.zeros((8, 3)))
    pos, quat, st = rp.fixed_goals(bb, 1, table, area, np.full((8, 2), 1.5), init_quat=np.tile([-1.0, 0.0, 0.0, 0.0], (8, 1)))
    assert (st == 1).all() and (quat[..., 0] == 1.0).all()                 # outside [0, 1] taken as is; w >= 0


@pytest.mark.gpu
def test_cuda_dominoes_are_achieved_on_a_live_block_scene():
    """rearrange_blocks5_tcp with per-environment domino sizes: boxes from body_aabb, domino_goals, the goals set and the
    blocks written to them, then forward(): the mod180 evaluation reports every placed environment as achieved"""
    import torch
    from robogym_b200 import engine
    from robogym_b200 import rearrange_goal as rg
    from robogym_b200.rearrange_scene import BatchedBlockScene

    blob = open(os.path.join(ASSETS, "rearrange_blocks5_tcp.rgm"), "rb").read()
    model = engine.DeviceModel(blob, 0)
    nenv = 512
    sim = engine.BatchedSim(model, nenv, 10, outputs=("ncon", "warn", "body_xpos", "body_xquat"), contact_capacity=64, row_capacity=160)
    rng = np.random.RandomState(12)
    bs = BatchedBlockScene(sim)
    size, ecc = rng.uniform(0.02, 0.03, nenv), rng.uniform(1.0, 4.5, nenv)
    bs.set_blocks((size[:, None] * np.stack([1.0 / ecc, np.ones(nenv), ecc], 1))[:, None].repeat(bs.nobj, 1))
    active = torch.ones(nenv, bs.nobj, dtype=torch.bool)
    table = rp.table_dimensions(model)
    area = rp.placement_area(table, active.sum(1), 1.0)
    bbox = bs.bounding_boxes()
    pos, quat, st, angle, _ = rp.domino_goals(bbox, active, table, area, *rp.PlacementSeed(4).next(), size, rng.uniform(2.0, 3.5, nenv), details=True)
    placed = (st == 1).cpu()
    assert placed.float().mean() > 0.9, placed.float().mean()
    goal = rg.BatchedRearrangeGoal(sim, bs.bodies, np.arange(bs.nobj), table, rot_dist_type="mod180")
    assert bool(goal.set_goal(pos, quat)[placed.to(pos.device)].all())                  # on the table
    bs.place(pos[..., :2], angle, pos[..., 2], active=active)
    sim.forward()
    info = goal.evaluate()
    assert bool(info["goal_achieved"].cpu()[placed].all())
    assert float(info["goal_distance"]["obj_pos"].cpu()[placed].max()) < 1e-5
