"""The reference's stacking, pick-and-place, training and reach goals (rg_goal_modify after rg_place_objects;
robogym_b200/rearrange_placement.py stack_goals / pick_and_place_goals / train_goals / reach_goals) and ObjectStackGoal's
gripper_pos / grasped goal-distance keys (rg_rearrange_goal).

The fixture tests/golden/reference_goal_variants.json.gz holds the reference's own results (tools/make_goal_variants_golden.py),
drawn from the same Philox counters as the kernels through the replay RandomState of tests/goal_variants_rng.py.  The CPU tier
runs the kernels' code on the emulation builds (tests/emu: rg_emu.cpp for the evaluation, rg_emu_modify.cpp for the modifier);
the GPU tier runs it on the device and compares with the emulation."""
import ctypes
import gzip
import json
import os

import numpy as np
import pytest

import pyemu
import pyemu_modify
from goal_variants_rng import GoalVariantsReplayRandomState
from placement_rng import bounded, philox, u53
from robogym_b200 import engine
from robogym_b200 import rearrange_goal as rg
from robogym_b200 import rearrange_placement as rp
from test_placement import emulated_place

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_goal_variants.json.gz")
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
TABLE = np.array([1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2])
KINDS = {"stack": "stack", "pick_and_place": "lift", "train": "train", "reach": "reach"}


def _p(a):
    return None if a is None else a.ctypes.data


def emulated_modify(kind, pos, active, seed, epoch, mask=None, object_size=None, ratio=None, target_height=None, height_range=(0.0, 0.0), pickup=0.0,
                    stacking=0.0, fixed_order=True):
    """rg_goal_modify's code on the emulation build, in place on pos [nenv, nobj, 3]"""
    nenv, nobj = pos.shape[:2]
    per = lambda v: None if v is None else np.ascontiguousarray(np.broadcast_to(v, (nenv,)), dtype=np.float64)
    act = np.ascontiguousarray(np.broadcast_to(active, (nenv, nobj)), dtype=np.uint8)
    mk = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
    osz, rat, th = per(object_size), per(ratio), per(target_height)
    rc = pyemu_modify.lib().rge_goal_modify(nenv, nobj, rp.MODIFY[kind], _p(act), _p(osz), _p(rat), _p(th), height_range[0], height_range[1], pickup, stacking,
                                     int(fixed_order), seed, epoch, _p(mk), _p(pos))
    if rc != 0:
        raise ValueError(pyemu_modify.lib().rge_modify_error().decode())
    return pos


def _first_active(active):
    first = np.zeros_like(active)
    idx = active.argmax(1)
    first[np.arange(len(active)), idx] = active[np.arange(len(active)), idx]
    return first


def emulated_goals(kind, bbox, active, area, seed, epoch, mask=None, pos=None, anchor=None, ratio=1.0, pickup=0.0, stacking=0.0,
                   height_range=(0.0, 0.0), object_size=0.0, target_height=0.0, fixed_order=True, table=TABLE):
    """the composition of rearrange_placement's generator functions on the emulation build: (pos, status, object pos or None)"""
    nenv, nobj = np.shape(bbox)[:2]
    active = np.ascontiguousarray(np.broadcast_to(active, (nenv, nobj)), dtype=np.uint8)
    obj = None
    if kind == "stack":
        pos, st = emulated_place(bbox, _first_active(active), table, area, "uniform", seed, epoch, mask=mask, pos=pos)
    elif kind == "pick_and_place":
        pos, st = emulated_place(bbox, active, table, area, "grid_then_uniform", seed, epoch, mask=mask, pos=pos)
    elif kind == "train":
        pos, st = emulated_place(bbox, active, table, area, "goal_distance_ratio", seed, epoch, anchor, ratio, mask=mask, pos=pos)
    else:
        pos, st = emulated_place(bbox, active, table, area, "uniform", seed, epoch, mask=mask, pos=pos)
        obj = pos.copy()
    emulated_modify(KINDS[kind], pos, active, seed, epoch, mask, object_size=object_size, ratio=ratio, target_height=target_height,
                    height_range=height_range, pickup=pickup, stacking=stacking, fixed_order=fixed_order)
    return pos, st, obj


@pytest.fixture(scope="module")
def golden():
    return json.loads(gzip.decompress(open(GOLDEN, "rb").read()))


def _case(c, table):
    """one fixture case as environment c["env"] of a batch holding it alone there"""
    n, nobj = c["env"] + 1, len(c["bbox"])
    bbox = np.zeros((n, nobj, 2, 3)); bbox[-1] = c["bbox"]
    active = np.zeros((n, nobj), np.uint8); active[-1] = c["active"]
    area = np.zeros((n, 6)); area[-1] = c["area"]
    anchor = None
    if c["anchor"] is not None:
        anchor = np.zeros((n, nobj, 3)); anchor[-1] = c["anchor"]
    mask = np.zeros(n, np.uint8); mask[-1] = 1
    return emulated_goals(c["kind"], bbox, active, area, c["seed"], c["epoch"], mask, anchor=anchor, ratio=c["ratio"], pickup=c["pickup"],
                          stacking=c["stacking"], height_range=c["height_range"], object_size=c["object_size"], target_height=c["target_height"],
                          fixed_order=c["fixed_order"], table=table)


# ---------------------------------------------------------------------------------------------- CPU
def test_replay_modifier_draws_read_their_documented_counters():
    rs = GoalVariantsReplayRandomState(9, 4, 2)
    r0, r1, r2 = (philox((d, 0, 3, 2), 9, 4) for d in range(3))
    assert rs.random() == u53(r0[0], r0[1])
    assert rs.uniform(0.05, 0.25) == 0.05 + (0.25 - 0.05) * u53(r1[0], r1[1])
    assert rs.randint(2, 6) == 2 + bounded(r2[0], 3) and rs.modifier_draws == 3 and rs.proposals == 0


def test_emulated_kernels_reproduce_every_reference_case(golden):
    seen = set()
    for i, c in enumerate(golden["cases"]):
        pos, st, obj = _case(c, np.array(golden["table"]))
        assert st[-1] == c["status"], (i, c["kind"], st[-1], c["status"])
        assert np.array_equal(pos[-1], np.array(c["pos"])), (i, c["kind"], pos[-1] - np.array(c["pos"]))
        if c["kind"] == "reach":
            assert np.array_equal(obj[-1], np.array(c["obj_pos"])), i
        assert (st[:-1] == -1).all() and not pos[:-1].any()
        n = sum(c["active"])
        seen.add((c["kind"], n, len(c["active"]) > n, c["pickup"], c["stacking"], c["ratio"] < 1, c["fixed_order"]))
    kinds = {s[0] for s in seen}
    assert kinds == set(KINDS)
    assert {n for k, n, *_ in seen if k == "stack"} == {2, 3, 4, 5} and {s[6] for s in seen if s[0] == "stack"} == {True, False}
    assert {(s[3], s[4]) for s in seen if s[0] == "train"} == {(0.0, 0.0), (1.0, 0.0), (0.0, 1.0), (0.3, 0.4)}
    assert any(s[5] for s in seen if s[0] == "train") and any(s[2] for s in seen if s[0] != "reach")


def test_fixture_draws_every_training_task(golden):
    """the mixed cases land on all three branches: nothing (one draw), a lift (three) and a tower (more)"""
    train = [c for c in golden["cases"] if c["kind"] == "train"]
    moved = lambda c: not np.array_equal(np.array(c["pos"])[np.array(c["active"], bool)][:, 2],
                                         np.full(sum(c["active"]), np.array(c["pos"])[np.array(c["active"], bool)][0, 2]))
    draws = {c["draws"] for c in train if (c["pickup"], c["stacking"]) == (0.3, 0.4)}
    assert 1 in draws and 3 in draws and max(draws) > 3
    assert all(c["draws"] == 0 for c in train if c["pickup"] + c["stacking"] == 0)
    assert any(moved(c) for c in train if c["stacking"] == 1.0 and sum(c["active"]) >= 2)


def test_emulated_masked_calls_equal_full_ones():
    rng = np.random.RandomState(3)
    nenv, nobj = 96, 6
    size = rng.uniform(0.015, 0.04, (nenv, nobj))
    bbox = np.stack([np.zeros((nenv, nobj, 3)), np.repeat(size[..., None], 3, -1)], 2)
    active = rng.rand(nenv, nobj) < 0.7
    active[:, :2] = True
    one = np.zeros((nenv, nobj), bool)
    one[np.arange(nenv), rng.randint(nobj, size=nenv)] = True
    area = rp.placement_area((TABLE[:3], TABLE[3:], 0.4), active.sum(1), 1.0)
    anchor = emulated_place(bbox, active, TABLE, area, "uniform", 1, 0)[0]
    mask = rng.rand(nenv) < 0.3
    for kind, kw in (("stack", dict(object_size=size[:, 0], fixed_order=False)), ("pick_and_place", dict(height_range=(0.05, 0.25))),
                     ("train", dict(anchor=anchor, ratio=0.5, pickup=0.3, stacking=0.4, height_range=(0.05, 0.25), object_size=size[:, 0])),
                     ("reach", dict(target_height=rng.uniform(0, 0.2, nenv)))):
        act = one if kind == "reach" else active
        ar = rp.placement_area((TABLE[:3], TABLE[3:], 0.4), act.sum(1), 1.0)
        full, st, _ = emulated_goals(kind, bbox, act, ar, 17, 5, **kw)
        before = rng.uniform(size=(nenv, nobj, 3))
        part, pst, _ = emulated_goals(kind, bbox, act, ar, 17, 5, mask=mask, pos=before.copy(), **kw)
        keep = np.where(act[..., None], full, before)
        assert np.array_equal(part[mask], keep[mask]) and np.array_equal(part[~mask], before[~mask]), kind
        assert np.array_equal(pst[mask], st[mask]) and (pst[~mask] == -1).all(), kind
        assert not full[~act].any(), kind                                  # inactive slots stay zero


def _eval(e, mode, keys, thr, gripper=None, grasped=None):
    """rg_rearrange_goal on the emulation build for one recorded state (one environment), with or without the new fields"""
    n, nmax = e["n"], e["nmax"]
    pos = np.ascontiguousarray(np.array(e["pos"])[None], dtype=np.float32)
    quat = np.ascontiguousarray(np.array(e["quat"])[None], dtype=np.float32)
    quat[0, n:, 0] = 1.0
    gp, gq = np.array(e["goal_pos"])[None], np.array(e["goal_quat"])[None]
    gq[0, n:, 0] = 1.0
    keep = dict(pos=pos, quat=quat, gp=np.ascontiguousarray(gp), gq=np.ascontiguousarray(gq), rows=np.arange(nmax, dtype=np.int32),
                g=np.where(np.arange(nmax) < n, np.arange(nmax), -1).astype(np.int32)[None], off=np.zeros(1), w=np.ones(1), prev=np.full(1, np.nan),
                grip=None if gripper is None else np.ascontiguousarray(gripper, dtype=np.float32),
                grasped=None if grasped is None else np.ascontiguousarray(grasped, dtype=np.float64)[None])
    z = lambda *s, d=np.float64: np.zeros(s, d)
    out = dict(obj_rot=z(1, nmax, 3), rel_pos=z(1, nmax, 3), rel_rot=z(1, nmax, 3), dist_pos=z(1, nmax), dist_rot=z(1, nmax), success=z(1, nmax, d=np.uint8),
               off_table=z(1, nmax, d=np.uint8), num_success=z(1), reward=z(1), achieved=z(1, d=np.uint8), any_off=z(1, d=np.uint8),
               pick=z(1, nmax, d=np.int32), rel_gripper=z(1, nmax, 3), dist_gripper=z(1, nmax))
    ci = engine.GoalIn()
    ci.nenv, ci.nobj = 1, nmax
    ci.pos, ci.quat, ci.pos_stride, ci.quat_stride = _p(keep["pos"]), _p(keep["quat"]), 3 * nmax, 4 * nmax
    ci.rows, ci.goal_pos, ci.goal_quat, ci.group = _p(keep["rows"]), _p(keep["gp"]), _p(keep["gq"]), _p(keep["g"])
    ci.pos_offset, ci.rot_weight = _p(keep["off"]), _p(keep["w"])
    ci.table[:] = TABLE.tolist()
    ci.rot_dist_type, ci.success_keys = rg.ROT_DIST[mode], keys
    ci.pos_threshold, ci.rot_threshold = float(thr.get("obj_pos", 0.0)), float(thr.get("obj_rot", 0.0))
    ci.gripper_threshold, ci.grasped_threshold = float(thr.get("gripper_pos", 0.0)), float(thr.get("grasped", 0.0))
    ci.reward_per_object = 1.0
    ci.gripper_pos, ci.gripper_stride, ci.grasped = _p(keep["grip"]), 3, _p(keep["grasped"])
    names = ("obj_rot", "rel_pos", "rel_rot", "dist_pos", "dist_rot", "success", "off_table", "num_success", "reward", "achieved", "any_off", "pick")
    co = engine.GoalOut(*[_p(out[k]) for k in names])
    if gripper is not None:
        co.rel_gripper, co.dist_gripper = _p(out["rel_gripper"]), _p(out["dist_gripper"])
    if pyemu.lib().rge_goal(ctypes.byref(ci), None, _p(keep["prev"]), ctypes.byref(co)) != 0:
        raise ValueError(pyemu.lib().rge_goal_error().decode())
    return out


def test_stack_goal_distance_keys_match_the_reference(golden):
    for i, e in enumerate(golden["evals"]):
        grasped = np.array(e["contacts"]).sum(1).astype(np.float64)
        assert np.array_equal(grasped, e["grasped"]), i
        for thr, want in zip(golden["thresholds"], e["num_success"]):
            keys = sum(rg.SUCCESS_KEYS[k] for k in thr)
            out = _eval(e, e["mode"], keys, thr, np.array(e["gripper"])[None], grasped)
            assert np.array_equal(out["rel_gripper"][0], e["rel_gripper"]), i
            assert np.array_equal(out["dist_gripper"][0], e["dist_gripper"]), i
            assert np.array_equal(out["rel_pos"][0], e["rel_pos"]) and np.array_equal(out["dist_pos"][0], e["dist_pos"]), i
            assert np.abs(out["dist_rot"][0] - e["dist_rot"]).max() <= 1e-7, i
            d = dict(obj_pos=out["dist_pos"][0], obj_rot=out["dist_rot"][0], gripper_pos=out["dist_gripper"][0], grasped=grasped)
            if all(np.abs(d[k] - v).min() > 1e-6 for k, v in thr.items()):    # no distance at its threshold
                assert out["num_success"][0] == want, (i, thr, out["num_success"][0], want)


def test_new_fields_unset_or_unused_leave_every_output_unchanged(golden):
    thr = dict(rg.SUCCESS_THRESHOLD)
    for e in golden["evals"]:
        base = _eval(e, e["mode"], 3, thr)
        with_grip = _eval(e, e["mode"], 3, thr, np.array(e["gripper"])[None], np.array(e["grasped"]))
        assert not base["rel_gripper"].any() and not base["dist_gripper"].any()
        for k in base:
            if k not in ("rel_gripper", "dist_gripper"):
                assert np.array_equal(base[k], with_grip[k], equal_nan=True), k


def test_bad_inputs_are_refused():
    pos = np.zeros((2, 3, 3))
    with pytest.raises(ValueError, match="height_range"):
        emulated_modify("lift", pos, 1, 0, 0, height_range=(0.3, 0.1))
    with pytest.raises(ValueError, match="pickup_proba"):
        emulated_modify("train", pos, 1, 0, 0, object_size=0.02, ratio=1.0, pickup=0.7, stacking=0.4)
    with pytest.raises(ValueError, match="object_size"):
        emulated_modify("stack", pos, 1, 0, 0)
    with pytest.raises(ValueError, match="target_height"):
        emulated_modify("reach", pos, 1, 0, 0)
    e = dict(n=1, nmax=1, pos=[[0, 0, 0]], quat=[[1, 0, 0, 0]], goal_pos=[[0, 0, 0]], goal_quat=[[1, 0, 0, 0]])
    with pytest.raises(ValueError, match="gripper_pos"):
        _eval(e, "full", 5, {"obj_pos": 0.04, "gripper_pos": 0.1})
    with pytest.raises(ValueError, match="grasped"):
        _eval(e, "full", 9, {"obj_pos": 0.04, "grasped": 1.0})
    with pytest.raises(ValueError, match="success_keys"):
        _eval(e, "full", 16, {})
    # the Python layer refuses these before touching the device
    table = (TABLE[:3], TABLE[3:], 0.4)
    bb = np.zeros((2, 3, 2, 3))
    with pytest.raises(ValueError, match="pickup_proba"):
        rp.train_goals(bb, 1, table, np.zeros(6), 0, 0, np.zeros((2, 3, 3)), pickup_proba=0.6, stacking_proba=0.6)
    with pytest.raises(ValueError, match="pickup_proba"):
        rp.train_goals(bb, 1, table, np.zeros(6), 0, 0, np.zeros((2, 3, 3)), pickup_proba=-0.1)
    with pytest.raises(ValueError, match="height_range"):
        rp.train_goals(bb, 1, table, np.zeros(6), 0, 0, np.zeros((2, 3, 3)), pickup_proba=0.5, height_range=(0.2, 0.1))
    with pytest.raises(ValueError, match="height_range"):
        rp.pick_and_place_goals(bb, 1, table, np.zeros(6), 0, 0, height_range=(0.25, 0.05))
    for fn, args in ((rp.stack_goals, (0.02,)), (rp.reach_goals, (0.1,))):
        with pytest.raises(ValueError, match="CUDA"):
            fn(bb, 1, table, np.zeros(6), 0, 0, *args)
    assert rg._settings("full", {"obj_pos": 0.04, "gripper_pos": 0.1, "grasped": 1.0})[1] == 13


# ---------------------------------------------------------------------------------------------- GPU
def _cuda(x):
    import torch

    return None if x is None else torch.as_tensor(np.asarray(x), device="cuda:0")


def _gpu_goals(kind, bbox, active, area, seed, epoch, mask=None, out=None, anchor=None, ratio=1.0, pickup=0.0, stacking=0.0, height_range=(0.0, 0.0),
               object_size=0.0, target_height=0.0, fixed_order=True):
    import torch

    table = (TABLE[:3], TABLE[3:], TABLE[2] + TABLE[5])
    a = (_cuda(np.asarray(bbox, dtype=np.float64)), _cuda(active), table, _cuda(area), seed, epoch)
    kw = dict(mask=_cuda(mask), out=None if out is None else _cuda(out).clone())
    obj = None
    if kind == "stack":
        pos, st = rp.stack_goals(*a, _cuda(object_size), fixed_order=fixed_order, **kw)
    elif kind == "pick_and_place":
        pos, st = rp.pick_and_place_goals(*a, height_range=height_range, **kw)
    elif kind == "train":
        pos, st = rp.train_goals(*a, _cuda(anchor), goal_distance_ratio=ratio, pickup_proba=pickup, stacking_proba=stacking, height_range=height_range,
                                 object_size=_cuda(object_size), **kw)
    else:
        pos, obj, st = rp.reach_goals(*a, _cuda(target_height), **kw)
        obj = obj.cpu().numpy()
    torch.cuda.synchronize()
    return pos.cpu().numpy(), st.cpu().numpy(), obj


def _batches():
    """2048 block environments x 5 (2 to 5 active) and 1024 ycb-like environments x 8 with padded slots"""
    rng = np.random.RandomState(31)
    out = []
    for nenv, nobj, lo, hi in ((2048, 5, 0.02, 0.03), (1024, 8, 0.01, 0.06)):
        size = rng.uniform(lo, hi, (nenv, nobj, 3))
        if nobj == 5:
            size[:] = size[..., :1]                                        # cubes
        bbox = np.stack([rng.uniform(-0.01, 0.01, (nenv, nobj, 3)) * (nobj == 8), size], 2)
        active = rng.rand(nenv, nobj) < 0.7
        active[np.arange(nenv), rng.randint(nobj, size=nenv)] = True
        active[np.arange(nenv), (rng.randint(1, nobj, size=nenv) + active.argmax(1)) % nobj] = True
        one = np.zeros((nenv, nobj), bool)
        one[np.arange(nenv), rng.randint(nobj, size=nenv)] = True
        out.append((rng, bbox, active, one, rng.uniform(0.02, 0.05, nenv)))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind", sorted(KINDS))
def test_cuda_generators_equal_emulation_and_masked_calls_touch_only_the_masked(kind):
    for rng, bbox, active, one, osz in _batches():
        nenv, nobj = active.shape
        act = one if kind == "reach" else active
        area = rp.placement_area((TABLE[:3], TABLE[3:], 0.4), act.sum(1), rng.uniform(0.6, 1.0, nenv))
        kw = dict(stack=dict(object_size=osz, fixed_order=False), pick_and_place=dict(height_range=(0.05, 0.25)),
                  train=dict(ratio=0.5, pickup=0.3, stacking=0.4, height_range=(0.05, 0.25), object_size=osz),
                  reach=dict(target_height=rng.uniform(0.0, 0.2, nenv)))[kind]
        if kind == "train":
            kw["anchor"] = emulated_place(bbox, act, TABLE, area, "grid_then_uniform", 4, 0)[0]
        want, wst, wobj = emulated_goals(kind, bbox, act, area, 77, 9, **kw)
        got, gst, gobj = _gpu_goals(kind, bbox, act, area, 77, 9, **kw)
        assert np.array_equal(gst, wst) and np.array_equal(got, want), (kind, nobj)
        assert (wst > 0).mean() > 0.5, (kind, np.bincount(wst + 1))
        if kind == "reach":
            assert np.array_equal(gobj, wobj)
        mask = rng.rand(nenv) < 0.1
        before = rng.uniform(size=(nenv, nobj, 3))
        part, pst, _ = _gpu_goals(kind, bbox, act, area, 77, 9, mask=mask, out=before, **kw)
        keep = np.where(act[..., None], got, before)
        assert np.array_equal(part[mask], keep[mask]) and np.array_equal(part[~mask], before[~mask]), kind
        assert np.array_equal(pst[mask], gst[mask]) and (pst[~mask] == -1).all(), kind


@pytest.mark.gpu
def test_cuda_generators_refuse_active_counts_the_reference_cannot_take():
    import torch

    table = (TABLE[:3], TABLE[3:], TABLE[2] + TABLE[5])
    bb = torch.zeros(3, 4, 2, 3, dtype=torch.float64, device="cuda:0")
    bb[..., 1, :] = 0.02
    area = rp.placement_area(table, 2, 1.0)
    act = _cuda(np.array([[1, 1, 0, 0], [1, 0, 0, 0], [1, 1, 1, 0]], np.uint8))
    with pytest.raises(ValueError, match="two or more"):
        rp.stack_goals(bb, act, table, area, 0, 0, 0.02)
    rp.stack_goals(bb, act, table, area, 0, 0, 0.02, mask=_cuda(np.array([1, 0, 1], bool)))      # the masked-out environment is not checked
    with pytest.raises(ValueError, match="exactly one"):
        rp.reach_goals(bb, act, table, area, 0, 0, 0.1)
    with pytest.raises(ValueError, match="active object"):
        rp.pick_and_place_goals(bb, torch.zeros(3, 4, dtype=torch.uint8, device="cuda:0"), table, area, 0, 0)
    rp.train_goals(bb, act, table, area, 0, 0, torch.zeros(3, 4, 3, dtype=torch.float64, device="cuda:0"), stacking_proba=1.0)   # n < 2: left as placed


@pytest.mark.gpu
def test_cuda_reach_and_gripper_keys_read_a_live_sims_site():
    """rearrange_blocks5_tcp after forward(): ObjectReachGoal evaluated from site_xpos of robot0:grip (rotation zero), and
    ObjectStackGoal's gripper keys from the same row next to the blocks' body_xpos"""
    import torch
    from robogym_b200.rearrange_scene import BatchedBlockScene

    blob = open(os.path.join(ASSETS, "rearrange_blocks5_tcp.rgm"), "rb").read()
    model = engine.DeviceModel(blob, 0)
    nenv = 512
    sim = engine.BatchedSim(model, nenv, 10, outputs=("ncon", "warn", "body_xpos", "body_xquat", "site_xpos"), contact_capacity=64, row_capacity=160)
    rng = np.random.RandomState(8)
    bs = BatchedBlockScene(sim)
    bs.set_blocks(np.full((nenv, bs.nobj), 0.025))
    active = torch.ones(nenv, bs.nobj, dtype=torch.bool)
    table = rp.table_dimensions(model)
    area = rp.placement_area(table, active.sum(1), 1.0)
    q = torch.zeros(nenv, bs.nobj, 4, dtype=torch.float64)
    q[..., 0] = 1.0
    pos, st = rp.object_placements(bs.bounding_boxes(q), active, table, area, *rp.PlacementSeed(3).next())
    bs.place(pos[..., :2], torch.zeros(nenv, bs.nobj), pos[..., 2], active=active)
    sim.forward()
    sid = model.name2id("site", "robot0:grip")
    # reach: goals target_height above a placed block
    one = torch.zeros(nenv, bs.nobj, dtype=torch.bool)
    one[:, 0] = True
    gpos, opos, gst = rp.reach_goals(bs.bounding_boxes(q), one, table, rp.placement_area(table, 1, 1.0), 5, 0, 0.1)
    assert (gst == 2).all() and torch.equal(gpos[:, 0, :2], opos[:, 0, :2]) and torch.equal(gpos[:, 0, 2], opos[:, 0, 2] + 0.1)
    goal = rg.BatchedRearrangeGoal(sim, None, [0], table, achieved_site="robot0:grip", success_threshold={"obj_pos": 0.04})
    quat = torch.zeros(nenv, 1, 4, dtype=torch.float64)
    quat[..., 0] = 1.0
    goal.set_goal(gpos[:, :1], quat)
    host = lambda o: {k: host(v) if isinstance(v, dict) else v.cpu().numpy() for k, v in o.items()}
    info = host(goal.evaluate())
    grip = sim.site_xpos[:, sid].double().cpu().numpy()
    rel = gpos[:, 0].cpu().numpy() - grip
    assert np.array_equal(info["rel_goal_obj_pos"][:, 0], rel) and not info["obj_rot"].any()
    # distances within 1e-12 of numpy's, as the rest of the suite compares the device's (its build relaxes division and roots)
    assert np.abs(info["goal_distance"]["obj_pos"][:, 0] - np.sqrt((rel[:, 0] * rel[:, 0] + rel[:, 1] * rel[:, 1]) + rel[:, 2] * rel[:, 2])).max() <= 1e-12
    assert np.array_equal(info["success"][:, 0], info["goal_distance"]["obj_pos"][:, 0] < 0.04)
    # stacking keys: the blocks against the gripper, pad contacts as given
    grasped = rng.randint(0, 3, (nenv, bs.nobj)).astype(np.float64)
    thr = {"obj_pos": 0.04, "obj_rot": 0.2, "gripper_pos": 0.5, "grasped": 1.0}
    sg = rg.BatchedRearrangeGoal(sim, bs.bodies, np.arange(bs.nobj), table, success_threshold=thr, gripper_site="robot0:grip")
    b = torch.as_tensor(bs.bodies, device="cuda:0")
    sg.set_goal(sim.body_xpos[:, b].double(), sim.body_xquat[:, b].double())
    out = sg.evaluate(grasped=_cuda(grasped))
    opos = sim.body_xpos[:, b].double().cpu().numpy()
    rg_ = opos - grip[:, None]
    dg = np.sqrt((rg_[..., 0] * rg_[..., 0] + rg_[..., 1] * rg_[..., 1]) + rg_[..., 2] * rg_[..., 2])
    got_dg = out["goal_distance"]["gripper_pos"].cpu().numpy()
    assert np.array_equal(out["rel_gripper_pos"].cpu().numpy(), rg_) and np.abs(got_dg - dg).max() <= 1e-12
    assert np.array_equal(out["goal_distance"]["grasped"].cpu().numpy(), grasped)
    assert np.array_equal(out["success"].cpu().numpy(), (out["goal_distance"]["obj_pos"].cpu().numpy() < 0.04) &
                          (out["goal_distance"]["obj_rot"].cpu().numpy() < 0.2) & (got_dg < 0.5) & (grasped < 1.0))
    # the same evaluation from tensors
    t = rg.goal_distance(sim.body_xpos[:, b], sim.body_xquat[:, b], sim.body_xpos[:, b].double(), sim.body_xquat[:, b].double(), np.arange(bs.nobj), table,
                         success_threshold=thr, gripper_pos=sim.site_xpos[:, sid], grasped=_cuda(grasped))
    for k in ("rel_gripper_pos", "success", "num_success"):
        assert torch.equal(t[k], out[k]), k
