"""Rearrange goal evaluation and goal orientations (robogym_b200/rearrange_goal.py, csrc/rg_goal.inl): relative goals, symmetric
rotation distances, greedy matching of duplicate objects, successes, off-table flags and the reward (rg_rearrange_goal), and the
goal orientation samplers (rg_goal_orientations).

The fixture tests/golden/reference_rearrange_goal.json.gz holds the reference's own results (tools/make_rearrange_goal_golden.py),
the orientation draws from the same Philox counters as the kernel (tests/goal_rng.py).  The CPU tier runs the kernel's code
on the emulation build (tests/emu); the GPU tier runs it on the device.  Tolerances: positions 1e-12, angles 1e-9 rad,
rotation distances 1e-7 (acos near 1 turns a last-bit difference of w into about 1e-8); decisions (the parallel quaternion,
the greedy assignment, success flags) must agree wherever the reference's margin is wider than last-bit noise."""
import ctypes
import gzip
import json
import os

import numpy as np
import pytest

import pyemu
from goal_rng import GoalRotReplayRandomState
from robogym_b200 import engine
from robogym_b200 import rearrange_goal as rg

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_rearrange_goal.json.gz")
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
TABLE = np.array([1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2])


def _p(a):
    return None if a is None else a.ctypes.data


def _keys(thr):
    return sum(rg.SUCCESS_KEYS[k] for k in thr), float(thr.get("obj_pos", 0.0)), float(thr.get("obj_rot", 0.0))


class EmuGoal:
    """the kernel's code on the emulation build, with [nenv, nobj] pose rows; outputs and the previous-count buffer persist
    across calls, as BatchedRearrangeGoal's do"""

    def __init__(self, nenv, nobj, mode, table=TABLE, threshold=rg.SUCCESS_THRESHOLD, reward_per_object=1.0):
        self.nenv, self.nobj = nenv, nobj
        self.prev = np.full(nenv, np.nan)
        z = lambda *s, d=np.float64: np.zeros(s, d)
        self.out = dict(obj_rot=z(nenv, nobj, 3), rel_pos=z(nenv, nobj, 3), rel_rot=z(nenv, nobj, 3), dist_pos=z(nenv, nobj), dist_rot=z(nenv, nobj),
                        success=z(nenv, nobj, d=np.uint8), off_table=z(nenv, nobj, d=np.uint8), num_success=z(nenv), reward=z(nenv),
                        achieved=z(nenv, d=np.uint8), any_off=z(nenv, d=np.uint8), pick=z(nenv, nobj, d=np.int32))
        o = self.out
        self.cout = engine.GoalOut(*[_p(o[k]) for k in ("obj_rot", "rel_pos", "rel_rot", "dist_pos", "dist_rot", "success", "off_table", "num_success",
                                                    "reward", "achieved", "any_off", "pick")])
        self.mode, self.table, self.threshold, self.reward_per_object = mode, np.asarray(table, dtype=np.float64), threshold, reward_per_object

    def __call__(self, pos, quat, goal_pos, goal_quat, groups, offset=0.0, weight=1.0, mask=None, rows=None, stride=None):
        n, k = self.nenv, self.nobj
        keep = dict(pos=np.ascontiguousarray(pos, dtype=np.float32), quat=np.ascontiguousarray(quat, dtype=np.float32),
                    gp=np.ascontiguousarray(np.broadcast_to(goal_pos, (n, k, 3)), dtype=np.float64),
                    gq=np.ascontiguousarray(np.broadcast_to(goal_quat, (n, k, 4)), dtype=np.float64),
                    g=np.ascontiguousarray(np.broadcast_to(groups, (n, k)), dtype=np.int32),
                    off=np.ascontiguousarray(np.broadcast_to(offset, (n,)), dtype=np.float64),
                    w=np.ascontiguousarray(np.broadcast_to(weight, (n,)), dtype=np.float64),
                    rows=np.ascontiguousarray(np.arange(k) if rows is None else rows, dtype=np.int32),
                    mask=None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8))
        ci = engine.GoalIn()
        ci.nenv, ci.nobj = n, k
        ci.pos, ci.quat = _p(keep["pos"]), _p(keep["quat"])
        ci.pos_stride, ci.quat_stride = (3 * k, 4 * k) if stride is None else stride
        ci.rows, ci.goal_pos, ci.goal_quat, ci.group = _p(keep["rows"]), _p(keep["gp"]), _p(keep["gq"]), _p(keep["g"])
        ci.pos_offset, ci.rot_weight = _p(keep["off"]), _p(keep["w"])
        ci.table[:] = self.table.tolist()
        ci.rot_dist_type = rg.ROT_DIST.get(self.mode, self.mode)
        ci.success_keys, ci.pos_threshold, ci.rot_threshold = _keys(self.threshold)
        ci.reward_per_object = self.reward_per_object
        rc = pyemu.lib().rge_goal(ctypes.byref(ci), _p(keep["mask"]), _p(self.prev), ctypes.byref(self.cout))
        if rc != 0:
            raise ValueError(pyemu.lib().rge_goal_error().decode())
        return {k: v.copy() for k, v in self.out.items()}


def emu_rot(base, active, seed, epoch, mode, mask=None, out=None):
    base = np.ascontiguousarray(base, dtype=np.float64)
    nenv, nobj = base.shape[:2]
    act = np.ascontiguousarray(np.broadcast_to(active, (nenv, nobj)), dtype=np.uint8)
    out = base.copy() if out is None else np.ascontiguousarray(out, dtype=np.float64)
    pyemu.lib().rge_goal_rot(nenv, nobj, _p(base), _p(act), rg.ROT_RANDOMIZE[mode], seed, epoch, _p(None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)), _p(out))
    return out


def _angle_err(a, b):
    """angle differences modulo 2 pi (normalize_angles may land on -pi or pi for a last-bit difference)"""
    d = np.abs(np.asarray(a) - np.asarray(b))
    return np.minimum(d, np.abs(d - 2 * np.pi))


@pytest.fixture(scope="module")
def golden():
    return json.loads(gzip.decompress(open(GOLDEN, "rb").read()))


def _case_groups(c):
    g = np.full(c["nmax"], -1, np.int32)
    for gid, ids in enumerate(c["groups"]):
        g[ids] = gid
    return g


def check_case(c, got, want):
    """one evaluation of a fixture case against the reference's, under the tolerances of the module docstring"""
    nm = c["name"]
    assert np.abs(got["rel_pos"][0] - want["rel_pos"]).max() <= 1e-12, nm
    assert _angle_err(got["obj_rot"][0], want["obj_rot"]).max() <= 1e-9, nm
    assert _angle_err(got["rel_rot"][0], want["rel_rot"]).max() <= 1e-9, (nm, got["rel_rot"][0], want["rel_rot"])
    assert np.abs(got["dist_pos"][0] - want["dist_pos"]).max() <= 1e-12, nm
    assert np.abs(got["dist_rot"][0] - want["dist_rot"]).max() <= 1e-7, (nm, got["dist_rot"][0], want["dist_rot"])
    pick, match = got["pick"][0] % 32, got["pick"][0] // 32
    for k in range(c["nmax"]):
        if want["match_margin"][k] > 1e-9:
            assert match[k] == want["match"][k], (nm, k)
        if want["pick_margin"][k] > 1e-9:
            assert (pick[k] if pick[k] != 31 else -1) == want["pick"][k], (nm, k, pick[k], want["pick"][k])
    assert np.array_equal(got["off_table"][0], want["off_table"]) and bool(got["any_off"][0]) == want["any_off"], nm
    gaps = np.abs(np.nan_to_num(np.array([want["pos_gap"], want["rot_gap"]], dtype=np.float64), nan=np.inf))
    decisive = (gaps > 1e-6).all(axis=0)
    assert np.array_equal(got["success"][0][decisive], np.array(want["success"])[decisive]), nm
    if decisive.all():
        assert got["num_success"][0] == want["num_success"] and bool(got["achieved"][0]) == want["achieved"], nm
    return decisive.all()


# ---------------------------------------------------------------------------------------------- CPU
def test_parallel_quaternion_tables_are_the_reference_tables(golden):
    out = np.zeros(112)
    pyemu.lib().rge_parallel_quats(_p(out))
    want = np.concatenate([np.ravel(golden["parallel_quats"]), np.ravel(golden["parallel_quats_180"])])
    assert np.array_equal(out, want) and np.array_equal(np.signbit(out), np.signbit(want))


def test_emulated_kernel_reproduces_every_reference_case(golden):
    seen, rewarded = set(), 0
    for c in golden["cases"]:
        ev = EmuGoal(1, c["nmax"], c["mode"], c["table"], c["threshold"], c["reward_per_object"])
        groups = _case_groups(c)
        decisive = True
        for st, want in zip(c["states"], c["out"]):
            got = ev(np.array(st["pos"])[None], np.array(st["quat"])[None], np.array(c["goal_pos"])[None], np.array(c["goal_quat"])[None], groups[None],
                     c["offset"], c["weight"])
            decisive = check_case(c, got, want) and decisive
            if decisive:
                assert got["reward"][0] == want["reward"], (c["name"], got["reward"][0], want["reward"])
                rewarded += want["reward"] != 0
        seen.add((c["mode"], len(c["groups"]) < sum(map(len, c["groups"])), c["nmax"] > sum(map(len, c["groups"]))))
    # every mode with and without duplicates and padding; rewards of both signs occur
    assert {(m, d, p) for m in rg.ROT_DIST for d in (False, True) for p in (False, True)} <= seen and rewarded > 10


def test_fixture_covers_ties_thresholds_and_the_table_edges(golden):
    outs = [o for c in golden["cases"] for o in c["out"]]
    assert sum(m <= 1e-9 for o in outs for m, p in zip(o["pick_margin"], o["pick"]) if p >= 0) >= 5        # tied parallel quaternions
    gaps = np.concatenate([np.nan_to_num(np.array(o["pos_gap"] + o["rot_gap"], dtype=np.float64), nan=1.0) for o in outs])
    assert ((gaps < 0) & (gaps > -1e-3)).any() and ((gaps > 0) & (gaps < 1e-3)).any()
    assert sum(o["any_off"] for o in outs) >= 2 and any(0 < sum(o["success"]) < len(o["success"]) for o in outs)


def test_goal_orientations_reproduce_the_reference_draws(golden):
    for r in golden["rotations"]:
        base = np.array(r["base"])[None]
        n = base.shape[1]
        rs = GoalRotReplayRandomState(r["seed"], r["env"], r["epoch"])
        assert np.array_equal(rs.uniform(0.0, 2.0 * np.pi, size=n), r["angle"])
        if r["face"] is not None:
            assert np.array_equal(GoalRotReplayRandomState(r["seed"], r["env"], r["epoch"]).randint(0, 24, size=n), r["face"])
        # environment r["env"] of a batch, the others masked out
        b = np.zeros((r["env"] + 1, n, 4)); b[:, :, 0] = 1.0; b[-1] = base[0]
        mask = np.zeros(r["env"] + 1, np.uint8); mask[-1] = 1
        got = emu_rot(b, 1, r["seed"], r["epoch"], r["mode"], mask)
        assert np.abs(got[-1] - np.array(r["quat"])).max() <= 1e-15, (r["mode"], got[-1] - np.array(r["quat"]))
        assert np.array_equal(got[:-1], b[:-1])


def test_goal_orientations_skip_inactive_slots_and_masked_calls_match_full_ones():
    rng = np.random.RandomState(4)
    nenv, nobj = 64, 6
    base = rng.normal(size=(nenv, nobj, 4))
    active = rng.rand(nenv, nobj) < 0.7
    full = emu_rot(base, active, 7, 3, "block")
    assert np.array_equal(full[~active], base[~active]) and not np.array_equal(full[active], base[active])
    assert np.allclose(np.linalg.norm(full[active], axis=-1), np.linalg.norm(base[active], axis=-1), atol=1e-12)
    mask = rng.rand(nenv) < 0.3
    part = emu_rot(base, active, 7, 3, "block", mask)
    assert np.array_equal(part[mask], full[mask]) and np.array_equal(part[~mask], base[~mask])


def test_duplicates_at_permuted_goals_are_all_achieved():
    """objects of a group sitting exactly on each other's goals: the greedy matching pairs each with the goal it sits on"""
    rng = np.random.RandomState(2)
    nenv, nobj = 32, 8
    groups = np.array([0, 0, 0, 1, 2, 2, -1, -1])
    gp = np.stack([rng.uniform(1.0, 1.6, (nenv, nobj)), rng.uniform(0.3, 1.2, (nenv, nobj)), np.full((nenv, nobj), 0.45)], -1).astype(np.float32)
    yaw = rng.uniform(-np.pi, np.pi, (nenv, nobj))
    gq = np.stack([np.cos(yaw / 2), 0 * yaw, 0 * yaw, np.sin(yaw / 2)], -1).astype(np.float32)
    perm = np.array([2, 0, 1, 3, 5, 4, 6, 7])
    for mode in rg.ROT_DIST:
        got = EmuGoal(nenv, nobj, mode)(gp[:, perm], gq[:, perm], gp, gq, groups)
        assert got["achieved"].all() and (got["num_success"] == nobj).all() and not got["rel_pos"].any()
        assert np.array_equal(got["pick"][0] // 32, perm)
        # distinct groups: the same poses are far from their goals
        far = EmuGoal(nenv, nobj, mode)(gp[:, perm], gq[:, perm], gp, gq, np.arange(nobj))
        assert not far["achieved"].any()


def test_emulated_masked_call_writes_only_the_masked_environments():
    rng = np.random.RandomState(5)
    nenv, nobj = 48, 5
    pos = rng.uniform(0.3, 1.5, (nenv, nobj, 3)); quat = rng.normal(size=(nenv, nobj, 4))
    gp = rng.uniform(0.3, 1.5, (nenv, nobj, 3)); gq = rng.normal(size=(nenv, nobj, 4))
    groups = np.array([0, 0, 1, 1, 1])
    full = EmuGoal(nenv, nobj, "mod90")
    a = full(pos, quat, gp, gq, groups)
    b2 = full(pos + 0.01, quat, gp, gq, groups)
    part = EmuGoal(nenv, nobj, "mod90")
    mask = rng.rand(nenv) < 0.4
    part(pos, quat, gp, gq, groups)
    prev_before = part.prev.copy()
    c = part(pos + 0.01, quat, gp, gq, groups, mask=mask)
    for k in c:
        assert np.array_equal(c[k][mask], b2[k][mask]) and np.array_equal(c[k][~mask], a[k][~mask]), k
    assert np.array_equal(part.prev[~mask], prev_before[~mask]) and np.array_equal(part.prev[mask], full.prev[mask])


def test_rows_read_in_place_from_a_wider_pose_array():
    rng = np.random.RandomState(6)
    nenv, nbody, nobj = 16, 11, 4
    xpos = rng.uniform(0.3, 1.5, (nenv, nbody, 3)); xquat = rng.normal(size=(nenv, nbody, 4))
    bodies = np.array([9, 2, 5, 7])
    gp = rng.uniform(0.3, 1.5, (nenv, nobj, 3)); gq = rng.normal(size=(nenv, nobj, 4))
    a = EmuGoal(nenv, nobj, "mod180")(xpos, xquat, gp, gq, np.array([0, 1, 1, 2]), rows=bodies, stride=(3 * nbody, 4 * nbody))
    b = EmuGoal(nenv, nobj, "mod180")(xpos[:, bodies], xquat[:, bodies], gp, gq, np.array([0, 1, 1, 2]))
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def test_bad_inputs_are_refused():
    import torch

    ev = EmuGoal(2, 3, "full")
    x = lambda *s: np.ones(s)
    with pytest.raises(ValueError, match="row id"):
        ev(x(2, 3, 3), x(2, 3, 4), x(2, 3, 3), x(2, 3, 4), 0, rows=np.array([0, 1, 3]))
    with pytest.raises(ValueError, match="rot_dist_type"):
        EmuGoal(1, 1, 5)(x(1, 1, 3), x(1, 1, 4), x(1, 1, 3), x(1, 1, 4), 0)
    with pytest.raises(ValueError, match="success_keys"):
        EmuGoal(1, 1, "full", threshold={})(x(1, 1, 3), x(1, 1, 4), x(1, 1, 3), x(1, 1, 4), 0)
    with pytest.raises(ValueError):
        EmuGoal(1, 65, "full")(x(1, 65, 3), x(1, 65, 4), x(1, 65, 3), x(1, 65, 4), 0)
    # the Python layer
    with pytest.raises(ValueError, match="rot_dist_type"):
        rg._settings("icp", None)
    with pytest.raises(ValueError, match="success_threshold"):
        rg._settings("full", {})
    with pytest.raises(ValueError, match="success_threshold"):
        rg._settings("full", {"obj_pos": 0.04, "obj_vel": 1.0})
    assert rg._settings("mod90", {"obj_rot": 0.2}) == (1, 2, 0.0, 0.2)
    with pytest.raises(ValueError, match="groups"):
        rg._groups(torch, [[0, 2]], 1, 2, "cpu")
    with pytest.raises(ValueError, match="groups"):
        rg._groups(torch, [[-2, 0]], 1, 2, "cpu")
    with pytest.raises(ValueError, match="finite"):
        rg._per_env(torch, float("nan"), 3, "goal_pos_offset", "cpu")
    with pytest.raises(ValueError, match="non-zero"):
        rg._quat_ok(torch, torch.zeros(1, 2, 4), "quat")
    with pytest.raises(ValueError, match="CUDA"):
        rg.goal_distance(np.zeros((1, 2, 3)), np.ones((1, 2, 4)), np.zeros((1, 2, 3)), np.ones((1, 2, 4)), 0, (TABLE[:3], TABLE[3:], 0.4))
    with pytest.raises(ValueError, match="full"):
        rg.goal_orientations(torch.ones(1, 2, 4), 1, 0, 0, mode="full")
    with pytest.raises(ValueError, match="rot_randomize_type"):
        rg.goal_orientations(torch.ones(1, 2, 4), 1, 0, 0, mode="spin")
    with pytest.raises(ValueError, match="CUDA"):
        rg.goal_orientations(torch.ones(1, 2, 4), 1, 0, 0)


# ---------------------------------------------------------------------------------------------- GPU
def _random_batch(rng, nenv, nobj):
    top = TABLE[2] + TABLE[5]
    gp = np.stack([rng.uniform(0.6, 2.0, (nenv, nobj)), rng.uniform(-0.1, 1.6, (nenv, nobj)), rng.uniform(0.75 * top - 0.05, top + 0.1, (nenv, nobj))], -1)
    gq = rng.normal(size=(nenv, nobj, 4))
    near = rng.rand(nenv, nobj) < 0.5
    pos = np.where(near[..., None], gp + rng.normal(scale=0.02, size=gp.shape), rng.uniform(0.3, 1.5, gp.shape)).astype(np.float32)
    quat = np.where(near[..., None], gq + rng.normal(scale=0.05, size=gq.shape), rng.normal(size=gq.shape)).astype(np.float32)
    groups = np.tile(np.array([0, 0, 1, 2, 2, 2, 3, -1])[:nobj], (nenv, 1))
    groups[rng.rand(nenv) < 0.3] = np.arange(nobj)                       # distinct objects
    groups[rng.rand(nenv, nobj) < 0.1] = -1                              # padded slots
    return pos, quat, gp, gq, groups


def _cuda(x, dtype=None):
    import torch

    t = torch.as_tensor(np.asarray(x), device="cuda:0")
    return t if dtype is None else t.to(dtype)


def _np(o):
    import torch

    return {k: (_np(v) if isinstance(v, dict) else v.cpu().numpy() if torch.is_tensor(v) else v) for k, v in o.items()}


def _check_equal_to_emulation(got, want, mask=None):
    sel = slice(None) if mask is None else mask
    assert np.abs(got["rel_goal_obj_pos"][sel] - want["rel_pos"][sel]).max() <= 1e-12
    assert _angle_err(got["obj_rot"][sel], want["obj_rot"][sel]).max() <= 1e-9
    assert _angle_err(got["rel_goal_obj_rot"][sel], want["rel_rot"][sel]).max() <= 1e-9
    assert np.abs(got["goal_distance"]["obj_pos"][sel] - want["dist_pos"][sel]).max() <= 1e-12
    assert np.abs(got["goal_distance"]["obj_rot"][sel] - want["dist_rot"][sel]).max() <= 1e-7
    assert np.array_equal(got["pick"][sel], want["pick"][sel])
    assert np.array_equal(got["objects_off_table"][sel], want["off_table"][sel].astype(bool))
    assert np.array_equal(got["done"][sel], want["any_off"][sel].astype(bool))
    # success flags away from the thresholds
    far = (np.abs(want["dist_pos"][sel] - 0.04) > 1e-6) & (np.abs(want["dist_rot"][sel] - 0.2) > 1e-6)
    assert np.array_equal(got["success"][sel][far], want["success"][sel][far].astype(bool))
    envs = far.all(axis=1)
    for k, w in (("num_success", "num_success"), ("goal_achieved", "achieved"), ("reward", "reward")):
        assert np.array_equal(got[k][sel][envs], want[w][sel][envs].astype(got[k].dtype)), k


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["full", "mod90", "mod180"])
def test_cuda_kernel_equals_emulation_and_masked_calls_touch_only_the_masked(mode):
    import torch

    rng = np.random.RandomState({"full": 1, "mod90": 2, "mod180": 3}[mode])
    nenv, nobj = 2048, 8
    pos, quat, gp, gq, groups = _random_batch(rng, nenv, nobj)
    off, w = rng.uniform(-0.04, 0.0, nenv), rng.uniform(0.0, 1.0, nenv)
    table = (TABLE[:3], TABLE[3:], TABLE[2] + TABLE[5])
    ev = EmuGoal(nenv, nobj, mode)
    want1 = ev(pos, quat, gp, gq, groups, off, w)
    pos2 = (pos + rng.normal(scale=0.01, size=pos.shape)).astype(np.float32)
    want2 = ev(pos2, quat, gp, gq, groups, off, w)
    prev = torch.full((nenv,), float("nan"), dtype=torch.float64, device="cuda:0")
    kw = dict(rot_dist_type=mode, goal_pos_offset=_cuda(off), goal_rot_weight=_cuda(w), previous=prev)
    got1 = _np(rg.goal_distance(_cuda(pos), _cuda(quat), _cuda(gp), _cuda(gq), _cuda(groups), table, **kw))
    got2 = _np(rg.goal_distance(_cuda(pos2), _cuda(quat), _cuda(gp), _cuda(gq), _cuda(groups), table, **kw))
    torch.cuda.synchronize()
    _check_equal_to_emulation(got1, want1)
    _check_equal_to_emulation(got2, want2)
    assert (want2["reward"] != 0).any() and (want1["pick"] % 32 != 31).any() == (mode != "full")
    # a masked call: only the masked environments and their previous counts change
    mask = rng.rand(nenv) < 0.1
    pos3 = (pos2 + rng.normal(scale=0.01, size=pos.shape)).astype(np.float32)
    want3 = EmuGoal(nenv, nobj, mode)
    want3.prev[:] = ev.prev
    w3 = want3(pos3, quat, gp, gq, groups, off, w)
    before = prev.clone()
    g = rg.goal_distance(_cuda(pos3), _cuda(quat), _cuda(gp), _cuda(gq), _cuda(groups), table, mask=_cuda(mask), **kw)
    got3 = _np(g)
    torch.cuda.synchronize()
    _check_equal_to_emulation(got3, w3, mask)
    assert torch.equal(prev[_cuda(~mask)], before[_cuda(~mask)])
    assert np.array_equal(prev.cpu().numpy()[mask], want3.prev[mask])
    assert not got3["rel_goal_obj_pos"][~mask].any() and not got3["goal_achieved"][~mask].any()   # fresh outputs: untouched zeros


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["z_axis", "block"])
def test_cuda_goal_orientations_equal_emulation(mode):
    rng = np.random.RandomState(9)
    nenv, nobj = 2048, 8
    base = rng.normal(size=(nenv, nobj, 4))
    active = rng.rand(nenv, nobj) < 0.8
    want = emu_rot(base, active, 123, 5, mode)
    got = rg.goal_orientations(_cuda(base), _cuda(active), 123, 5, mode=mode).cpu().numpy()
    assert np.abs(got - want).max() <= 1e-15 * np.abs(base).max() * 4
    mask = rng.rand(nenv) < 0.2
    part = rg.goal_orientations(_cuda(base), _cuda(active), 123, 5, mode=mode, mask=_cuda(mask)).cpu().numpy()
    assert np.array_equal(part[mask], got[mask]) and np.array_equal(part[~mask], base[~mask])


def _blocks_batch(nenv, seed):
    """rearrange_blocks5_tcp: nenv environments with their 5 blocks placed by rg_place_objects and forward()"""
    import torch
    from robogym_b200 import build, engine
    from robogym_b200 import rearrange_placement as rp
    from robogym_b200.rearrange_scene import BatchedBlockScene

    build.build()
    blob = open(os.path.join(ASSETS, "rearrange_blocks5_tcp.rgm"), "rb").read()
    model = engine.DeviceModel(blob, 0)
    sim = engine.BatchedSim(model, nenv, 10, outputs=("ncon", "warn", "body_xpos", "body_xquat"), contact_capacity=64, row_capacity=160)
    rng = np.random.RandomState(seed)
    bs = BatchedBlockScene(sim)
    bs.set_blocks(np.full((nenv, bs.nobj), 0.025))
    yaw = rng.uniform(-np.pi, np.pi, (nenv, bs.nobj))
    q = torch.as_tensor(np.stack([np.cos(0.5 * yaw), 0 * yaw, 0 * yaw, np.sin(0.5 * yaw)], -1))
    active = torch.ones(nenv, bs.nobj, dtype=torch.bool)
    table = rp.table_dimensions(model)
    area = rp.placement_area(table, active.sum(1), 1.0)
    pos, st = rp.object_placements(bs.bounding_boxes(q), active, table, area, *rp.PlacementSeed(seed).next())
    bs.place(pos[..., :2], torch.as_tensor(yaw), pos[..., 2], active=active)
    sim.forward()
    torch.cuda.synchronize()
    return sim, bs, table, st.cpu().numpy()


@pytest.mark.gpu
def test_cuda_batched_goal_reads_the_sim_rows_as_goal_distance_reads_tensors():
    import torch

    sim, bs, table, st = _blocks_batch(256, 3)
    rng = np.random.RandomState(4)
    b = torch.as_tensor(bs.bodies, device="cuda:0")
    groups = np.tile([0, 0, 1, 2, 2], (sim.nenv, 1))
    gp = sim.body_xpos[:, b].double() + _cuda(rng.normal(scale=0.03, size=(sim.nenv, 5, 3)))
    gq = _cuda(rng.normal(size=(sim.nenv, 5, 4)))
    for mode in rg.ROT_DIST:
        goal = rg.BatchedRearrangeGoal(sim, bs.bodies, groups, table, rot_dist_type=mode, goal_pos_offset=-0.01, goal_rot_weight=0.5)
        valid = goal.set_goal(gp, gq)
        a = _np(goal.evaluate())
        t = _np(rg.goal_distance(sim.body_xpos[:, b], sim.body_xquat[:, b], gp, gq, _cuda(groups), table, rot_dist_type=mode, goal_pos_offset=-0.01,
                                 goal_rot_weight=0.5))
        for k in a:
            if k == "goal_distance":
                for kk in a[k]:
                    assert np.array_equal(a[k][kk], t[k][kk]), (mode, kk)
            elif k != "previous":
                assert np.array_equal(a[k], t[k]), (mode, k)
        assert valid.all() and (a["reward"] == 0).all()


@pytest.mark.gpu
def test_cuda_end_to_end_on_placed_blocks():
    """2048 block environments: goals at the placed objects' own poses are all achieved with reward 0; one goal moved 5 cm drops
    num_success by one and the next reward is -1; a goal turned 90 degrees about z is achieved under mod90, not under full"""
    import torch

    sim, bs, table, st = _blocks_batch(2048, 5)
    assert (st > 0).all()
    b = torch.as_tensor(bs.bodies, device="cuda:0")
    nobj = len(bs.bodies)
    own_p, own_q = sim.body_xpos[:, b].double().clone(), sim.body_xquat[:, b].double().clone()
    for mode in ("full", "mod90"):
        goal = rg.BatchedRearrangeGoal(sim, bs.bodies, np.arange(nobj), table, rot_dist_type=mode)
        assert goal.set_goal(own_p, own_q).all()
        info = goal.evaluate()
        assert bool(info["goal_achieved"].all()) and bool((info["reward"] == 0).all()) and bool((info["num_success"] == nobj).all())
        assert not bool(info["done"].any())
        k = torch.arange(sim.nenv, device="cuda:0") % nobj
        goal.goal_pos[torch.arange(sim.nenv), k, 0] += 0.05          # one goal per environment moves 5 cm, the count carries over
        info = goal.evaluate()
        assert bool((info["num_success"] == nobj - 1).all()) and bool((info["reward"] == -1).all()) and not bool(info["goal_achieved"].any())
        # a goal turned 90 degrees about z
        turn = torch.tensor([np.cos(np.pi / 4), 0.0, 0.0, np.sin(np.pi / 4)], dtype=torch.float64, device="cuda:0")
        w0, x0, y0, z0 = turn
        q = own_q
        w1, x1, y1, z1 = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
        tq = torch.stack([w0 * w1 - z0 * z1, w0 * x1 - z0 * y1, w0 * y1 + z0 * x1, w0 * z1 + z0 * w1], -1)
        goal.set_goal(own_p, tq)
        info = goal.evaluate()
        assert bool(info["goal_achieved"].all()) == (mode == "mod90")
        if mode == "full":
            assert bool((info["num_success"] == 0).all()) and bool((info["reward"] == 0).all())
