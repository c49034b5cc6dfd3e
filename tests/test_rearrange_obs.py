"""Rearrange observations (robogym_b200/rearrange_obs.py, csrc/rg_obs.inl): the reference's `_observe_simple` dict, the
placement-area masks, the contact flags and the simulation penalties of one env-step (rg_rearrange_obs).

The fixture tests/golden/reference_rearrange_obs.json.gz (tools/make_rearrange_obs_golden.py) holds the reference's own
results on float32-rounded rows, with those rows, the goal and the index tables the reference's name lookups give.  The CPU tier
runs the kernel's code on the emulation build (tests/emu); the GPU tier runs it on the device.  Positions, velocities,
qpos, forces, contacts, masks, penalties and done must be bit-identical; angles and the qpos_goal quaternions agree within
1e-14 (sin / cos / atan2, and the shim builds body_xmat with its own quat2mat)."""
import ctypes
import gzip
import json
import os

import numpy as np
import pytest

import pyemu
from robogym_b200 import engine
from robogym_b200 import rearrange_goal as rg
from robogym_b200 import rearrange_obs as ro

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_rearrange_obs.json.gz")
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
ANGLE_KEYS = ("obj_rot", "goal_obj_rot", "masked_obj_rot", "masked_goal_obj_rot")


@pytest.fixture(scope="module")
def golden():
    with gzip.open(GOLDEN) as f:
        return json.load(f)


def _p(a):
    return None if a is None else a.ctypes.data


class EmuObs:
    """rg_rearrange_obs on the emulation build over host arrays: `rows` has the sim rows ([nenv, ...] float32), `tables` the
    index tables (the fixture's keys), `goal` the goal inputs, `reset` bbox_size / colors / boundary; outputs persist."""

    def __init__(self, tables, nenv, mask_obs, penalty, margin):
        T = tables
        self.nenv, self.nobj, self.T = nenv, T["nobj"], T
        self.narm, self.ngrip, self.nq = len(T["arm_qpos"]), len(T["grip_qpos"]), T["nq"]
        n, k = nenv, self.nobj
        z = lambda *s, d=np.float64: np.zeros(s, d)
        self.out = dict(obj_pos=z(n, k, 3), obj_rel_pos=z(n, k, 3), obj_vel_pos=z(n, k, 3), obj_rot=z(n, k, 3), obj_vel_rot=z(n, k, 3),
                        robot_joint_pos=z(n, self.narm), gripper_pos=z(n, 3), gripper_velp=z(n, 3), gripper_controls=z(n, 1),
                        gripper_qpos=z(n, self.ngrip), gripper_vel=z(n, self.ngrip), qpos=z(n, self.nq), qpos_goal=z(n, self.nq),
                        goal_obj_pos=z(n, k, 3), goal_obj_rot=z(n, k, 3), rel_goal_obj_pos=z(n, k, 3), rel_goal_obj_rot=z(n, k, 3),
                        is_goal_achieved=z(n, 1, d=np.int32), obj_gripper_contact=z(n, k, 2), obj_bbox_size=z(n, k, 3), obj_colors=z(n, k, 4),
                        safety_stop=z(n, 1, d=np.uint8), tcp_force=z(n, 3), tcp_torque=z(n, 3), gripper_table_contact=z(n, d=np.uint8),
                        wrist_cam_contacts=z(n, 4, d=np.uint8), sim_reward=z(n), sim_done=z(n, d=np.uint8))
        if mask_obs:
            self.out.update(placement_mask=z(n, k, 1), goal_placement_mask=z(n, k, 1))
            for key in ro.OBJECT_KEYS + ro.GOAL_KEYS:
                self.out["masked_" + key] = np.zeros_like(self.out[key])
        self.cout = engine.ObsOut(**{f: _p(self.out.get(f)) for f in ro.OUT_FIELDS})
        self.keep = dict(obj_body=np.asarray(T["obj_body"], np.int32), obj_qpos=np.asarray(T["obj_qpos"], np.int32),
                         geom_object=np.asarray(T["geom_object"], np.int32), geom_flags=np.asarray(T["geom_flags"], np.uint8))
        c = self.cin = engine.ObsIn()
        c.nenv, c.nobj = n, k
        c.nbody, c.nq, c.nv, c.nu, c.nsensordata, c.ngeom = T["nbody"], T["nq"], T["nv"], T["nu"], T["nsensordata"], T["ngeom"]
        c.obj_body, c.obj_qpos = _p(self.keep["obj_body"]), _p(self.keep["obj_qpos"])
        c.tcp_body, c.narm, c.ngrip, c.grip_act = T["tcp_body"], self.narm, self.ngrip, T["grip_act"]
        c.arm_qpos[:self.narm] = T["arm_qpos"]
        c.grip_qpos[:self.ngrip] = T["grip_qpos"]
        c.grip_qvel[:self.ngrip] = T["grip_qvel"]
        c.force_adr, c.torque_adr = T["force_adr"], T["torque_adr"]
        c.geom_object, c.geom_flags = _p(self.keep["geom_object"]), _p(self.keep["geom_flags"])
        c.table_plane, c.wrist_sphere = T["table_plane"], T["wrist_sphere"]
        c.pad[:] = T["pad"]
        c.penalty[:] = ro._penalty(penalty)
        c.mask_obs, c.mask_margin = int(mask_obs), float(margin)

    def __call__(self, rows, goal, reset, mask=None):
        f32 = lambda x: np.ascontiguousarray(x, dtype=np.float32)
        f64 = lambda x: np.ascontiguousarray(x, dtype=np.float64)
        k = dict(body_xpos=f32(rows["body_xpos"]), body_xquat=f32(rows["body_xquat"]), body_xvel=f32(rows["body_xvel"]), qpos=f32(rows["qpos"]),
                 qvel=f32(rows["qvel"]), ctrl=f32(rows["ctrl"]), sensordata=f32(rows["sensordata"]), contact=f32(rows["contact"]),
                 ncon=np.ascontiguousarray(rows["ncon"], dtype=np.int32), goal_pos=f64(goal["goal_pos"]), goal_quat=f64(goal["goal_quat"]),
                 rel_pos=f64(goal["rel_pos"]), rel_rot=f64(goal["rel_rot"]), achieved=np.ascontiguousarray(goal["achieved"], dtype=np.uint8),
                 off_table=np.ascontiguousarray(goal["off_table"], dtype=np.uint8), group=np.ascontiguousarray(goal["group"], dtype=np.int32),
                 qpos_at_goal=f32(goal["qpos_at_goal"]), bbox_size=f64(reset["bbox_size"]), colors=f64(reset["colors"]), boundary=f64(reset["boundary"]),
                 mask=None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8))
        c = self.cin
        c.ncontact = k["contact"].shape[1]
        for name in ("body_xpos", "body_xquat", "body_xvel", "qpos", "qvel", "ctrl", "sensordata", "contact", "ncon", "goal_pos", "goal_quat", "rel_pos",
                     "rel_rot", "achieved", "off_table", "group", "qpos_at_goal", "bbox_size", "colors", "boundary"):
            setattr(c, name, _p(k[name]))
        if pyemu.lib().rge_obs(ctypes.byref(c), _p(k["mask"]), ctypes.byref(self.cout)) != 0:
            raise ValueError(pyemu.lib().rge_obs_error().decode())
        return self.out


def _case_inputs(case):
    """the fixture's steps of one case as a batch: one environment per step"""
    T, st = case["tables"], case["steps"]
    n, k = len(st), T["nobj"]
    cap = max(1, max(len(s["rows"]["contact"]) for s in st))
    con = np.zeros((n, cap, 4), np.float32)
    for e, s in enumerate(st):
        if s["rows"]["contact"]:
            con[e, :len(s["rows"]["contact"])] = np.asarray(s["rows"]["contact"], dtype=np.float64)
    rows = {r: np.stack([np.asarray(s["rows"][r]) for s in st]) for r in ("body_xpos", "body_xquat", "body_xvel", "qpos", "qvel", "ctrl", "sensordata")}
    rows.update(contact=con, ncon=np.array([len(s["rows"]["contact"]) for s in st]))
    goal = dict(goal_pos=np.stack([s["goal_pos"] for s in st]).reshape(n, k, 3), goal_quat=np.stack([s["goal_quat"] for s in st]).reshape(n, k, 4),
                rel_pos=np.stack([s["rel_pos"] for s in st]).reshape(n, k, 3), rel_rot=np.stack([s["rel_rot"] for s in st]).reshape(n, k, 3),
                achieved=np.array([s["achieved"] for s in st]), off_table=np.array([s["off_table"] for s in st]), group=np.array([s["group"] for s in st]),
                qpos_at_goal=np.stack([s["qpos_at_goal"] for s in st]))
    reset = dict(bbox_size=np.stack([s["bbox_size"] for s in st]).reshape(n, k, 3), colors=np.broadcast_to(np.reshape(case["colors"], (k, 4)), (n, k, 4)),
                 boundary=np.broadcast_to(case["boundary"], (n, 6)))
    return rows, goal, reset


def _run_case(case, mask=None):
    rows, goal, reset = _case_inputs(case)
    e = EmuObs(case["tables"], len(case["steps"]), case["mask_obs"], case["penalty"], case["mask_margin"])
    return e, e(rows, goal, reset, mask)


CASES = ("blocks5", "blocks3of5", "ycb")


@pytest.mark.parametrize("name", CASES)
def test_emulated_kernel_reproduces_the_reference_dict(golden, name):
    case = golden[name]
    e, out = _run_case(case)
    T = case["tables"]
    quat_cols = np.zeros(T["nq"], bool)
    for k in range(T["num_objects"]):
        quat_cols[T["obj_qpos"][k] + 3:T["obj_qpos"][k] + 7] = True
    for i, s in enumerate(case["steps"]):
        for key, want in s["obs"].items():
            want = np.asarray(want, dtype=np.float64)
            got = np.asarray(out[key][i], dtype=np.float64).ravel()
            assert got.shape == want.shape, (name, s["note"], key)
            if key in ANGLE_KEYS:
                np.testing.assert_allclose(got, want, rtol=0, atol=1e-14, err_msg=f"{name} {s['note']} {key}")
            elif key == "qpos_goal":
                assert np.array_equal(got[~quat_cols], want[~quat_cols]), (name, s["note"], key)
                np.testing.assert_allclose(got[quat_cols], want[quat_cols], rtol=0, atol=1e-14, err_msg=f"{name} {s['note']} {key}")
            else:
                # bit for bit: the sign of a zero counts (masked_* = obs * mask is -0 for a negative value)
                assert np.array_equal(got.view(np.uint64), want.view(np.uint64)), (name, s["note"], key, got, want)
        assert bool(out["gripper_table_contact"][i]) == s["gripper_table"], (name, s["note"])
        assert [bool(x) for x in out["wrist_cam_contacts"][i]] == [s["wrist_cam"][k] for k in ro.WRIST_KEYS], (name, s["note"])
        assert out["sim_reward"][i] == s["reward"] and bool(out["sim_done"][i]) == s["done"], (name, s["note"], out["sim_reward"][i], s["reward"])


def test_fixture_covers_pad_and_table_contacts_masks_and_the_table_edge(golden):
    steps = [s for n in CASES for s in golden[n]["steps"]]
    assert any(max(s["obs"]["obj_gripper_contact"]) > 0 for s in steps)
    assert any(s["gripper_table"] for s in steps)
    assert any(0.0 in s["obs"].get("placement_mask", []) for s in steps)
    assert any(s["done"] for s in steps)
    assert any(s["reward"] not in (0.0, -golden["blocks5"]["penalty"]["objects_off_table"]) for s in steps)
    assert -1 in golden["blocks3of5"]["steps"][0]["group"] and -1 in golden["ycb"]["steps"][0]["group"]
    # a finger pad on a slot other than 0, a wrist-camera contact in every case (its penalty included), a goal outside the area
    assert any(max(s["obs"]["obj_gripper_contact"][2:]) > 0 for s in steps)
    for n in CASES:
        assert any(s["wrist_cam"]["any"] and s["reward"] <= -golden[n]["penalty"]["wrist_collision"] for s in golden[n]["steps"]), n
    assert any(0.0 in s["obs"]["goal_placement_mask"] for s in golden["ycb"]["steps"])
    negz = [s for s in golden["ycb"]["steps"] for k, v in s["obs"].items() if k.startswith("masked_") and any(np.signbit(x) and x == 0 for x in v)]
    assert negz, "a masked value that is -0 in the reference"


def test_obj_rot_equals_the_goal_kernels_emulation(golden):
    from test_rearrange_goal import EmuGoal

    case = golden["ycb"]
    e, out = _run_case(case)
    rows, goal, _ = _case_inputs(case)
    T = case["tables"]
    n, k = len(case["steps"]), T["nobj"]
    pos = rows["body_xpos"].reshape(n, -1, 3)[:, T["obj_body"]]
    quat = rows["body_xquat"].reshape(n, -1, 4)[:, T["obj_body"]]
    g = EmuGoal(n, k, "full")(pos, quat, goal["goal_pos"], goal["goal_quat"], goal["group"])
    assert np.array_equal(out["obj_rot"], g["obj_rot"])


def test_contact_flags_equal_the_contact_queries(golden):
    """BatchedRearrangeContacts' three queries, restated on the same contact lists"""
    for name in CASES:
        case = golden[name]
        T = case["tables"]
        e, out = _run_case(case)
        flags, gobj = np.asarray(T["geom_flags"]), np.asarray(T["geom_object"])
        for i, s in enumerate(case["steps"]):
            con = s["rows"]["contact"]
            gt = any((flags[g1] & 1 and g2 == T["table_plane"]) or (flags[g2] & 1 and g1 == T["table_plane"]) for g1, g2, _, _ in con)
            wr = dict(table_collision_plane=False, robot=False, object=False)
            for g1, g2, _, _ in con:
                if T["wrist_sphere"] in (g1, g2):
                    other = g2 if g1 == T["wrist_sphere"] else g1
                    wr["table_collision_plane" if other == T["table_plane"] else ("robot" if flags[other] & 2 else "object")] = True
            pads = np.zeros((T["nobj"], 2))
            for g1, g2, dist, _ in con:
                for sd, pad in enumerate(T["pad"]):
                    for a, b in ((g1, g2), (g2, g1)):
                        if dist < 1e-5 and a == pad and gobj[b] >= 0:
                            pads[gobj[b], sd] = 1.0
            assert bool(out["gripper_table_contact"][i]) == gt
            assert [bool(x) for x in out["wrist_cam_contacts"][i][:3]] == [wr[k] for k in ro.WRIST_KEYS[:3]]
            assert np.array_equal(out["obj_gripper_contact"][i], pads)


def test_contact_classes_pad_sides_and_slots_on_chosen_contact_lists(golden):
    """every branch of the scan on hand-made contact lists over the blocks5 model's geoms: the wrist sphere against the table
    plane, a robot geom and an object (each class and its penalty), finger pads on slots 4 and 1 from either side of the pair,
    the 1e-5 distance cut-off, and a gripper geom on the table plane"""
    case = golden["blocks5"]
    T = case["tables"]
    flags, gobj = np.asarray(T["geom_flags"]), np.asarray(T["geom_object"])
    geom_of = lambda k: int(np.flatnonzero(gobj == k)[0])
    robot = int(np.flatnonzero(((flags & 2) > 0) & (np.arange(len(flags)) != T["wrist_sphere"]))[0])
    gripper = int(np.flatnonzero(flags & 1)[0])
    wr, tp, (left, right) = T["wrist_sphere"], T["table_plane"], T["pad"]
    lists = [[(wr, tp, -1e-3)], [(robot, wr, -1e-3)], [(wr, geom_of(2), 0.0)], [(left, geom_of(4), -1e-3), (geom_of(1), right, 0.0)],
             [(left, geom_of(2), 2e-5), (gripper, tp, -1e-3)], [(geom_of(0), tp, -1e-4)]]
    rows, goal, reset = _case_inputs(case)
    n = len(lists)
    one = lambda d: {k: np.repeat(v[:1], n, axis=0) for k, v in d.items()}
    rows, goal, reset = one(rows), one(goal), one(reset)
    con = np.zeros((n, 4, 4), np.float32)
    for e, l in enumerate(lists):
        for i, (g1, g2, d) in enumerate(l):
            con[e, i] = (g1, g2, d, 3)
    rows.update(contact=con, ncon=np.array([len(l) for l in lists]))
    assert case["steps"][0]["reward"] == 0.0        # no other penalty in the row used
    out = EmuObs(T, n, False, case["penalty"], 0.02)(rows, goal, reset)
    wrist = np.array([[1, 0, 0, 1], [0, 1, 0, 1], [0, 0, 1, 1], [0, 0, 0, 0], [0, 0, 0, 0], [0, 0, 0, 0]])
    assert np.array_equal(out["wrist_cam_contacts"], wrist)
    assert np.array_equal(out["gripper_table_contact"], [0, 0, 0, 0, 1, 0])
    pads = np.zeros((n, T["nobj"], 2))
    pads[3, 4, 0] = pads[3, 1, 1] = 1.0
    assert np.array_equal(out["obj_gripper_contact"], pads)
    p = case["penalty"]
    assert np.array_equal(out["sim_reward"], [-p["wrist_collision"]] * 3 + [0.0, -p["table_collision"], 0.0])
    assert not out["sim_done"].any()


def test_emulated_masked_call_writes_only_the_masked_environments(golden):
    case = golden["blocks5"]
    rows, goal, reset = _case_inputs(case)
    n = len(case["steps"])
    full = EmuObs(case["tables"], n, True, case["penalty"], 0.02)
    want = {k: v.copy() for k, v in full(rows, goal, reset).items()}
    part = EmuObs(case["tables"], n, True, case["penalty"], 0.02)
    mask = np.arange(n) % 3 == 1
    got = part(rows, goal, reset, mask)
    for key, v in got.items():
        assert np.array_equal(v[mask], want[key][mask]), key
        assert not v[~mask].any(), key


def test_bad_inputs_are_refused(golden):
    case = golden["blocks5"]
    rows, goal, reset = _case_inputs(case)
    n = len(case["steps"])
    e = EmuObs(case["tables"], n, False, case["penalty"], 0.02)
    e.keep["obj_body"][1] = case["tables"]["nbody"]
    with pytest.raises(ValueError, match="object body"):
        e(rows, goal, reset)
    e = EmuObs(case["tables"], n, False, case["penalty"], 0.02)
    e.keep["obj_qpos"][0] = case["tables"]["nq"] - 3
    with pytest.raises(ValueError, match="qpos address"):
        e(rows, goal, reset)
    e = EmuObs(case["tables"], n, False, case["penalty"], 0.02)
    e.cin.force_adr = case["tables"]["nsensordata"] - 1
    with pytest.raises(ValueError, match="sensor"):
        e(rows, goal, reset)
    e = EmuObs(case["tables"], n, True, case["penalty"], 0.02)
    e.cout.masked_obj_pos = None
    with pytest.raises(ValueError, match="masked"):
        e(rows, goal, reset)
    with pytest.raises(ValueError, match="penalty"):
        ro._penalty({"table": 1.0})

    class Sim:
        torch = None
        body_xpos = body_xquat = body_xvel = contact = ncon = object()
        sensordata = None

    with pytest.raises(ValueError, match="sensordata"):
        ro.BatchedRearrangeObservation(Sim(), None, [1], bbox_size=0, colors=0, placement_area_boundary=0)
    with pytest.raises(ValueError, match="soft_mask"):
        ro.BatchedRearrangeObservation(Sim(), None, [1], bbox_size=0, colors=0, placement_area_boundary=0, soft_mask=True)


def test_placement_area_boundary_is_the_references(golden):
    from robogym_b200 import rearrange_placement as rp

    blob = open(os.path.join(ASSETS, "rearrange_blocks5_tcp.rgm"), "rb").read()
    table = rp.table_dimensions(blob)
    area = rp.placement_area(table, 5)
    assert np.array_equal(ro.placement_area_boundary(table, area)[0], golden["blocks5"]["boundary"])


def test_index_tables_from_the_model_names_are_the_references(golden):
    """the tables BatchedRearrangeObservation builds from the committed model's name tables equal the reference's lookups"""
    from robogym_b200 import modelblob

    blob = open(os.path.join(ASSETS, "rearrange_blocks5_tcp.rgm"), "rb").read()
    T = golden["blocks5"]["tables"]
    got = ro.index_tables(modelblob.unpack(blob), modelblob.unpack_names(blob), T["obj_body"])
    for k in ("obj_qpos", "tcp_body", "arm_qpos", "grip_qpos", "grip_qvel", "grip_act", "force_adr", "torque_adr", "geom_object", "geom_flags",
              "table_plane", "wrist_sphere", "pad"):
        assert np.array_equal(np.asarray(got[k]), np.asarray(T[k])), k


# ---------------------------------------------------------------- GPU
def _np(x):
    return x.detach().cpu().numpy()


def _emulate(obs_fn):
    """the emulation on host copies of everything the device call reads"""
    sim, goal, c = obs_fn.sim, obs_fn.goal, obs_fn.cin
    T = dict(nobj=obs_fn.nobj, nbody=c.nbody, nq=c.nq, nv=c.nv, nu=c.nu, nsensordata=c.nsensordata, ngeom=c.ngeom, obj_body=list(obs_fn.obj_body),
             obj_qpos=list(obs_fn.obj_qpos), tcp_body=c.tcp_body, arm_qpos=list(c.arm_qpos[:c.narm]), grip_qpos=list(c.grip_qpos[:c.ngrip]),
             grip_qvel=list(c.grip_qvel[:c.ngrip]), grip_act=c.grip_act, force_adr=c.force_adr, torque_adr=c.torque_adr,
             geom_object=_np(obs_fn.geom_object), geom_flags=_np(obs_fn.geom_flags), table_plane=c.table_plane, wrist_sphere=c.wrist_sphere, pad=list(c.pad))
    pen = dict(zip(("table_collision", "wrist_collision", "objects_off_table", "safety_stop"), list(c.penalty)))
    e = EmuObs(T, sim.nenv, bool(c.mask_obs), pen, c.mask_margin)
    rows = {k: _np(getattr(sim, k)) for k in ("body_xpos", "body_xquat", "body_xvel", "qpos", "qvel", "ctrl", "sensordata", "contact", "ncon")}
    go = goal._e.out
    g = dict(goal_pos=_np(goal.goal_pos), goal_quat=_np(goal.goal_quat), rel_pos=_np(go["rel_goal_obj_pos"]), rel_rot=_np(go["rel_goal_obj_rot"]),
             achieved=_np(go["goal_achieved"]), off_table=_np(go["objects_off_table"]), group=_np(goal.groups), qpos_at_goal=_np(obs_fn.qpos_at_goal))
    return e(rows, g, dict(bbox_size=_np(obs_fn.bbox_size), colors=_np(obs_fn.colors), boundary=_np(obs_fn.boundary)))


def _batch(asset, nenv, nobj_active, seed, mask_obs):
    """random states of `asset`: objects around the table (some off it, some outside the area), random arm, random goals"""
    import torch

    from robogym_b200 import engine, rearrange_placement as rp

    blob = open(os.path.join(ASSETS, asset + ".rgm"), "rb").read()
    model = engine.DeviceModel(blob, 0)
    sim = engine.BatchedSim(model, nenv, 10, outputs=("ncon", "warn", "body_xpos", "body_xquat", "body_xvel", "contact", "sensordata", "geom_xpos"),
                            contact_capacity=64, row_capacity=160)
    g = torch.Generator().manual_seed(seed)
    names = [model.id2name("body", b) for b in range(model.host["nbody"])]
    bodies = [b for b, n in enumerate(names) if n and n.startswith("object") and ":" not in n]
    nobj = len(bodies)
    table = rp.table_dimensions(blob)
    qadr = [int(model.host["jnt_qposadr"][model.name2id("joint", f"object{k}:joint")]) for k in range(nobj)]
    q = sim.qpos.cpu()
    for k, a in enumerate(qadr):
        q[:, a] = 1.3 + 0.8 * (torch.rand(nenv, generator=g) - 0.5) * 2
        q[:, a + 1] = 0.75 + 1.0 * (torch.rand(nenv, generator=g) - 0.5) * 2
        q[:, a + 2] = 0.45 + 0.1 * torch.rand(nenv, generator=g)
        qq = torch.randn(nenv, 4, generator=g)
        q[:, a + 3:a + 7] = qq / qq.norm(dim=1, keepdim=True)
    # every eighth environment keeps all its objects over the middle of the table, so some environments are not done
    tp, ts = table[0], table[1]
    mid = torch.arange(nenv) % 8 == 7
    for a in qadr:
        for c in range(2):
            q[mid, a + c] = float(tp[c]) + 0.5 * float(ts[c]) * (torch.rand(int(mid.sum()), generator=g) * 2 - 1)
    q[:, :6] += 0.3 * torch.randn(nenv, 6, generator=g)
    sim.qpos.copy_(q)
    sim.qvel.copy_(0.5 * torch.randn(sim.qvel.shape, generator=g))
    sim.step()
    # contacts on purpose: in environment e, active slot e % nobj_active is moved into the left pad (e % 4 == 0), the right pad
    # (1) or the wrist camera's sphere (2)
    from robogym_b200 import modelblob
    T = ro.index_tables(model.host, modelblob.unpack_names(blob), bodies)
    q = sim.qpos.cpu()
    gx = sim.geom_xpos.cpu()
    for e in range(nenv):
        if e % 4 < 3:
            geom = (T["pad"][0], T["pad"][1], T["wrist_sphere"])[e % 4]
            a = qadr[e % nobj_active]
            q[e, a:a + 3] = gx[e, geom]
    sim.qpos.copy_(q)
    sim.forward()
    groups = np.tile(np.arange(nobj), (nenv, 1))
    groups[:, nobj_active:] = -1
    goal = rg.BatchedRearrangeGoal(sim, bodies, groups, table)
    gp = torch.stack([1.3 + 0.7 * (torch.rand(nenv, nobj, generator=g) - 0.5) * 2, 0.75 + 0.9 * (torch.rand(nenv, nobj, generator=g) - 0.5) * 2,
                      torch.full((nenv, nobj), 0.43)], -1)
    gq = torch.randn(nenv, nobj, 4, generator=g, dtype=torch.float64)
    goal.set_goal(gp, gq / gq.norm(dim=-1, keepdim=True))
    goal.evaluate()
    area = rp.placement_area(table, nobj_active)
    colors = torch.rand(nenv, nobj, 4, generator=g, dtype=torch.float64)
    bbox = 0.02 + 0.03 * torch.rand(nenv, nobj, 3, generator=g, dtype=torch.float64)
    obs_fn = ro.BatchedRearrangeObservation(sim, goal, bodies, bbox_size=bbox, colors=colors, placement_area_boundary=ro.placement_area_boundary(table, area),
                                            penalty=dict(table_collision=0.5, wrist_collision=0.25, objects_off_table=2.0, safety_stop=0.125),
                                            mask_obs_outside_placement_area=mask_obs)
    obs_fn.set_goal_qpos()
    return sim, goal, obs_fn


def _check_equal(got_obs, got_info, want, mask=None):
    """bit-identical, except where the device's sin / cos / atan2 enter: angles within 1e-9 rad (modulo 2 pi, as the goal
    kernel's tests compare them) and the qpos_goal quaternions within 1e-12"""
    keys = set(want) - {"gripper_table_contact", "wrist_cam_contacts", "sim_reward", "sim_done"}
    for k in keys:
        g, w = _np(got_obs[k]), want[k]
        g = g.reshape(w.shape).astype(w.dtype)
        if mask is not None:
            g, w = g[mask], w[mask]
        if k in ANGLE_KEYS:
            d = np.abs(g - w)
            assert np.minimum(d, np.abs(2 * np.pi - d)).max() <= 1e-9, k
        elif k == "qpos_goal":
            assert np.abs(g - w).max() <= 1e-12, k
        else:
            assert np.array_equal(g, w), k
    for k in ("gripper_table_contact", "wrist_cam_contacts", "sim_reward", "sim_done"):
        g, w = _np(got_info[k]).astype(want[k].dtype), want[k]
        if mask is not None:
            g, w = g[mask], w[mask]
        assert np.array_equal(g, w), k


@pytest.mark.gpu
@pytest.mark.parametrize("asset,nenv,active,mask_obs", [("rearrange_blocks5_tcp", 2048, 5, False), ("rearrange_blocks5_tcp", 2048, 5, True),
                                                        ("rearrange_ycb8_tcp", 1024, 5, True)])
def test_cuda_kernel_equals_emulation_and_masked_calls_touch_only_the_masked(asset, nenv, active, mask_obs):
    import torch

    sim, goal, obs_fn = _batch(asset, nenv, active, 11, mask_obs)
    obs, info = obs_fn.observe()
    torch.cuda.synchronize()
    want = {k: v.copy() for k, v in _emulate(obs_fn).items()}
    _check_equal(obs, info, want)
    assert int(sim.ncon.max()) > 0
    assert bool(info["sim_done"].any()) and not bool(info["sim_done"].all())
    # the contacts put there are found: both pads, every active slot, and the wrist sphere against an object
    gc = obs["obj_gripper_contact"]
    for side in range(2):
        for k in range(active):
            assert bool((gc[:, k, side] > 0).any()), (side, k)
    assert int(info["wrist_cam_contacts"][:, 2].sum()) > nenv // 8
    if mask_obs:
        pm = obs["placement_mask"][:, :active]
        assert bool((pm == 0).any()) and bool((pm == 1).any())
    # masked: every output of the other environments is left as it was
    before = {k: v.clone() for k, v in list(obs.items()) + [(k, v) for k, v in info.items() if k != "objects_off_table"]}
    sim.qpos[:, :6] += 0.05
    sim.forward()
    goal.evaluate()
    mask = torch.arange(nenv, device=sim.device) % 5 == 2
    obs, info = obs_fn.observe(mask)
    torch.cuda.synchronize()
    m = _np(mask).astype(bool)
    for k, v in list(obs.items()) + [(k, v) for k, v in info.items() if k != "objects_off_table"]:
        assert torch.equal(v[~mask], before[k][~mask]), k
    want = _emulate(obs_fn)
    _check_equal(obs, info, want, m)


def _restate(sim, goal, obs_fn):
    """the observation dict as tensor ops (fp64 on float32 rows), key by key"""
    import torch as t

    c = obs_fn.cin
    b = t.as_tensor(obs_fn.obj_body, device=sim.device).long()
    act = (goal.groups >= 0)
    a3 = act.unsqueeze(-1).double()
    xpos, xvel, xq = sim.body_xpos.double(), sim.body_xvel.double(), sim.body_xquat.double()
    tcp, tcpv = xpos[:, c.tcp_body], xvel[:, c.tcp_body, 3:]
    pos = xpos[:, b]
    o = dict(obj_pos=pos * a3, obj_rel_pos=(pos - tcp[:, None]) * a3, obj_vel_pos=(xvel[:, b, 3:] - tcpv[:, None]) * a3, obj_vel_rot=xvel[:, b, :3] * a3,
             robot_joint_pos=sim.qpos.double()[:, list(c.arm_qpos[:c.narm])], gripper_pos=tcp, gripper_velp=tcpv,
             gripper_controls=sim.ctrl.double()[:, [c.grip_act]], gripper_qpos=sim.qpos.double()[:, list(c.grip_qpos[:c.ngrip])],
             gripper_vel=sim.qvel.double()[:, list(c.grip_qvel[:c.ngrip])], qpos=sim.qpos.double(), goal_obj_pos=goal.goal_pos * a3,
             rel_goal_obj_pos=goal._e.out["rel_goal_obj_pos"], rel_goal_obj_rot=goal._e.out["rel_goal_obj_rot"],
             is_goal_achieved=goal._e.out["goal_achieved"].int()[:, None], obj_bbox_size=obs_fn.bbox_size * a3, obj_colors=obs_fn.colors * act.unsqueeze(-1),
             tcp_force=sim.sensordata.double()[:, c.force_adr:c.force_adr + 3], tcp_torque=sim.sensordata.double()[:, c.torque_adr:c.torque_adr + 3])
    o["safety_stop"] = (o["tcp_force"].norm(dim=1) > 150)[:, None]
    return o


@pytest.mark.gpu
def test_cuda_obs_equal_the_tensor_op_restatement():
    import torch

    sim, goal, obs_fn = _batch("rearrange_blocks5_tcp", 2048, 4, 5, False)
    obs, info = obs_fn.observe()
    want = _restate(sim, goal, obs_fn)
    torch.cuda.synchronize()
    for k, w in want.items():
        if k == "safety_stop":          # torch's norm need not round as numpy's left-to-right sum does: away from the threshold only
            far = ((obs["tcp_force"].norm(dim=1) - 150).abs() > 1e-9)[:, None]
            assert torch.equal(obs[k][far], w[far]), k
            continue
        assert torch.equal(obs[k], w.to(obs[k].dtype)), k
    rot = goal._e.out["obj_rot"]
    assert torch.equal(obs["obj_rot"], rot)


@pytest.mark.gpu
def test_cuda_contact_flags_equal_the_contact_queries():
    import torch

    from robogym_b200.rearrange_contacts import BatchedRearrangeContacts

    sim, goal, obs_fn = _batch("rearrange_blocks5_tcp", 2048, 5, 3, False)
    obs, info = obs_fn.observe()
    q = BatchedRearrangeContacts(sim, 5)
    torch.cuda.synchronize()
    assert torch.equal(info["gripper_table_contact"], q.gripper_table_contact())
    w = q.wrist_cam_collisions()
    for i, k in enumerate(ro.WRIST_KEYS):
        assert torch.equal(info["wrist_cam_contacts"][:, i], w[k]), k
    assert torch.equal(obs["obj_gripper_contact"], q.object_gripper_contact().double())


def _restate_reward(info, done, safety, penalty):
    """_get_simulation_reward_with_done's penalty part from the flags, subtracted in the reference's order"""
    import torch as t

    r = t.zeros(done.shape[0], dtype=t.float64, device=done.device)
    for flag, w in ((info["gripper_table_contact"], penalty["table_collision"]), (info["wrist_cam_contacts"][:, 3], penalty["wrist_collision"]),
                    (done, penalty["objects_off_table"]), (safety, penalty["safety_stop"])):
        r = t.where(flag, r - w, r)
    return r


@pytest.mark.gpu
def test_cuda_gripper_driven_onto_a_block_through_the_controller():
    """64 environments of placed blocks stepped by BatchedTcpArmController (the reference's dual-simulation loop): block
    k = 1 + e % 4 is put under the tool, the gripper goes down onto it open, closes, leaves upward and goes down onto the table.
    Every env-step the observation equals the tensor-op restatement and the emulation, the reward the restated penalties; the
    pads report block k on both sides while it is held, and the fingers reach the table plane."""
    import torch

    from robogym_b200 import engine, rearrange_placement as rp
    from robogym_b200.rearrange_arm import BatchedTcpArmController
    from robogym_b200.rearrange_scene import BatchedBlockScene

    nenv, dev = 64, "cuda:0"
    blob = open(os.path.join(ASSETS, "rearrange_blocks5_tcp.rgm"), "rb").read()
    model = engine.DeviceModel(blob, 0)
    sim = engine.BatchedSim(model, nenv, 40, outputs=("ncon", "warn", "body_xpos", "body_xquat", "body_xvel", "contact", "sensordata"),
                            contact_capacity=64, row_capacity=160, dofs_per_contact=16)
    solver_model = engine.DeviceModel(open(os.path.join(ASSETS, "rearrange_solver_arm.rgm"), "rb").read(), 0)
    solver = engine.BatchedSim(solver_model, nenv, 40, outputs=("body_xpos", "body_xquat", "warn"))
    ctl = BatchedTcpArmController(sim, solver, max_position_change=0.1)
    arm0 = torch.tensor(np.deg2rad([135.0, -90.0, 135.0, -100.0, -240.0, 135.0]), dtype=torch.float32, device=dev)   # TABLETOP_EXPERIMENT_INITIAL_POS
    sim.qpos[:, ctl.arm_qadr_main] = arm0
    sim.ctrl[:, ctl.arm_act_main] = arm0
    bs = BatchedBlockScene(sim)
    bs.set_blocks(np.full((nenv, bs.nobj), 0.025))
    yaw = torch.zeros(nenv, bs.nobj, dtype=torch.float64)
    active = torch.ones(nenv, bs.nobj, dtype=torch.bool)
    table = rp.table_dimensions(model)
    q1 = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64).repeat(nenv, bs.nobj, 1)
    pos, st = rp.object_placements(bs.bounding_boxes(q1), active, table, rp.placement_area(table, active.sum(1), 1.0), *rp.PlacementSeed(9).next())
    assert bool((st > 0).all())
    bs.place(pos[..., :2], yaw, pos[..., 2], active=active)
    sim.forward()
    tcp_body = model.name2id("body", "robot0:gripper_tcp")
    slot = 1 + torch.arange(nenv) % 4
    q = sim.qpos.cpu()
    for e in range(nenv):
        q[e, bs.qadr[int(slot[e])]:bs.qadr[int(slot[e])] + 2] = sim.body_xpos[e, tcp_body, :2].cpu()
    sim.qpos.copy_(q)
    sim.forward()
    ctl.reset()
    goal = rg.BatchedRearrangeGoal(sim, bs.bodies, np.arange(bs.nobj), table)
    b = torch.as_tensor(bs.bodies, device=dev)
    goal.set_goal(sim.body_xpos[:, b].double(), sim.body_xquat[:, b].double())
    penalty = dict(table_collision=0.5, wrist_collision=0.25, objects_off_table=2.0, safety_stop=0.125)
    obs_fn = ro.BatchedRearrangeObservation(sim, goal, bs.bodies, bbox_size=bs.bounding_boxes(q1)[..., 1, :], colors=torch.rand(nenv, bs.nobj, 4, dtype=torch.float64),
                                            placement_area_boundary=ro.placement_area_boundary(table, rp.placement_area(table, 5)), penalty=penalty,
                                            mask_obs_outside_placement_area=True)
    obs_fn.set_goal_qpos()
    actions = [[0, 0, -1, 0, 0, 1]] * 4 + [[0, 0, -1, 0, 0, -1]] * 4 + [[0, 1, 0.6, 0, 0, 1]] * 4 + [[0, 0, -1, 0, 0, 0]] * 14
    held = torch.zeros(nenv, bs.nobj, 2, dtype=torch.bool, device=dev)
    table_hit = torch.zeros(nenv, dtype=torch.bool, device=dev)
    ar = torch.arange(nenv, device=dev)
    for k, a in enumerate(actions):
        ctl.step(torch.tensor([a] * nenv, dtype=torch.float32, device=dev))
        goal.evaluate()
        obs, info = obs_fn.observe()
        for key, w in _restate(sim, goal, obs_fn).items():
            if key != "safety_stop":
                assert torch.equal(obs[key], w.to(obs[key].dtype)), (k, key)
        assert torch.equal(info["sim_reward"], _restate_reward(info, info["sim_done"], obs["safety_stop"][:, 0], penalty)), k
        torch.cuda.synchronize()
        _check_equal(obs, info, {kk: v.copy() for kk, v in _emulate(obs_fn).items()})
        if k < 8:
            held |= obs["obj_gripper_contact"] > 0
        table_hit |= info["gripper_table_contact"]
    # block `slot` is held on both pads, and no other block is touched by a pad while going down onto it
    on_slot = held[ar, slot.to(dev)]
    assert float(on_slot.all(dim=1).float().mean()) >= 0.9, on_slot.float().mean(0)
    others = held.clone()
    others[ar, slot.to(dev)] = False
    assert float(others.any(dim=(1, 2)).float().mean()) <= 0.1
    assert float(table_hit.float().mean()) >= 0.5
    assert int(sim.warn.max()) & 4 == 0
