"""The object groups of a rearrange reset on the GPU (rg_object_groups; robogym_b200/rearrange_groups.py): the device equals the
kernel's CPU emulation on large batches in every mode, a masked call touches only its environments, and the drawn groups,
scales, yaws and colours carry through a live block scene and a live YCB mesh scene to the placement, the goal's duplicate
matching and the observation.

The group counts come from choice decisions against a CDF built with exp; the device's exp and the host's libm may differ
in the last bit, which can flip a decision whose uniform lies within rounding of a CDF edge.  Environments with a decision
within 1e-12 of an edge are counted, reported and left out of the exact comparison."""
import ctypes
import os

import numpy as np
import pytest

import pyemu_groups as pg
from placement_rng import philox, u53
from robogym_b200 import rearrange_groups as rgr

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
TABLE_TOP = 0.453 + 0.03324
INTS = ("group", "count", "material", "mesh", "ngroups")
FLOATS_EXACT = ("rgba", "yaw")
FLOATS_CLOSE = ("scale", "quat")


def _batch(seed, nenv, nobj=8):
    rng = np.random.RandomState(seed)
    active = rng.randint(0, nobj + 1, nenv)
    fixed = np.zeros((nenv, nobj), np.int32)
    for e in range(nenv):
        left, k = active[e], 0
        while left:
            fixed[e, k] = rng.randint(1, left + 1); left -= fixed[e, k]; k += 1
    return rng, active, fixed


def choice_margins(active, seed, epoch, lam, mode):
    """per environment, the smallest |cdf value - u| over its group-count decisions, replayed in numpy (inf: no decision)"""
    margin = np.full(len(active), np.inf)
    if mode not in ("random", "single"):
        return margin
    for e, n in enumerate(active):
        d, left = 0, int(n)
        while left > 0:
            w = philox(np.array([(d, 0, 6, epoch), (d + 1, 0, 6, epoch)], dtype=np.uint64), seed, e)
            lm = lam[0] + (lam[1] - lam[0]) * u53(w[0][0], w[0][1])
            u = u53(w[1][0], w[1][1])
            p = np.array([np.exp(-i * lm) for i in range(1, left + 1)])
            p /= sum(p)
            cdf = p.cumsum()
            cdf /= cdf[-1]
            margin[e] = min(margin[e], float(np.abs(cdf - u).min()))
            left -= int(cdf.searchsorted(u, side="right")) + 1
            d += 2
    return margin


def _gpu(active, seed, epoch, nobj=8, mask=None, out=None, **kw):
    import torch

    if "n_candidates" in kw:
        kw["mesh_candidates"] = list(range(kw.pop("n_candidates")))
    m = None if mask is None else torch.as_tensor(mask, device="cuda:0")
    g = rgr.object_groups(active, seed, epoch, mask=m, nobj=nobj, out=out, **kw)
    torch.cuda.synchronize()
    return g, {k: v.cpu().numpy() for k, v in g._asdict().items()}


def _rel_close(a, b, rel=1e-15):
    return bool((np.abs(a - b) <= rel * np.maximum(np.abs(b), 1e-300)).all())


MODES = [("blocks", 2048, dict(group_mode="random", color_mode="palette", palette=np.array(rgr.BLOCK_COLORS, float), n_materials=3, scale_range=(0.2, 0.4))),
         ("blocks", 2048, dict(group_mode="random", color_mode="random", lam=(2.0, 8.0))),
         ("blocks", 2048, dict(group_mode="dedupe", color_mode="grey", n_materials=4, scale_range=(0.3, 0.1))),
         ("blocks", 2048, dict(group_mode="single", color_mode="palette", palette=np.array(rgr.BLOCK_COLORS, float), lam=(0.5, 1.0))),
         ("blocks", 2048, dict(group_mode="fixed", color_mode="random", n_materials=2)),
         ("ycb", 1024, dict(group_mode="random", color_mode="random", scale_range=(0.5, 0.5), n_candidates=79, replace=True)),
         ("ycb", 1024, dict(group_mode="random", color_mode="grey", scale_range=(0.5, 0.5), n_candidates=11, replace=False, n_materials=4)),
         ("ycb", 1024, dict(group_mode="dedupe", color_mode="random", n_candidates=79, replace=False))]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", range(len(MODES)))
def test_cuda_groups_equal_emulation_and_masked_calls_touch_only_the_masked(mode):
    kind, nenv, kw = MODES[mode]
    rng, active, fixed = _batch(100 + mode, nenv)
    if kw["group_mode"] == "fixed":
        kw = dict(kw, fixed_counts=fixed)
    seed, epoch = 12345 + mode, 77
    want = pg.call(nenv, 8, active, seed, epoch, **kw)
    g, got = _gpu(active, seed, epoch, **kw)
    margin = choice_margins(active, seed, epoch, kw.get("lam", rgr.LAM), kw["group_mode"])
    near = margin < 1e-12
    print(f"{kind} {kw['group_mode']}: {near.sum()} of {nenv} environments with a choice within 1e-12 of a CDF edge "
          f"(smallest margin {margin.min():.3g}); groups per environment {np.bincount(want['ngroups'])}")
    ok = ~near
    assert near.mean() < 0.01
    for k in INTS + FLOATS_EXACT:
        assert np.array_equal(got[k][ok], want[k][ok]), k
    for k in FLOATS_CLOSE:
        assert _rel_close(got[k][ok], want[k][ok]), (k, np.abs(got[k][ok] - want[k][ok]).max())
    assert np.array_equal(got["yaw"], want["yaw"])                       # the yaws never depend on the group draws
    if kw["group_mode"] == "random":
        assert (want["ngroups"] < active).any() and (want["ngroups"] > 1).any()
    # masked: the selected environments as the full call, the others as they were
    import torch

    mask = rng.rand(nenv) < 0.1
    noise = pg.empty_outputs(nenv, 8, rng)
    out = rgr.ObjectGroups(**{k: torch.as_tensor(v, device="cuda:0") for k, v in noise.items()})
    _, part = _gpu(active, seed, epoch, mask=mask, out=out, **kw)
    for k in part:
        assert np.array_equal(part[k][mask], got[k][mask]) and np.array_equal(part[k][~mask], noise[k][~mask]), k


@pytest.mark.gpu
def test_cuda_abi_refuses_what_the_emulation_refuses():
    import torch

    from robogym_b200 import engine

    n = np.array([3, 5])
    with pytest.raises(engine.EngineError, match="fewer rows"):
        rgr.object_groups(n, 0, 0, nobj=8, color_mode="palette", palette=np.ones((4, 4)))
    with pytest.raises(engine.EngineError, match="more groups than candidates"):
        rgr.object_groups(n, 0, 0, nobj=8, mesh_candidates=[0, 1, 2, 3], replace=False)
    with pytest.raises(ValueError, match="mask"):                       # the wrapper checks the mask's shape first ...
        rgr.object_groups(n, 0, 0, nobj=8, mask=torch.ones(3, dtype=torch.uint8, device="cuda:0"))
    c, o = engine.GroupsIn(nenv=2, nobj=8, group_mode=1, color_mode=1, n_materials=1), engine.GroupsOut()
    counts = np.ascontiguousarray(n, dtype=np.int32)
    c.active = counts.ctypes.data
    g = rgr.object_groups(n, 0, 0, nobj=8)
    for k, x in g._asdict().items():
        setattr(o, k, engine.ptr(x))
    mask = torch.ones(3, dtype=torch.uint8, device="cuda:0")
    assert engine.lib().rg_object_groups(ctypes.byref(c), engine.ptr(mask), 3, ctypes.byref(o), None) == -1    # ... and the ABI its length
    assert "mask_len == nenv" in engine.lib().rg_last_error().decode()
    with pytest.raises(engine.EngineError, match="n_materials"):
        rgr.object_groups(n, 0, 0, nobj=8, n_materials=0)
    with pytest.raises(engine.EngineError, match="active counts"):
        rgr.object_groups(np.array([3, 9]), 0, 0, nobj=8)


def _swap_checks(goal, pos, quat, g):
    """goals at the objects' own poses (pos / quat [nenv, nobj]): all achieved; the goals of two objects of one group swapped:
    still every object a success; the goals of two objects of different groups swapped: those two are not.  Environments
    without objects (groups all -1) are left out.  Returns how many environments each swap was tried on."""
    import torch

    grp = g.group.cpu().numpy()
    assert bool(goal.set_goal(pos, quat).all())
    live = torch.as_tensor((grp >= 0).any(1), device=pos.device)
    assert bool(goal.evaluate()["goal_achieved"][live].all())
    same, diff = [], []
    for e in range(len(grp)):
        ids = grp[e][grp[e] >= 0]
        dup = [k for k in range(len(ids)) if (ids == ids[k]).sum() > 1]
        if len(dup) >= 2:
            same.append((e, dup[0], next(k for k in dup if k != dup[0] and ids[k] == ids[dup[0]])))
        if len(set(ids)) >= 2:
            diff.append((e, 0, int(np.nonzero(ids != ids[0])[0][0])))
    for pairs, success in ((same, True), (diff, False)):
        p, q = pos.clone(), quat.clone()
        for e, i, j in pairs:
            p[e, [i, j]] = pos[e, [j, i]]
            q[e, [i, j]] = quat[e, [j, i]]
        goal.set_goal(p, q)
        s = goal.evaluate()["success"].cpu().numpy()
        for e, i, j in pairs:
            assert s[e, i] == success and s[e, j] == success, (e, i, j, success, grp[e])
    goal.set_goal(pos, quat)
    return len(same), len(diff)


def _observe_colors(sim, goal, bodies, g, bbox_size, table, area):
    """the drawn colours through the per-reset path: set_reset_rows(colors=g.rgba, mask=...) for half the environments, then
    for the other half; observe()'s obj_colors shows each object its group's colour, and the other half's rows only after
    their own call"""
    import torch

    from robogym_b200 import rearrange_obs as ro

    nenv = g.group.shape[0]
    obs_fn = ro.BatchedRearrangeObservation(sim, goal, bodies, bbox_size=bbox_size, colors=torch.zeros_like(g.rgba),
                                            placement_area_boundary=ro.placement_area_boundary(table, area))
    act, want = (g.group >= 0).cpu().numpy(), g.rgba.cpu().numpy()
    half = np.arange(nenv) % 2 == 0
    goal.evaluate()
    for mask, done in ((half, half), (~half, np.ones(nenv, bool))):
        obs_fn.set_reset_rows(colors=g.rgba, mask=torch.as_tensor(mask, device=g.rgba.device))
        obs, _ = obs_fn.observe()
        got = obs["obj_colors"].cpu().numpy()
        on, off = act & done[:, None], act & ~done[:, None]
        assert np.array_equal(got[on], want[on]) and not got[off].any()
    # within a group every object shows its group's colour
    grp = g.group.cpu().numpy()
    for e in range(0, len(grp), 7):
        for k in range(grp.shape[1]):
            if grp[e, k] >= 0:
                assert np.array_equal(got[e, k], got[e, int(np.argmax(grp[e] == grp[e, k]))])


OBS_OUTPUTS = ("ncon", "warn", "body_xpos", "body_xquat", "body_xvel", "contact", "sensordata")


@pytest.mark.gpu
def test_cuda_groups_drive_a_live_block_scene():
    """rearrange_blocks5_tcp: groups -> rescale -> bounding_boxes(quat) -> object_placements -> place -> BatchedRearrangeGoal
    with the drawn groups, and observe()'s obj_colors"""
    import torch

    from robogym_b200 import engine, rearrange_goal as rg, rearrange_placement as rp
    from robogym_b200.rearrange_scene import BatchedBlockScene

    nenv = 512
    model = engine.DeviceModel(open(os.path.join(ASSETS, "rearrange_blocks5_tcp.rgm"), "rb").read(), 0)
    sim = engine.BatchedSim(model, nenv, 10, outputs=OBS_OUTPUTS, contact_capacity=64, row_capacity=160, dofs_per_contact=16)
    bs = BatchedBlockScene(sim)
    bs.set_blocks(np.full((nenv, bs.nobj), 0.025))
    rng = np.random.RandomState(4)
    n = rng.randint(1, bs.nobj + 1, nenv)
    seed = rp.PlacementSeed(11)
    g = rgr.object_groups(n, *seed.next(), nobj=bs.nobj, color_mode="palette", palette=rgr.BLOCK_COLORS, scale_range=(0.2, 0.2))
    scale = rgr.block_scale(g)
    bs.rescale(scale)
    act = rgr.active(g)
    table = rp.table_dimensions(model)
    area = rp.placement_area(table, act.sum(1), 1.0)
    bbox = bs.bounding_boxes(rgr.initial_quat(g))
    pos, st = rp.object_placements(bbox, act, table, area, *seed.next())
    assert bool((st > 0).all())
    bs.place(pos[..., :2], g.yaw, pos[..., 2], active=act)
    sim.forward()
    torch.cuda.synchronize()
    # the blocks carry the drawn scales and yaws
    half = bs.bounding_boxes()[..., 1, :].cpu()
    assert torch.allclose(half, 0.025 * scale.cpu()[..., None], rtol=1e-6, atol=0)
    q = torch.stack([sim.qpos[:, a + 3:a + 7] for a in bs.qadr], 1).double().cpu()
    w = rgr.initial_quat(g).cpu()
    assert float((q - w).abs()[act.cpu()].max()) < 1e-6
    goal = rg.BatchedRearrangeGoal(sim, bs.bodies, rgr.goal_groups(g), table, rot_dist_type="mod90")
    b = torch.as_tensor(bs.bodies, device=sim.device)
    same, diff = _swap_checks(goal, sim.body_xpos[:, b].double(), sim.body_xquat[:, b].double(), g)
    assert same > 50 and diff > 50, (same, diff)
    _observe_colors(sim, goal, bs.bodies, g, bs.bounding_boxes(rgr.initial_quat(g))[..., 1, :], table, area)


@pytest.mark.gpu
@pytest.mark.parametrize("replace", [True, False])
def test_cuda_groups_drive_a_live_mesh_scene(replace):
    """rearrange_ycb8's slotted model: the groups' mesh draw through object_scales -> set_objects -> bounding_boxes(quat) ->
    object_placements -> place -> BatchedRearrangeGoal with the drawn groups, and observe()'s obj_colors"""
    import torch

    from robogym_b200 import engine, rearrange_goal as rg, rearrange_mesh_scene as rms, rearrange_placement as rp

    b8, bt = (open(os.path.join(ASSETS, f + ".rgm"), "rb").read() for f in ("rearrange_ycb8", "rearrange_ycb8_tcp"))
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    sb = rms.slotted_model(b8, lib)
    nenv = 256
    model = engine.DeviceModel(sb, 0)
    sim = engine.BatchedSim(model, nenv, 20, outputs=OBS_OUTPUTS, contact_capacity=64, row_capacity=128)
    sc = rms.BatchedMeshScene(sim, lib)
    cand = list(range(len(lib.entries)))
    rng = np.random.RandomState(5 + replace)
    n = rng.randint(1, min(sc.nslot, len(cand)) + 1, nenv)
    seed = rp.PlacementSeed(12)
    g = rgr.object_groups(n, *seed.next(), nobj=sc.nslot, mesh_candidates=cand, replace=replace, scale_range=(0.3, 0.3))
    draw = rgr.mesh_draw(g, cand)
    scale = rgr.mesh_scale(g, lib, cand)
    grp, mesh = g.group.cpu().numpy(), draw.cpu().numpy()
    for e in range(nenv):                            # one mesh per group; without replacement, distinct groups' meshes differ
        ids = grp[e][grp[e] >= 0]
        for k in set(ids):
            assert len(set(mesh[e][:len(ids)][ids == k])) == 1
        if not replace:
            assert len(set(mesh[e][:len(ids)])) == len(set(ids))
    sc.set_objects(draw, scale)
    act = rgr.active(g)
    table = rp.table_dimensions(model)
    area = rp.placement_area(table, act.sum(1), 1.0)
    bbox = sc.bounding_boxes(rgr.initial_quat(g))
    pos, st = rp.object_placements(bbox, act, table, area, *seed.next())
    ok = (st > 0).cpu().numpy()
    assert ok.mean() > 0.5, ok.mean()
    sc.place(pos[..., :2], g.yaw, TABLE_TOP)
    sim.forward()
    torch.cuda.synchronize()
    # keep the placed environments: the goal test needs every object on the table
    keep = torch.as_tensor(ok, device=g.group.device)
    g = g._replace(group=torch.where(keep[:, None], g.group, torch.full_like(g.group, -1)))
    goal = rg.BatchedRearrangeGoal(sim, sc.bodies, rgr.goal_groups(g), table, rot_dist_type="full")
    b = torch.as_tensor(sc.bodies, device=sim.device)
    pos0, quat0 = sim.body_xpos[:, b].double(), sim.body_xquat[:, b].double()
    pos0[~keep] = 0.0
    quat0[~keep] = torch.tensor([1.0, 0.0, 0.0, 0.0], dtype=torch.float64, device=sim.device)
    same, diff = _swap_checks(goal, pos0, quat0, g)
    assert diff > 50 and (same > 20 if replace else True), (same, diff)
    _observe_colors(sim, goal, sc.bodies, g, sc.bounding_boxes(rgr.initial_quat(g))[..., 1, :], table, area)
