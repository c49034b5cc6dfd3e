"""The first stage of a rearrange reset, for a whole batch on the device: which of an environment's objects are duplicates of
each other, each group's material, colour, size scale and mesh, and every object's initial yaw.

The reference draws these on the host at every reset (`RearrangeEnv._randomize_object_groups` and
`_randomize_object_initial_rotations`, robogym/envs/rearrange/common/base.py:498-630): `sample_group_counts`
(common/utils.py:47-73) splits the objects into groups, `_sample_group_attributes` draws a material, colour and size scale per
group (and a mesh in the mesh environments), and `_sample_default_quaternions` turns every object by a uniform yaw.  Here
`object_groups` is one launch (`rg_object_groups`, one thread per environment, robogym_b200/csrc/rg_groups.inl) with the
reference's arithmetic and draw order.  Random numbers are the placement's Philox4x32-10 keyed by (seed, environment) under
their own purpose, addressed by an `epoch` per call, so a masked redraw gives an environment what a full call gives it.

The environments' variants are arguments: `group_mode` "random" (sample_group_counts), "dedupe" (wordblocks, chessboard,
table_setting: every object its own group), "single" (blocks_duplicate: one group) or "fixed" (holdout's task_object_configs,
`fixed_counts`); `color_mode` "random", "palette" (blocks: a permutation of a palette, e.g. BLOCK_COLORS) or "grey"
(use_grey_colors); `mesh_candidates` (ycb: the sorted candidate list, drawn with or without replacement).  Material values
stay a caller table: `material` indexes it, and BatchedBlockScene / BatchedMeshScene.set_material take the rows.

The outputs feed the later reset stages as they are, or through the small helpers below:

    seed = rp.PlacementSeed(0)
    g = object_groups(n_active, *seed.next(), nobj=scene.nobj, color_mode="palette", palette=BLOCK_COLORS, scale_range=(0.1, 0.1))
    scene.rescale(block_scale(g))                                   # BatchedBlockScene; mesh scenes: mesh_draw / mesh_scale
    bbox = scene.bounding_boxes(initial_quat(g))
    pos, status = rp.object_placements(bbox, active(g), table, area, *seed.next())
    scene.place(pos[..., :2], g.yaw, pos[..., 2], active=active(g))
    goal.set_groups(goal_groups(g))                                 # BatchedRearrangeGoal
    obs.set_reset_rows(colors=g.rgba)                               # BatchedRearrangeObservation
"""
import ctypes
from collections import namedtuple

import numpy as np

from . import engine
from .engine import current_stream, device_mask, ptr

GROUP_MODES = {"random": 1, "dedupe": 2, "single": 3, "fixed": 4}
COLOR_MODES = {"random": 1, "palette": 2, "grey": 3}
MAX_OBJECTS = 64
# envs/rearrange/common/base.py RearrangeEnvConstants.sample_lam_low / sample_lam_high
LAM = (0.1, 5.0)
# envs/rearrange/blocks.py BlockRearrangeEnv.OBJECT_COLORS
BLOCK_COLORS = ((1, 0, 0, 1), (0, 1, 0, 1), (0, 0, 1, 1), (1, 1, 0, 1), (0, 1, 1, 1), (1, 0, 1, 1), (0, 0, 0, 1), (1, 1, 1, 1))

ObjectGroups = namedtuple("ObjectGroups", "group count material rgba scale mesh yaw quat ngroups")
ObjectGroups.__doc__ = """Device tensors of object_groups: group, count, material, mesh (int32 [nenv, nobj]; -1, or count 0, past an
environment's objects), rgba (float64 [nenv, nobj, 4]), scale, yaw (float64 [nenv, nobj]; 0 past the objects), quat (float64
[nenv, nobj, 4], w x y z; 0 past the objects), ngroups (int32 [nenv])."""


def _counts(active, nobj):
    """[nenv] int32 host counts and nobj from counts ([nenv]) or a [nenv, nobj] mask of leading slots"""
    a = np.asarray(active.cpu() if hasattr(active, "cpu") else active)
    if a.ndim == 2:
        if nobj is not None and int(nobj) != a.shape[1]:
            raise ValueError("nobj: the active mask's width")
        n = a.astype(bool).sum(1)
        if not (a.astype(bool) == (np.arange(a.shape[1])[None] < n[:, None])).all():
            raise ValueError("active: the environment's objects are its leading slots")
        return np.ascontiguousarray(n, dtype=np.int32), a.shape[1]
    if a.ndim != 1 or nobj is None:
        raise ValueError("active: [nenv] object counts with nobj, or a [nenv, nobj] mask of leading slots")
    if not np.array_equal(a, np.round(a)):
        raise ValueError("active: integer counts")
    return np.ascontiguousarray(a, dtype=np.int32), int(nobj)


def object_groups(active, seed, epoch, mask=None, group_mode="random", lam=LAM, n_materials=1, color_mode="random", palette=None,
                  scale_range=(0.0, 0.0), mesh_candidates=None, replace=True, fixed_counts=None, nobj=None, device="cuda:0", out=None):
    """The reference's `_randomize_object_groups` and initial yaws for every environment, or those of `mask` [nenv] (the
    others keep what `out` holds).

    active: each environment's object count ([nenv], with `nobj` slots) or a [nenv, nobj] mask of its leading slots;
    seed, epoch: the random stream (e.g. rearrange_placement.PlacementSeed().next());
    group_mode: "random", "dedupe", "single" or "fixed" (fixed_counts [nenv, nobj] or [nobj]: positive counts summing to the
    active count, then zeros); lam: (sample_lam_low, sample_lam_high); n_materials: the length of the material table
    (`material_names`); color_mode: "random", "palette" (palette [rows, 4]: at least the largest count of rows) or "grey";
    scale_range: (object_scale_low, object_scale_high), the scale exp(uniform(-low, high)); mesh_candidates: the candidate
    list (e.g. library indices, sorted as the reference sorts its candidates) or None for no mesh draw, drawn with or without
    `replace`.  The candidates' values do not enter the draw: `mesh` indexes them (see mesh_draw).
    out: an ObjectGroups to write into (a masked call leaves its other environments as they are).  Returns an ObjectGroups."""
    import torch as t

    n, nobj = _counts(active, nobj)
    nenv = len(n)
    if nobj > MAX_OBJECTS:
        raise ValueError(f"at most {MAX_OBJECTS} objects per environment")
    if group_mode not in GROUP_MODES or color_mode not in COLOR_MODES:
        raise ValueError(f"group_mode: one of {sorted(GROUP_MODES)}; color_mode: one of {sorted(COLOR_MODES)}")
    if not (0 <= int(seed) < 1 << 32 and 0 <= int(epoch) < 1 << 32):
        raise ValueError("seed and epoch: 32-bit unsigned integers")
    c = engine.GroupsIn()
    keep = [n]
    c.nenv, c.nobj, c.active = nenv, nobj, n.ctypes.data
    c.group_mode, c.lam_low, c.lam_high = GROUP_MODES[group_mode], float(lam[0]), float(lam[1])
    if group_mode == "fixed":
        if fixed_counts is None:
            raise ValueError("group_mode 'fixed' needs fixed_counts")
        raw = np.asarray(fixed_counts.cpu() if hasattr(fixed_counts, "cpu") else fixed_counts)
        if not (np.array_equal(raw, np.round(raw)) and ((raw >= 0) & (raw <= nobj)).all()):
            raise ValueError(f"fixed_counts: integer counts in [0, {nobj}]")      # (before the int32 cast could wrap them)
        fc = np.ascontiguousarray(np.broadcast_to(raw, (nenv, nobj)), dtype=np.int32)
        keep.append(fc)
        c.fixed_counts = fc.ctypes.data
    c.n_materials, c.color_mode = int(n_materials), COLOR_MODES[color_mode]
    if color_mode == "palette":
        if palette is None:
            raise ValueError("color_mode 'palette' needs a palette")
        pal = np.ascontiguousarray(np.asarray(palette.cpu() if hasattr(palette, "cpu") else palette, dtype=np.float64))
        if pal.ndim != 2 or pal.shape[1] != 4:
            raise ValueError("palette: [rows, 4] rgba")
        keep.append(pal)
        c.palette, c.n_palette = pal.ctypes.data, len(pal)
    c.scale_low, c.scale_high = float(scale_range[0]), float(scale_range[1])
    ncand = 0 if mesh_candidates is None else len(mesh_candidates)
    c.mesh_mode = 0 if mesh_candidates is None else (1 if replace else 2)
    c.n_candidates = ncand
    c.seed, c.epoch = int(seed), int(epoch)
    dev = t.device(device) if out is None else out.group.device
    if out is None:
        i32, f64 = dict(dtype=t.int32, device=dev), dict(dtype=t.float64, device=dev)
        out = ObjectGroups(t.full((nenv, nobj), -1, **i32), t.zeros(nenv, nobj, **i32), t.full((nenv, nobj), -1, **i32),
                           t.zeros(nenv, nobj, 4, **f64), t.zeros(nenv, nobj, **f64), t.full((nenv, nobj), -1, **i32), t.zeros(nenv, nobj, **f64),
                           t.zeros(nenv, nobj, 4, **f64), t.zeros(nenv, **i32))
    else:
        for k, x in out._asdict().items():
            want = (nenv,) if k == "ngroups" else (nenv, nobj, 4) if k in ("rgba", "quat") else (nenv, nobj)
            dt = t.float64 if k in ("rgba", "scale", "yaw", "quat") else t.int32
            if not t.is_tensor(x) or tuple(x.shape) != want or x.dtype != dt or not x.is_contiguous() or x.device != dev:
                raise ValueError(f"out.{k}: a contiguous {dt} tensor {want} on {dev}")
    o = engine.GroupsOut(**{k: ptr(x) for k, x in out._asdict().items()})
    mk = device_mask(t, mask, nenv, dev)
    with t.cuda.device(dev):
        engine._check(engine.lib().rg_object_groups(ctypes.byref(c), ptr(mk), nenv, ctypes.byref(o), current_stream(t, dev)))
    del keep
    return out


# ---- hand-offs to the later reset stages
def active(g):
    """[nenv, nobj] bool: the slots that hold an object (the placement's and BatchedBlockScene.place's `active`)"""
    return g.group >= 0


def goal_groups(g):
    """group ids for BatchedRearrangeGoal.set_groups (a masked call into the same `out` keeps the other environments' ids)"""
    return g.group


def block_scale(g):
    """size scales for BatchedBlockScene.rescale: 1 where a slot holds no object, so a parked block keeps its size"""
    import torch as t

    return t.where(g.group >= 0, g.scale, t.ones_like(g.scale))


def mesh_draw(g, candidates):
    """BatchedMeshScene.set_objects' draw: candidates[mesh] per slot ([nenv, nobj] int64), -1 for an empty slot"""
    import torch as t

    cand = t.as_tensor(np.asarray(candidates, dtype=np.int64), device=g.mesh.device)
    return t.where(g.mesh >= 0, cand[g.mesh.clamp(min=0).long()], t.full_like(g.mesh, -1, dtype=t.int64))


def mesh_scale(g, library, candidates, **kw):
    """ObjectLibrary.object_scales of the drawn objects at their size scales (keywords: mesh_scale, normalize_mesh,
    normalized_mesh_size), as BatchedMeshScene.set_objects takes it"""
    return library.object_scales(mesh_draw(g, candidates), g.scale, **kw)


def initial_quat(g):
    """the initial rotations for bounding_boxes(quat): each object's yaw quaternion, the identity where a slot holds no object"""
    import torch as t

    ident = t.zeros_like(g.quat)
    ident[..., 0] = 1.0
    return t.where((g.group >= 0)[..., None], g.quat, ident)
