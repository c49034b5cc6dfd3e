"""Per-environment YCB object draws as ONE padded batch (SURVEY 8(f) row 3: per-env mesh sets over a shared hull library).

The reference's ycb environments draw their objects again at every reset, with replacement (robogym/envs/rearrange/ycb.py:67-84,
common/mesh.py:49-52), and rebuild the model with them.  Here ONE "slotted" model is compiled per scene: every `object<k>` body
holds P mesh part geoms (P = the largest part count of the library), and the hulls of every library object sit in its mesh
tables.  An environment picks its objects by its own `geom_dataid` row (a part that its object does not have is disabled:
geom_dataid -1), its own part and body rows, and its own pair list, which the engine derives from that row
(`BatchedSim.update_pairs`, include/robogym_b200.h: rg_batch_update_pairs), so the collision stage streams only the pairs of
the parts that exist.

* `ObjectLibrary.from_blobs(*blobs)`: the objects of compiled rearrange scenes (hulls, part geom rows, body rows), identical
  ones merged.
* `slotted_model(base, library)`: the padded model every environment of a batch shares.
* `compact_model(base, library, draw, scale)`: the model the reference would build for one draw (exactly the parts drawn), with
  every object at its own scale.
* `BatchedMeshScene(sim, library)`: writes a draw per environment into a batch of the slotted model, each object at its own
  scale.

Object scale.  The reference compiles every object with `<mesh scale="s s s">` on each of its parts (common/utils.py:250-281,
make_mesh_object; s from common/mesh.py:66-102 and simulation/mesh.py:59, restated by `ObjectLibrary.object_scales`).  The
compiler then scales the hull, the part's position in its body, its size, bounding sphere and bounding box by s, the body's mass
by s^3, its inertia by s^5 and its centre of mass by s (`SCALED_PART_FIELDS`, `scaled_body_rows`).  Two slots that draw the same
object share its library hulls, so a batch scales a part in the narrow phase with the engine's per-environment
`geom_mesh_scale` row instead of editing the hull; its geom_aabb stays the unscaled hull's, which the engine scales.
"""
import numpy as np

from . import mjcf, modelblob, rearrange_placement

GEOM_MESH = 7
# rows of a part geom that come from the library (relative to its body); geom_bodyid / geom_dataid are the slot's
PART_FIELDS = ("geom_type", "geom_contype", "geom_conaffinity", "geom_condim", "geom_priority", "geom_size", "geom_pos", "geom_quat",
               "geom_rbound", "geom_aabb", "geom_friction", "geom_margin", "geom_gap", "geom_solmix", "geom_solref", "geom_solimp")
BODY_FIELDS = ("body_mass", "body_inertia", "body_ipos", "body_iquat")
# what a draw changes per environment (BatchedMeshScene.set_objects)
SCENE_GEOM_FIELDS = ("geom_pos", "geom_quat", "geom_size", "geom_rbound", "geom_aabb")
GEOM_ARRAYS = [name for _, name, cnt in modelblob.ARRAYS if cnt.split("*")[0].strip() == "ngeom"]
SET_CONST_FIELDS = ("dof_invweight0", "body_invweight0", "body_subtreemass", "opt_meaninertia")
# part rows that scale with the object (geom_aabb too in a compiled model, but not in a batch: the engine scales it there)
SCALED_PART_FIELDS = ("geom_pos", "geom_size", "geom_rbound")
# part rows a draw does NOT write per environment: the int ones cannot be bound per environment, and the material ones are
# set per slot (BatchedMeshScene.set_material), not per object.  Every part of every library object must share them.
SHARED_PART_FIELDS = tuple(f for f in PART_FIELDS if f not in SCENE_GEOM_FIELDS)


def _rows(m, name, count_name):
    return np.asarray(m[name]).reshape(m[count_name], -1)


def scaled_body_rows(body, s):
    """an object's body rows (BODY_FIELDS) at uniform scale s: mass s^3, inertia s^5, centre of mass s, principal axes kept"""
    return dict(body_mass=body["body_mass"] * s ** 3, body_inertia=body["body_inertia"] * s ** 5, body_ipos=body["body_ipos"] * s,
                body_iquat=body["body_iquat"])


def _slot_bodies(m, names):
    out = []
    while f"object{len(out)}" in names["body"]:
        out.append(names["body"].index(f"object{len(out)}"))
    return out


class Hull:
    """One convex hull: vertices [n, 3], triangles [f, 3] and the edge adjacency (local ids, CSR)."""

    def __init__(self, vert, face, adjadr, adj):
        self.vert, self.face, self.adjadr, self.adj = vert, face, adjadr, adj
        self.key = b"".join(np.ascontiguousarray(a).tobytes() for a in (vert.astype("<f8"), face.astype("<i4"), adjadr.astype("<i4"), adj.astype("<i4")))

    @classmethod
    def of(cls, m, mid):
        va, nv = int(m["mesh_vertadr"][mid]), int(m["mesh_vertnum"][mid])
        fa, nf = int(m["mesh_faceadr"][mid]), int(m["mesh_facenum"][mid])
        aa = np.asarray(m["mesh_adjadr"][va:va + nv + 1])
        return cls(_rows(m, "mesh_vert", "nmeshvert")[va:va + nv].copy(), _rows(m, "mesh_face", "nmeshface")[fa:fa + nf].copy(),
                   aa - aa[0], np.asarray(m["mesh_adj"][aa[0]:aa[-1]]).copy())


class LibraryEntry:
    def __init__(self, hulls, parts, body):
        self.hulls = hulls              # [Hull] one per part
        self.parts = parts              # field -> [nparts, width] rows of the part geoms (PART_FIELDS)
        self.body = body                # field -> [width] rows of the object's body (BODY_FIELDS)
        self.nparts = len(hulls)
        self.key = b"".join([h.key for h in hulls] + [np.ascontiguousarray(parts[f]).tobytes() for f in PART_FIELDS]
                            + [np.ascontiguousarray(body[f]).tobytes() for f in BODY_FIELDS])

    def _points(self):
        """every hull vertex in the body frame"""
        return np.concatenate([h.vert @ _quat2mat(self.parts["geom_quat"][j]).T + self.parts["geom_pos"][j] for j, h in enumerate(self.hulls)])

    def lowest_point(self):
        """lowest hull point of the object in its body frame (z), for placing it on a surface (at scale s: s times this)"""
        z = np.inf
        for j, h in enumerate(self.hulls):
            R = _quat2mat(self.parts["geom_quat"][j])
            z = min(z, float((h.vert @ R.T)[:, 2].min() + self.parts["geom_pos"][j][2]))
        return z

    @property
    def extents(self):
        """[3] size of the object's axis-aligned box in its body frame.  A hull keeps the extreme points of its mesh, so this is
        what the reference measures as get_combined_mesh(files).extents (common/mesh.py:76-80)."""
        p = self._points()
        return p.max(0) - p.min(0)


def _quat2mat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


class ObjectLibrary:
    """The `object<k>` bodies of compiled rearrange scenes; identical objects of different blobs are one entry.
    `identity[i]` is the draw that reproduces blob i (its objects' entry indices, slot by slot)."""

    def __init__(self):
        self.entries, self.identity, self._index = [], [], {}

    @classmethod
    def from_blobs(cls, *blobs):
        lib = cls()
        for blob in blobs:
            m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
            draw = []
            for b in _slot_bodies(m, names):
                geoms = np.nonzero(np.asarray(m["geom_bodyid"]) == b)[0]
                if not all(m["geom_type"][g] == GEOM_MESH for g in geoms):
                    raise ValueError("mesh scenes: every part of an object must be a mesh geom")
                e = LibraryEntry([Hull.of(m, int(m["geom_dataid"][g])) for g in geoms],
                                 {f: _rows(m, f, "ngeom")[geoms].copy() for f in PART_FIELDS},
                                 {f: _rows(m, f, "nbody")[b].copy() for f in BODY_FIELDS})
                if e.key not in lib._index:
                    lib._index[e.key] = len(lib.entries)
                    lib.entries.append(e)
                draw.append(lib._index[e.key])
            lib.identity.append(draw)
        ref = lib.entries[0].parts
        for e in lib.entries:
            for f in SHARED_PART_FIELDS:
                if not (e.parts[f] == ref[f][0]).all():
                    raise ValueError(f"mesh scenes: every part of every object must have the same {f} (a draw does not write it)")
        return lib

    @property
    def part_counts(self):
        return [e.nparts for e in self.entries]

    @property
    def max_parts(self):
        return max(self.part_counts)

    def object_scales(self, draw, size_scale, mesh_scale=1.0, normalize_mesh=False, normalized_mesh_size=0.05):
        """The scale the reference compiles each drawn object with ([nenv, nslot] float64; 1 for an empty slot), from the
        randomised size scales `size_scale` [nenv, nslot] (sample_object_size_scales), as MeshRearrangeEnv._recreate_sim
        (common/mesh.py:66-102) and make_objects_xml (simulation/mesh.py:59) compute it: in an environment with 10 or more
        objects (drawn slots; the reference's num_objects) no object is scaled up by its size scale and all shrink by
        (10 / n) ** 0.5; `normalize_mesh` scales an object so that half its largest extent is `normalized_mesh_size`;
        `mesh_scale` (simulation_params.mesh_scale) multiplies everything."""
        draw = np.asarray(draw.cpu() if hasattr(draw, "cpu") else draw, dtype=np.int64)
        size = np.broadcast_to(np.asarray(size_scale.cpu() if hasattr(size_scale, "cpu") else size_scale, dtype=np.float64), draw.shape)
        n = (draw >= 0).sum(-1, keepdims=True)
        glob = np.where(n < 10, 1.0, np.sqrt(10.0 / np.maximum(n, 1)))
        s = np.where(n >= 10, np.minimum(size, 1.0), size)
        if normalize_mesh:
            half = np.array([e.extents.max() / 2.0 for e in self.entries])
            s = s * (normalized_mesh_size / half[np.maximum(draw, 0)])
        return np.where(draw >= 0, s * glob * mesh_scale, 1.0)


def sample_object_size_scales(nenv, nslot, low, high, generator=None, device=None):
    """exp(U(-low, high)) per environment and slot ([nenv, nslot] float64 tensor on the generator's device, else `device`): the
    randomised object size scale of the reference (common/base.py:594-601, parameters object_scale_low / object_scale_high)."""
    import torch

    dev = generator.device if generator is not None else device
    u = torch.rand(nenv, nslot, generator=generator, device=dev, dtype=torch.float64)
    return torch.exp(-low + (low + high) * u)


def _build(base_blob, library, slots, set_const):
    """The base scene with slot k holding slots[k] = (entry index or -1, part geoms, scale): the entry's parts, then disabled
    ones (geom_dataid -1); a drawn object at scale s != 1 gets hulls scaled by s and the rows the compiler makes for them.  Non-object geoms keep their rows and order; meshes identical to one of the base's are shared, the
    others appended; the pair list is the base's, expanded from parts to slots."""
    m, names = modelblob.unpack(base_blob), modelblob.unpack_names(base_blob)
    bodies = _slot_bodies(m, names)
    if len(slots) != len(bodies):
        raise ValueError(f"the base scene has {len(bodies)} object slots, the draw {len(slots)}")
    out = {k: m[k] for k in modelblob.DIMS}
    gb = np.asarray(m["geom_bodyid"])
    slot_of_body = {b: k for k, b in enumerate(bodies)}
    # ---- meshes: the base's table, then the library hulls it does not hold
    mesh_ids = {Hull.of(m, i).key: i for i in range(m["nmesh"])}
    new_hulls = []

    def mesh_id(h):
        if h.key not in mesh_ids:
            mesh_ids[h.key] = m["nmesh"] + len(new_hulls)
            new_hulls.append(h)
        return mesh_ids[h.key]

    # ---- geoms: walk the base, replacing each object's parts by the slot's
    rows = {f: [] for f in GEOM_ARRAYS}
    gnames, key = [], []          # key: ("s", k) for part geoms of slot k, ("g", old id) for the others
    old2new, done = {}, set()
    for g in range(m["ngeom"]):
        b = int(gb[g])
        if b not in slot_of_body:
            old2new[g] = len(key)
            for f in GEOM_ARRAYS:
                rows[f].append(_rows(m, f, "ngeom")[g])
            gnames.append(names["geom"][g]); key.append(("g", g))
            continue
        k = slot_of_body[b]
        if k in done:
            continue
        done.add(k)
        e, P, sc = slots[k]
        tmpl = library.entries[e] if e >= 0 else library.entries[library.identity[0][0]]
        if e >= 0 and sc != 1.0:
            tmpl = LibraryEntry([Hull(h.vert * sc, h.face, h.adjadr, h.adj) for h in tmpl.hulls],
                                {f: tmpl.parts[f] * sc if f in SCALED_PART_FIELDS + ("geom_aabb",) else tmpl.parts[f] for f in PART_FIELDS},
                                scaled_body_rows(tmpl.body, sc))
        for j in range(P):
            on = e >= 0 and j < tmpl.nparts
            for f in GEOM_ARRAYS:
                if f == "geom_bodyid":
                    rows[f].append(np.array([b]))
                elif f == "geom_dataid":
                    rows[f].append(np.array([mesh_id(tmpl.hulls[j]) if on else -1]))
                elif on or f in ("geom_type", "geom_contype", "geom_conaffinity", "geom_condim", "geom_priority", "geom_friction",
                                 "geom_margin", "geom_gap", "geom_solmix", "geom_solref", "geom_solimp"):
                    rows[f].append(tmpl.parts[f][j if on else 0])
                else:                                              # a disabled part: no extent, identity frame
                    rows[f].append(np.array([1.0, 0, 0, 0]) if f == "geom_quat" else np.zeros(_rows(m, f, "ngeom").shape[1]))
            gnames.append(f"object{k}-{j}"); key.append(("s", k))
        if e >= 0:
            for f in BODY_FIELDS:
                _rows(m, f, "nbody")[b] = tmpl.body[f]
    ngeom = len(key)
    for f in GEOM_ARRAYS:
        out[f] = np.concatenate([np.asarray(r, dtype=m[f].dtype).reshape(-1) for r in rows[f]])
    out["ngeom"] = ngeom
    # bodies: geom ranges
    bid = out["geom_bodyid"]
    out["body_geomnum"] = np.bincount(bid, minlength=m["nbody"]).astype(np.int32)
    adr = np.full(m["nbody"], -1, np.int32)
    for g in range(ngeom - 1, -1, -1):
        adr[bid[g]] = g
    out["body_geomadr"] = adr
    # tendon wraps around geoms follow them
    wt, wo = np.asarray(m["wrap_objid"]).copy(), np.asarray(m["wrap_type"])
    for w in range(m["nwrap"]):
        if wt[w] >= 0 and wo[w] in (4, 5):
            wt[w] = old2new[int(wt[w])]
    out["wrap_objid"] = wt
    mnames = _add_hulls(out, m, names["mesh"], new_hulls)
    # ---- pairs: slot k <-> X exists iff the base had a pair between a part of object k and X; expanded to every part
    kid = {}
    kg = np.array([kid.setdefault(k, len(kid)) for k in key])
    rel = np.zeros((len(kid), len(kid)), bool)
    okey = [("s", slot_of_body[int(gb[g])]) if int(gb[g]) in slot_of_body else ("g", g) for g in range(m["ngeom"])]
    for a, c in zip(m["pair_geom1"], m["pair_geom2"]):
        if okey[a] in kid and okey[c] in kid:              # (an empty slot has no geoms)
            ka, kc = kid[okey[a]], kid[okey[c]]
            rel[ka, kc] = rel[kc, ka] = True
    g1, g2 = np.nonzero(np.triu(rel[kg][:, kg], 1))           # row-major: the compiler's (g1 < g2) order
    t = out["geom_type"]
    swap = t[g1] > t[g2]                                        # type1 <= type2, as the compiler orders a pair
    out["pair_geom1"], out["pair_geom2"] = np.where(swap, g2, g1), np.where(swap, g1, g2)
    out["npair"] = len(g1)
    for _, name, _ in modelblob.ARRAYS:
        out.setdefault(name, m[name])
    new_names = dict(names, geom=gnames, mesh=mnames)
    blob = modelblob.pack(out, new_names)
    if set_const:
        cm = mjcf.CompiledModel.from_blob(blob, new_names)
        mjcf.set_const(cm.m)
        for f in SET_CONST_FIELDS:
            out[f] = np.asarray(cm.m[f], dtype=np.float64).reshape(-1)
        blob = modelblob.pack(out, new_names)
    return blob


def slotted_model(base_blob, library, parts_per_slot=None):
    """The model a batch of per-environment draws shares: every object slot holds `parts_per_slot` (default: the library's
    largest part count) mesh geoms `object<k>-<j>`, the library's hulls are in its mesh tables, and its own rows hold the base
    scene's objects (surplus parts disabled: geom_dataid -1).  Geoms stay contiguous per body; the other geoms keep their rows
    and order."""
    P = library.max_parts if parts_per_slot is None else int(parts_per_slot)
    if P < library.max_parts:
        raise ValueError(f"parts_per_slot={P} is below the library's largest object ({library.max_parts} parts)")
    m, names = modelblob.unpack(base_blob), modelblob.unpack_names(base_blob)
    ident = _base_draw(base_blob, library)
    blob = _build(base_blob, library, [(e, P, 1.0) for e in ident], set_const=False)
    # every library hull, so that any draw is a change of geom_dataid rows only
    m2 = modelblob.unpack(blob)
    have = {Hull.of(m2, i).key for i in range(m2["nmesh"])}
    extra = [h for e in library.entries for h in e.hulls if h.key not in have and not have.add(h.key)]
    if extra:
        blob = _append_hulls(blob, extra)
    return blob


def _append_hulls(blob, hulls):
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    out = dict(m)
    return modelblob.pack(out, dict(names, mesh=_add_hulls(out, m, names["mesh"], hulls)))


def _add_hulls(out, m, mesh_names, hulls):
    """out's mesh tables = m's followed by `hulls` (named library<i>); returns the mesh names"""
    nv, nf, na = m["nmeshvert"], m["nmeshface"], m["nmeshadj"]
    vadr, vnum, fadr, fnum = list(m["mesh_vertadr"]), list(m["mesh_vertnum"]), list(m["mesh_faceadr"]), list(m["mesh_facenum"])
    vert, face, adjadr, adj = [_rows(m, "mesh_vert", "nmeshvert")], [_rows(m, "mesh_face", "nmeshface")], [np.asarray(m["mesh_adjadr"][:-1])], [np.asarray(m["mesh_adj"])]
    for h in hulls:
        vadr.append(nv); vnum.append(len(h.vert)); fadr.append(nf); fnum.append(len(h.face))
        vert.append(h.vert); face.append(h.face); adjadr.append(h.adjadr[:-1] + na); adj.append(h.adj)
        nv += len(h.vert); nf += len(h.face); na += len(h.adj)
    out.update(nmesh=len(vadr), nmeshvert=nv, nmeshface=nf, nmeshadj=na, mesh_vertadr=np.array(vadr), mesh_vertnum=np.array(vnum),
               mesh_faceadr=np.array(fadr), mesh_facenum=np.array(fnum), mesh_vert=np.concatenate(vert).reshape(-1),
               mesh_face=np.concatenate(face).reshape(-1), mesh_adjadr=np.concatenate(adjadr + [np.array([na])]), mesh_adj=np.concatenate(adj))
    nl = sum(1 for n in mesh_names if n and n.startswith("library"))
    return list(mesh_names) + [f"library{nl + i}" for i in range(len(hulls))]


def _base_draw(base_blob, library):
    m, names = modelblob.unpack(base_blob), modelblob.unpack_names(base_blob)
    draw = []
    for b in _slot_bodies(m, names):
        geoms = np.nonzero(np.asarray(m["geom_bodyid"]) == b)[0]
        e = LibraryEntry([Hull.of(m, int(m["geom_dataid"][g])) for g in geoms], {f: _rows(m, f, "ngeom")[geoms].copy() for f in PART_FIELDS},
                         {f: _rows(m, f, "nbody")[b].copy() for f in BODY_FIELDS})
        if e.key not in library._index:
            raise ValueError("the base scene's objects must be in the library")
        draw.append(library._index[e.key])
    return draw


def compact_model(base_blob, library, draw, scale=None):
    """The model the reference builds for one draw (`draw`: a library index per slot, -1 = empty slot) with the objects at
    `scale` (a finite scale > 0 per slot, None = all 1): each slot holds exactly the drawn object's parts, a scaled object
    its own hulls with the vertices multiplied by its scale, and the constants mj_setConst derives are recomputed.  The
    identity draw at scale 1 is the base scene itself, byte for byte."""
    draw = [int(e) for e in draw]
    scale = [1.0] * len(draw) if scale is None else [float(x) for x in np.asarray(scale, dtype=np.float64).reshape(-1)]
    if len(scale) != len(draw) or not all(np.isfinite(x) and x > 0 for x in scale):
        raise ValueError("compact_model: scale needs one finite value > 0 per slot")
    if draw == _base_draw(base_blob, library) and all(s == 1.0 for s in scale):
        return bytes(base_blob)
    return _build(base_blob, library, [(e, library.entries[e].nparts if e >= 0 else 0, s) for e, s in zip(draw, scale)], set_const=True)


class BatchedMeshScene:
    """A draw per environment on a batch of `slotted_model(...)`: set_objects writes each environment's part geom rows,
    geom_dataid row and object body rows, recomputes the derived constants on the device and rederives the pair lists."""

    def __init__(self, sim, library, prefix="object", park_origin=(3.0, -1.0), park_pitch=0.25):
        self.sim, self.t, self.library = sim, sim.torch, library
        m = sim.model.host
        self.m = m
        self.bodies, self.geoms, self.qadr, self.dadr = [], [], [], []
        while True:
            try:
                b = sim.model.name2id("body", f"{prefix}{len(self.bodies)}")
            except ValueError:
                break
            g = np.nonzero(np.asarray(m["geom_bodyid"]) == b)[0]
            j = sim.model.name2id("joint", f"{prefix}{len(self.bodies)}:joint")
            self.bodies.append(b); self.geoms.append(g); self.qadr.append(int(m["jnt_qposadr"][j])); self.dadr.append(int(m["jnt_dofadr"][j]))
        self.nslot = len(self.bodies)
        if not self.nslot:
            raise ValueError("no objects in the model")
        self.P = len(self.geoms[0])
        if any(len(g) != self.P or g[-1] - g[0] + 1 != self.P for g in self.geoms) or self.P < library.max_parts:
            raise ValueError("the model is not a slotted model of this library (slotted_model)")
        mesh = {Hull.of(m, i).key: i for i in range(m["nmesh"])}
        try:
            self.mesh_ids = [[mesh[h.key] for h in e.hulls] for e in library.entries]
        except KeyError:
            raise ValueError("the model lacks hulls of this library (slotted_model)") from None
        self.lowest = np.array([e.lowest_point() for e in library.entries])
        self.park_origin, self.park_pitch = park_origin, park_pitch
        self.draw = self.scale = None
        self._rows = {}

    def _row(self, name):
        if name not in self._rows:
            dt = np.int64 if name == "geom_dataid" else np.float64
            self._rows[name] = np.repeat(np.asarray(self.m[name], dtype=dt).reshape(1, -1), self.sim.nenv, axis=0)
        return self._rows[name]

    def set_objects(self, draw, scale=None):
        """draw [nenv, nslot]: a library index per environment and slot, -1 = empty slot: all parts disabled and the body keeps
        the shared model's rows, so its constants do not depend on earlier draws.  Nothing collides with an empty slot's body:
        place() parks it, and it then falls freely under gravity for the rest of the episode, so its pose and velocity are not
        observations of anything.
        scale [nenv, nslot] (finite, > 0; None = 1 everywhere): each drawn object at its own uniform scale, with the rows the
        model compiler makes for `<mesh scale="s s s">` (module docstring) and the engine's geom_mesh_scale row = s on the slot's
        part geoms.  Without scales the batch binds no geom_mesh_scale row (or writes ones into one bound before)."""
        draw = np.asarray(draw.cpu() if hasattr(draw, "cpu") else draw, dtype=np.int64).reshape(self.sim.nenv, self.nslot)
        if ((draw < -1) | (draw >= len(self.library.entries))).any():
            raise ValueError("draw: library indices or -1")
        nenv = self.sim.nenv
        if scale is not None:
            scale = np.asarray(scale.cpu() if hasattr(scale, "cpu") else scale, dtype=np.float64).reshape(nenv, self.nslot)
            if not (np.isfinite(scale).all() and (scale > 0).all()):
                raise ValueError("scale: finite and > 0 per environment and slot")
            scale = np.where(draw >= 0, scale, 1.0)
        did = self._row("geom_dataid")
        grow = {f: self._row(f).reshape(nenv, self.m["ngeom"], -1) for f in SCENE_GEOM_FIELDS}
        brow = {f: self._row(f).reshape(nenv, self.m["nbody"], -1) for f in BODY_FIELDS}
        for k in range(self.nslot):
            g0 = int(self.geoms[k][0])
            for e in np.unique(draw[:, k]):
                envs = np.nonzero(draw[:, k] == e)[0]
                n = self.library.entries[e].nparts if e >= 0 else 0
                ids = np.full(self.P, -1)
                ids[:n] = self.mesh_ids[e] if e >= 0 else []
                did[np.ix_(envs, np.arange(g0, g0 + self.P))] = ids
                for f in SCENE_GEOM_FIELDS:
                    r = np.zeros((self.P, grow[f].shape[2]))
                    if f == "geom_quat":
                        r[:, 0] = 1.0
                    if n:
                        r[:n] = self.library.entries[e].parts[f]
                    if scale is not None and f in SCALED_PART_FIELDS:
                        grow[f][envs, g0:g0 + self.P] = r[None] * scale[envs, k, None, None]
                    else:
                        grow[f][envs, g0:g0 + self.P] = r
                for f in BODY_FIELDS:
                    if e < 0:
                        brow[f][envs, self.bodies[k]] = _rows(self.m, f, "nbody")[self.bodies[k]]
                    elif scale is None:
                        brow[f][envs, self.bodies[k]] = self.library.entries[e].body[f]
                    else:
                        brow[f][envs, self.bodies[k]] = scaled_body_rows(self.library.entries[e].body, scale[envs, k, None])[f]
        self.draw, self.scale = draw, scale
        names = ("geom_dataid",) + SCENE_GEOM_FIELDS + BODY_FIELDS
        if scale is not None or "geom_mesh_scale" in self._rows:
            gs = self._rows.setdefault("geom_mesh_scale", np.ones((nenv, self.m["ngeom"])))
            gs[:] = 1.0
            if scale is not None:
                for k in range(self.nslot):
                    gs[:, self.geoms[k]] = scale[:, k, None]
            names += ("geom_mesh_scale",)
        for f in names:
            self.sim.set_param(f, self._rows[f])
        out = self.sim.set_const(fields=SET_CONST_FIELDS)
        self.sim.update_pairs()
        return out

    def place(self, xy, yaw, surface_z, clearance=1e-3):
        """Put the objects down: xy [nenv, nslot, 2], yaw [nenv, nslot], each drawn object resting `clearance` above
        `surface_z` (scalar or [nenv]) by its lowest hull point (at the object's scale); empty slots go to their parking spots on
        the floor, from which their geom-less bodies fall freely.  Velocities zeroed."""
        t, sim = self.t, self.sim
        dev, dt = sim.qpos.device, sim.qpos.dtype
        f = lambda v: (v if t.is_tensor(v) else t.as_tensor(np.asarray(v, dtype=np.float64))).to(device=dev, dtype=dt)
        xy, yaw = f(xy), f(yaw)
        zs = f(surface_z) * t.ones(sim.nenv, device=dev, dtype=dt)
        if self.draw is None:
            raise ValueError("place(): set_objects() first")
        draw = self.draw
        for k in range(self.nslot):
            a, d = self.qadr[k], self.dadr[k]
            on = t.as_tensor(draw[:, k] >= 0, device=dev)
            low = np.where(draw[:, k] >= 0, self.lowest[np.maximum(draw[:, k], 0)], 0.0)
            if self.scale is not None:
                low = low * self.scale[:, k]
            low = t.as_tensor(low, device=dev, dtype=dt)
            px = self.park_origin[0] + self.park_pitch * (k % 4)
            py = self.park_origin[1] + self.park_pitch * (k // 4)
            sim.qpos[:, a] = t.where(on, xy[:, k, 0], t.full_like(zs, px))
            sim.qpos[:, a + 1] = t.where(on, xy[:, k, 1], t.full_like(zs, py))
            sim.qpos[:, a + 2] = t.where(on, zs - low + clearance, t.zeros_like(zs))
            half = t.where(on, 0.5 * yaw[:, k], t.zeros_like(zs))
            sim.qpos[:, a + 3] = t.cos(half); sim.qpos[:, a + 4] = 0.0; sim.qpos[:, a + 5] = 0.0; sim.qpos[:, a + 6] = t.sin(half)
            sim.qvel[:, d:d + 6] = 0.0

    def bounding_boxes(self, quat=None, mask=None):
        """The reference's `_get_bounding_box` of every slot's object (get_mesh_bounding_box) with the object rotated by quat
        ([nenv, nslot, 4] w x y z; None = unrotated): [nenv, nslot, 2, 3] float64 (center relative to the body origin, half size)
        on the device, from each environment's drawn, scaled parts (rg_batch_body_aabb); an empty slot gets a zero box.  Its
        xy feeds rearrange_placement, whose positions place() takes as they are."""
        return rearrange_placement.body_aabb(self.sim, self.bodies, quat, mask)

    def set_material(self, friction=None, solref=None, solimp=None, margin=None):
        """Material rows of every part of a slot, per environment and slot: friction [nenv, nslot, 3], solref [nenv, nslot, 2],
        solimp [nenv, nslot, 5], margin [nenv, nslot]; None leaves an attribute as it is."""
        nenv = self.sim.nenv
        for name, val, w in (("geom_friction", friction, 3), ("geom_solref", solref, 2), ("geom_solimp", solimp, 5), ("geom_margin", margin, 1)):
            if val is None:
                continue
            v = np.broadcast_to(np.asarray(val.cpu() if hasattr(val, "cpu") else val, dtype=np.float64).reshape(nenv, self.nslot, w), (nenv, self.nslot, w))
            rows = self._row(name).reshape(nenv, self.m["ngeom"], w)
            for k in range(self.nslot):
                rows[:, self.geoms[k]] = v[:, k, None, :]
            self.sim.set_param(name, self._rows[name])

