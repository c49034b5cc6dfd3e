"""Per-reset heterogeneous block scenes as ONE padded batch (SURVEY 8(f) row 3).

The reference rebuilds its MuJoCo model on every `reset()` (robogym/envs/rearrange/common/base.py:850-856,897-906): the number of
blocks, their size (`make_block`, common/utils.py:195-216: a box geom of the sampled half-size, mass and inertia from the material's
density), a per-object scale applied to the compiled model (`rescale_object_sizes`, simulation/base.py:712-730: geom_size and
geom_pos only) and the material (friction / solref / solimp / margin, envs/rearrange/materials/*.jsonnet) differ from episode to
episode -- and, in a batch, from environment to environment.  Recompiling 2048 models per reset is not an option on the device;
instead ONE model is compiled with the maximum number of blocks and every environment carries its own rows of the arrays that
differ (`rg_batch_bind_param`), its derived constants recomputed on the device (`rg_set_const`), and a mask of the blocks it uses:

* size: geom_size, geom_rbound, geom_aabb, body_mass, body_inertia, body_iquat rows of each block, computed exactly as the model compiler does
  for a box (robogym_b200/mjcf.py: mass = density * volume, principal inertia m/3 (b^2 + c^2) ...), then body_subtreemass,
  dof_invweight0, body_invweight0 through `BatchedSim.set_const`;
* scale: geom_size *= s (what `_rescale_object` does to a primitive geom: no mass update, like the reference);
* material: geom_friction / geom_solref / geom_solimp / geom_margin rows;
* inactive blocks are parked on the floor away from the table (they rest there; their target geoms do not collide).

Works on any BatchedSim-like object with `set_param` / `set_const`; the per-environment arithmetic is plain torch.
"""
import numpy as np

from . import mjcf, rearrange_placement

GEOM_BOX = 6


def object_dofs(m, bodies):
    """The dof ids of the joints of `bodies` (body_jntadr / body_jntnum), each joint's dofs selected as the reference's
    get_object_damping does (robogym/envs/rearrange/simulation/base.py:530-546: dof_jntid == the object's joint)."""
    dof_jntid = np.asarray(m["dof_jntid"])
    out = []
    for b in bodies:
        j0, nj = int(m["body_jntadr"][b]), int(m["body_jntnum"][b])
        for j in range(j0, j0 + nj):
            out += np.nonzero(dof_jntid == j)[0].tolist()
    return out


def stabilize_objects(sim, bodies, mask=None, n_steps=100, damping=1e-3):
    """The reference's stabilize_objects (robogym/envs/rearrange/common/utils.py:76-93, run by every rearrange reset after
    the objects are placed, base.py:912-913): the objects' dofs get the damping 1e-3, the simulation takes `n_steps` env-steps,
    the damping is put back and forward() runs.  Here that is one launch of n_steps x sim.n_substeps substeps with the damping
    as a launch constant (BatchedSim.settle), then the final forward with each environment's own damping, for every
    environment or those of `mask` (the launch covers just those).

    `bodies` are the object bodies, e.g. BatchedBlockScene.bodies / BatchedMeshScene.bodies.  Every slot's dofs are in the
    list, the parked ones (unused blocks, empty mesh slots) included: environments are independent and a parked object never
    touches the table's objects, so the active objects settle as they would without the parked ones in the list."""
    dofs = object_dofs(sim.model.host, bodies)
    sim.settle(dofs, damping, int(n_steps) * sim.n_substeps, mask=mask, final_forward=True)


class BatchedBlockScene:
    def __init__(self, sim, max_objects=None, prefix="object", park_origin=(3.0, -1.0), park_pitch=0.25):
        self.sim, self.t = sim, sim.torch
        m = sim.model.host
        self.m = m
        n = 0
        self.bodies, self.geoms, self.qadr, self.dadr = [], [], [], []
        while max_objects is None or n < max_objects:
            try:
                b = sim.model.name2id("body", f"{prefix}{n}")
            except ValueError:
                break
            g = [k for k in range(m["ngeom"]) if m["geom_bodyid"][k] == b]
            assert len(g) == 1 and m["geom_type"][g[0]] == GEOM_BOX, "block scenes: one box geom per object"
            j = sim.model.name2id("joint", f"{prefix}{n}:joint")
            self.bodies.append(b); self.geoms.append(g[0]); self.qadr.append(int(m["jnt_qposadr"][j])); self.dadr.append(int(m["jnt_dofadr"][j]))
            n += 1
        assert n > 0, "no objects in the model"
        self.nobj = n
        self.park_origin, self.park_pitch = park_origin, park_pitch
        self.active = self.t.ones(sim.nenv, n, dtype=self.t.bool, device=sim.qpos.device)
        self._rows = {}

    # ---- per-environment model rows
    def _row(self, name):
        """float64 host-side master copy [nenv, count] of a model array, created from the shared model on first use"""
        if name not in self._rows:
            self._rows[name] = self.t.tensor(np.asarray(self.m[name], dtype=np.float64).reshape(1, -1)).repeat(self.sim.nenv, 1)
        return self._rows[name]

    def _push(self, names):
        for n in names:
            self.sim.set_param(n, self._rows[n])

    def set_blocks(self, half_size, density=1000.0):
        """`make_block` with a per-environment size: half_size [nenv, nobj, 3] (or [nenv, nobj] / [nenv] for cubes), density as the
        material gives it (MuJoCo's default 1000 when the material has none).  Writes the size-dependent rows and recomputes the
        derived constants on the device."""
        t = self.t
        hs = t.as_tensor(np.asarray(half_size, dtype=np.float64)) if not t.is_tensor(half_size) else half_size.to(t.float64).cpu()
        if hs.dim() == 1:
            hs = hs[:, None].expand(-1, self.nobj)
        if hs.dim() == 2:
            hs = hs[:, :, None].expand(-1, -1, 3)
        hs = hs.contiguous()
        assert hs.shape == (self.sim.nenv, self.nobj, 3)
        dens = t.as_tensor(np.broadcast_to(np.asarray(density, dtype=np.float64), (self.sim.nenv, self.nobj)).copy())
        size, rb, aabb = self._row("geom_size").view(self.sim.nenv, -1, 3), self._row("geom_rbound"), self._row("geom_aabb").view(self.sim.nenv, -1, 6)
        mass, inertia = self._row("body_mass"), self._row("body_inertia").view(self.sim.nenv, -1, 3)
        iquat = self._row("body_iquat").view(self.sim.nenv, -1, 4)
        vol = 8.0 * hs.prod(dim=2)
        mk = dens * vol
        a2 = hs * hs
        # the compiler's inertial frame: principal moments in decreasing order, right-handed axes (mjcf._eig_frame); for a box
        # in its own frame that is a permutation of the axes -- computed once per distinct shape
        frames = {}
        for k in range(self.nobj):
            g, b = self.geoms[k], self.bodies[k]
            size[:, g] = hs[:, k]
            rb[:, g] = hs[:, k].norm(dim=1)
            aabb[:, g, :3] = 0.0
            aabb[:, g, 3:] = hs[:, k]
            mass[:, b] = mk[:, k]
            diag = t.stack([a2[:, k, 1] + a2[:, k, 2], a2[:, k, 0] + a2[:, k, 2], a2[:, k, 0] + a2[:, k, 1]], dim=1) * (mk[:, k] / 3.0)[:, None]
            cube = (hs[:, k, 0] == hs[:, k, 1]) & (hs[:, k, 1] == hs[:, k, 2])     # cubes: equal moments, the compiler keeps the geom axes
            inertia[cube, b] = diag[cube]
            iquat[cube, b] = t.tensor([1.0, 0.0, 0.0, 0.0], dtype=iquat.dtype)
            for e in (~cube).nonzero().flatten().tolist():
                key = tuple(hs[e, k].tolist())
                if key not in frames:
                    w, v = mjcf._eig_frame(np.diag(np.array([key[1] ** 2 + key[2] ** 2, key[0] ** 2 + key[2] ** 2, key[0] ** 2 + key[1] ** 2])))
                    order = [int(np.argmax(np.abs(v[:, c]))) for c in range(3)]
                    frames[key] = (order, t.tensor(mjcf.mat2quat(v)))
                order, q = frames[key]
                inertia[e, b] = diag[e, order]
                iquat[e, b] = q
        self._push(("geom_size", "geom_rbound", "geom_aabb", "body_mass", "body_inertia", "body_iquat"))
        return self.sim.set_const(fields=("dof_invweight0", "body_invweight0", "body_subtreemass", "opt_meaninertia"))

    def rescale(self, scale):
        """`RearrangeSimulationInterface.rescale_object_sizes` (simulation/base.py:712-730) per environment: the box geom's size (and
        its offset in the body) times `scale` [nenv, nobj]; masses stay, as in the reference.  The bounding data follow the size."""
        t = self.t
        sc = t.as_tensor(np.asarray(scale, dtype=np.float64)) if not t.is_tensor(scale) else scale.to(t.float64).cpu()
        size, rb, aabb = self._row("geom_size").view(self.sim.nenv, -1, 3), self._row("geom_rbound"), self._row("geom_aabb").view(self.sim.nenv, -1, 6)
        gpos = self._row("geom_pos").view(self.sim.nenv, -1, 3)
        for k in range(self.nobj):
            g = self.geoms[k]
            size[:, g] *= sc[:, k:k + 1]
            gpos[:, g] *= sc[:, k:k + 1]
            rb[:, g] = size[:, g].norm(dim=1)
            aabb[:, g, 3:] = size[:, g]
        self._push(("geom_size", "geom_pos", "geom_rbound", "geom_aabb"))

    def set_material(self, friction=None, solref=None, solimp=None, margin=None):
        """Material rows of the blocks per environment (envs/rearrange/materials/*.jsonnet -> geom attributes): friction [nenv, 3],
        solref [nenv, 2], solimp [nenv, 5], margin [nenv]; None leaves an attribute as compiled."""
        t = self.t
        for name, val, w in (("geom_friction", friction, 3), ("geom_solref", solref, 2), ("geom_solimp", solimp, 5), ("geom_margin", margin, 1)):
            if val is None:
                continue
            v = t.as_tensor(np.asarray(val, dtype=np.float64)).reshape(self.sim.nenv, w)
            rows = self._row(name).view(self.sim.nenv, -1, w)
            for g in self.geoms:
                rows[:, g] = v
            self._push((name,))

    def bounding_boxes(self, quat=None, mask=None):
        """The reference's `_get_bounding_box` of every block (get_block_bounding_box) rotated by quat ([nenv, nobj, 4] w x y z;
        None = unrotated): [nenv, nobj, 2, 3] float64 (center relative to the body origin, half size) on the device, from each
        environment's size and scale rows (rg_batch_body_aabb).  Feeds rearrange_placement, whose positions place() takes."""
        return rearrange_placement.body_aabb(self.sim, self.bodies, quat, mask)

    # ---- which blocks an environment uses, and where they are
    def place(self, xy, yaw, z, active=None):
        """Put the blocks down: xy [nenv, nobj, 2], yaw [nenv, nobj], z [nenv, nobj] (centre height); `active` [nenv, nobj] bool --
        the others go to their parking spots on the floor, out of everything's reach, velocities zeroed."""
        t, sim = self.t, self.sim
        dev, dt = sim.qpos.device, sim.qpos.dtype
        if active is not None:
            self.active = active.to(device=dev, dtype=t.bool)
        f = lambda v: (v if t.is_tensor(v) else t.as_tensor(np.asarray(v))).to(device=dev, dtype=dt)
        xy, yaw, z = f(xy), f(yaw), f(z)
        size = self._row("geom_size").view(sim.nenv, -1, 3).to(device=dev, dtype=dt) if "geom_size" in self._rows else None
        for k in range(self.nobj):
            a, d = self.qadr[k], self.dadr[k]
            on = self.active[:, k]
            px = t.full_like(z[:, k], self.park_origin[0] + self.park_pitch * (k % 4))
            py = t.full_like(z[:, k], self.park_origin[1] + self.park_pitch * (k // 4))
            hz = size[:, self.geoms[k], 2] if size is not None else t.full_like(z[:, k], float(np.asarray(self.m["geom_size"]).reshape(-1, 3)[self.geoms[k], 2]))
            sim.qpos[:, a] = t.where(on, xy[:, k, 0], px)
            sim.qpos[:, a + 1] = t.where(on, xy[:, k, 1], py)
            sim.qpos[:, a + 2] = t.where(on, z[:, k], hz + 1e-3)           # parked: resting on the floor plane (z = 0)
            half = t.where(on, 0.5 * yaw[:, k], t.zeros_like(yaw[:, k]))
            sim.qpos[:, a + 3] = t.cos(half); sim.qpos[:, a + 4] = 0.0; sim.qpos[:, a + 5] = 0.0; sim.qpos[:, a + 6] = t.sin(half)
            sim.qvel[:, d:d + 6] = 0.0
