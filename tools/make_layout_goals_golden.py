"""Record the reference's domino, attached-block and fixed layout goals into tests/golden/reference_layout_goals.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_layout_goals_golden.py`.  It imports
the reference on the mujoco_py shim (as tools/make_goal_variants_golden.py does) and runs the reference's OWN functions on
generator instances over a minimal simulation stand-in:

- `DominoStateGoal._sample_next_goal_positions` (goals/dominos.py), whose target boxes are the reference's
  `get_block_bounding_box` of target bodies whose quaternions the reference's `set_target_quat` wrote; the stand-in's
  `get_body_xmat` is MuJoCo's kinematics of such a body (mju_normalize4, then mju_quat2Mat);
- `AttachedBlockStateGoal._sample_next_goal_positions` (goals/attached_block_state.py);
- `ObjectFixedStateGoal._sample_next_goal_positions` (goals/object_state_fixed.py) with table_setting's and wordblocks'
  relative placements and rotations, and with placements beyond the area.

Random numbers come from the replay RandomState of tests/layout_goals_rng.py (draw d at the layout goals' counter d).  Each
domino case records the fitting retry (-1 when none fitted within the reference's MAX_RETRY) and the angles of the last arc
the reference tried."""
import gzip
import json
import logging
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
REF = os.environ.get("ROBOGYM_REFERENCE", "/root/reference")
for p in (os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests"), REF, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_layout_goals.json.gz")
PLACEMENT = os.path.join(ROOT, "tests", "golden", "reference_placement.json.gz")
TABLE = [1.3, 0.75, 0.2, 0.6075, 0.7655, 0.2]          # rearrange scenes: table body pos, table geom half size


def mj_body_xmat(q):
    """MuJoCo's xmat of a body under the world body with quaternion q: mju_normalize4, then mju_quat2Mat"""
    q = np.array(q, dtype=np.float64)
    n = np.sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    if n < 1e-15:
        q = np.array([1.0, 0.0, 0.0, 0.0])
    elif abs(n - 1.0) > 1e-15:
        q = q / n
    if q[0] == 1 and q[1] == 0 and q[2] == 0 and q[3] == 0:
        return np.eye(3)
    q00, q01, q02, q03 = q[0] * q[0], q[0] * q[1], q[0] * q[2], q[0] * q[3]
    q11, q12, q13, q22, q23, q33 = q[1] * q[1], q[1] * q[2], q[1] * q[3], q[2] * q[2], q[2] * q[3], q[3] * q[3]
    return np.array([[q00 + q11 - q22 - q33, 2 * (q12 - q03), 2 * (q13 + q02)],
                     [2 * (q12 + q03), q00 - q11 + q22 - q33, 2 * (q23 - q01)],
                     [2 * (q13 - q02), 2 * (q23 + q01), q00 - q11 - q22 + q33]])


def main():
    import robogym_b200.mujoco_py_shim as shim
    from layout_goals_rng import LayoutReplayRandomState

    shim.install()
    logging.disable(logging.WARNING)
    from robogym.envs.rearrange.common.utils import PlacementArea, get_block_bounding_box
    from robogym.envs.rearrange.goals import dominos
    from robogym.envs.rearrange.goals.attached_block_state import AttachedBlockStateGoal
    from robogym.envs.rearrange.goals.dominos import DominoStateGoal
    from robogym.envs.rearrange.goals.object_state_fixed import ObjectFixedStateGoal
    from robogym.envs.rearrange.simulation.base import RearrangeSimulationInterface as RSI
    from robogym.utils.rotation import quat_from_angle_and_axis

    table_pos, table_size = np.array(TABLE[:3]), np.array(TABLE[3:])
    ref_table = RSI.compute_table_dimension(table_pos.copy(), table_size.copy())

    class MjSim:
        """the model and data arrays get_block_bounding_box and set_target_quat read: one box geom per target body"""

        def __init__(self, bbox):
            n = len(bbox)
            self.names = [f"target:object{i}" for i in range(n)]
            self.model = SimpleNamespace(body_quat=np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)), geom_pos=np.array(bbox[:, 0]), geom_size=np.array(bbox[:, 1]),
                                         body_geomadr=np.arange(n), body_geomnum=np.ones(n, dtype=int), body_name2id=self.names.index)
            self.data = SimpleNamespace(get_body_xmat=lambda name: mj_body_xmat(self.model.body_quat[self.names.index(name)]))

    class Sim:
        """what the layout goal generators read and write of a rearrange simulation"""
        get_table_setting = RSI.get_table_setting
        set_target_quat = RSI.set_target_quat

        def __init__(self, bbox, portion, area=None, **params):
            self.bbox, self.num_objects, self.used_table_portion = bbox, len(bbox), portion
            self.area = area
            self.simulation_params = SimpleNamespace(**params)
            self.mj_sim = MjSim(bbox)

        def forward(self):
            pass                                   # get_body_xmat derives xmat from body_quat when it is read

        def get_object_bounding_boxes(self):
            return self.bbox.copy()

        def get_target_bounding_boxes(self):
            return np.array([get_block_bounding_box(self.mj_sim, f"target:object{i}") for i in range(self.num_objects)])

        def get_table_dimensions(self):
            return ref_table

        def get_placement_area(self):
            return RSI.get_placement_area(self) if self.area is None else self.area

        def target_quat(self):
            return self.mj_sim.model.body_quat.copy()

    def generator(cls, sim, **attrs):
        g = object.__new__(cls)
        g.mujoco_simulation = sim
        for k, v in attrs.items():
            setattr(g, k, v)
        return g

    rng = np.random.RandomState(20261018)
    cases = []

    def case(kind, bbox, active, portion, area=None, **kw):
        bbox, active = np.asarray(bbox, dtype=np.float64), np.asarray(active, dtype=bool)
        sel = np.nonzero(active)[0]
        nobj = len(bbox)
        seed, env, epoch = int(rng.randint(1 << 31)), int(rng.randint(4096)), int(rng.randint(64))
        rs = LayoutReplayRandomState(seed, env, epoch)
        ar = None if area is None else PlacementArea(offset=tuple(area[:3]), size=tuple(area[3:]))
        angles, retry = None, None
        if kind == "domino":
            sim = Sim(bbox[sel], portion, ar, object_size=kw["object_size"], domino_distance_mul=kw["distance_mul"])
            g = generator(DominoStateGoal, sim)
            tried = []
            g._set_target_quat = lambda n, a: (tried.append(np.array(a)), DominoStateGoal._set_target_quat(g, n, a))
            pl, ok = DominoStateGoal._sample_next_goal_positions(g, rs)
            angles = tried[-1]
            retry = (rs.modifier_draws - 4) // 2 if ok else -1
            assert rs.modifier_draws == (2 * retry + 4 if ok else 2 * dominos.MAX_RETRY) and len(tried) == (retry + 1 if ok else dominos.MAX_RETRY)
        elif kind == "attached":
            sim = Sim(bbox[sel], portion, ar, object_size=kw["object_size"])
            pl, ok = AttachedBlockStateGoal._sample_next_goal_positions(generator(AttachedBlockStateGoal, sim), rs)
            assert rs.modifier_draws == 9
        else:
            sim = Sim(bbox[sel], portion, ar)
            g = generator(ObjectFixedStateGoal, sim, relative_placements=np.asarray(kw["rel"], dtype=np.float64)[sel],
                          init_quats=np.asarray(kw["init_quat"], dtype=np.float64)[sel])
            pl, ok = ObjectFixedStateGoal._sample_next_goal_positions(g, rs)
            assert rs.modifier_draws == 0
        pos, quat, ang = np.zeros((nobj, 3)), np.tile([1.0, 0.0, 0.0, 0.0], (nobj, 1)), np.zeros(nobj)
        pos[sel], quat[sel] = pl, sim.target_quat()
        if angles is not None:
            ang[sel] = angles
        area = sim.get_placement_area()
        c = dict(kind=kind, bbox=bbox.tolist(), active=active.astype(int).tolist(), area=list(area.offset) + list(area.size), seed=seed, env=env,
                 epoch=epoch, object_size=kw.get("object_size", 0.0), distance_mul=kw.get("distance_mul", 0.0), status=int(bool(ok)),
                 pos=pos.tolist(), quat=quat.tolist(), angle=ang.tolist(), retry=retry, draws=rs.modifier_draws,
                 rel=None if kind != "fixed" else np.asarray(kw["rel"], dtype=np.float64).tolist(),
                 init_quat=None if kind != "fixed" else np.asarray(kw["init_quat"], dtype=np.float64).tolist())
        cases.append(c)
        return c

    def domino_boxes(nobj, size, ecc):
        return np.array([[np.zeros(3), size * np.array([1.0 / ecc, 1.0, ecc])]] * nobj)

    # dominoes: 1, 2, 5 and 8 of 8 slots, every eccentricity and distance multiplier of the randomisable range's ends and default
    for n in (1, 2, 5, 8):
        for ecc in (1.0, 1.5, 4.5):
            for mul in (2.0, 5.0):
                active = np.zeros(8, dtype=bool)
                active[np.sort(rng.choice(8, n, replace=False)) if n in (2, 5) else np.arange(n)] = True
                case("domino", domino_boxes(8, 0.0254, ecc), active, float(rng.choice([1.0, 0.9])), object_size=0.0254, distance_mul=mul)
    # per-case sizes, off-centre boxes
    for k in range(6):
        n = int(rng.randint(1, 9))
        bb = domino_boxes(8, float(rng.uniform(0.015, 0.035)), float(rng.uniform(1.0, 4.5)))
        bb[:, 0] = rng.uniform(-0.005, 0.005, (8, 3))
        case("domino", bb, np.arange(8) < n, 1.0, object_size=float(bb[0, 1, 1]), distance_mul=float(rng.uniform(2.0, 5.0)))
    # tight areas: many retries, and one that never fits within MAX_RETRY
    for k in range(60):                        # the first draw that needs 40 or more retries in a narrowing area
        side = 0.9 - 0.005 * k
        c = case("domino", domino_boxes(8, 0.0254, 4.5), np.ones(8, bool), 1.0, area=[0.3, 0.4, 0.4, side, side * 0.8, 0.26], object_size=0.0254,
                 distance_mul=5.0)
        if c["retry"] >= 40:
            break
        cases.pop()
    assert c["retry"] >= 40, c["retry"]
    case("domino", domino_boxes(8, 0.0254, 1.5), np.ones(8, bool), 1.0, area=[0.5, 0.5, 0.4, 0.12, 0.1, 0.26], object_size=0.0254, distance_mul=4.0)

    # attached blocks: two block sizes, two areas (used_table_portion 0.8 -- the clip for 8 objects -- and 1.0), padded slots
    for size in (0.0254, 0.04):
        for portion in (0.8, 1.0):
            for nobj in (8, 10):
                active = np.zeros(nobj, dtype=bool)
                active[np.sort(rng.choice(nobj, 8, replace=False))] = True
                bb = np.array([[np.zeros(3), np.full(3, size)]] * nobj)
                case("attached", bb, active, portion, object_size=size)

    # fixed layouts: table_setting (the library's mesh boxes, the spoon turned), wordblocks, and placements beyond the area
    meshes = [np.array(b["bbox"]) for b in json.loads(gzip.decompress(open(PLACEMENT, "rb").read()))["boxes"] if b["kind"] == "mesh"]
    mesh_boxes = np.concatenate(meshes)[:5]
    ident = [1.0, 0.0, 0.0, 0.0]
    spoon = quat_from_angle_and_axis(0.38, np.array([0, 0, 1.0]))
    case("fixed", mesh_boxes, np.ones(5, bool), 1.0, rel=[[0.6, 0.5], [0.6, 0.68], [0.6, 0.75], [0.6, 0.36], [0.6, 0.28]],
         init_quat=[ident] * 4 + [spoon.tolist()])
    words = [[0.5, 0.05], [0.5, 0.2], [0.5, 0.35], [0.5, 0.65], [0.5, 0.8], [0.5, 0.95]]
    case("fixed", np.array([[np.zeros(3), np.full(3, 0.0254)]] * 6), np.ones(6, bool), 1.0, rel=words, init_quat=[ident] * 6)
    case("fixed", np.array([[np.zeros(3), np.full(3, 0.0254)]] * 8), np.arange(8) % 4 != 1, 0.7, rel=words + [[0.1, 0.1], [0.9, 0.9]],
         init_quat=[ident] * 8)
    beyond = rng.uniform(-0.5, 1.5, (6, 2))
    beyond[0] = [-0.3, 1.2]
    bb = np.stack([rng.uniform(-0.01, 0.01, (6, 3)), rng.uniform(0.01, 0.05, (6, 3))], 1)
    case("fixed", bb, np.ones(6, bool), 1.0, rel=beyond, init_quat=[ident] * 6)

    doc = dict(table=TABLE, max_retry=dominos.MAX_RETRY, cases=cases,
               source="robogym v1.0.0 goals/dominos.py, goals/attached_block_state.py, goals/object_state_fixed.py, common/utils.py "
                      "place_targets_with_fixed_position / get_block_bounding_box; replay RandomState of tests/layout_goals_rng.py")
    with open(OUT, "wb") as f:
        f.write(gzip.compress(json.dumps(doc).encode(), mtime=0))
    kinds = {}
    for c in cases:
        kinds[c["kind"]] = kinds.get(c["kind"], 0) + 1
    dom = [c for c in cases if c["kind"] == "domino"]
    print(f"{OUT}: {len(cases)} cases {kinds}; domino retries {sorted(c['retry'] for c in dom)}")


if __name__ == "__main__":
    main()
