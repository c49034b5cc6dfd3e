"""Record the reference's placement and bounding boxes into tests/golden/reference_placement.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_placement_golden.py`.  It imports the
reference on the mujoco_py shim with the `collision` stand-in of tests/stubs and runs the reference's OWN functions:

- `RearrangeEnv._generate_object_placements` (grid, then the uniform fallback), `place_objects_in_grid`,
  `place_objects_with_no_constraint` and `place_targets_with_goal_distance_ratio`
  (robogym/envs/rearrange/common/{base,utils}.py), with a replay RandomState (tests/placement_rng.py) whose `shuffle` and
  `uniform` draw from the same Philox counters as the placement kernel;
- `RearrangeSimulationInterface.get_placement_area` for 1 to 8 objects at several `used_table_portion` values;
- `get_block_bounding_box` and `get_mesh_bounding_box` on a minimal sim view of compiled models: blocks of rearrange_blocks5 at
  several sizes and yaws, and library objects (compact models of rearrange_ycb8 draws) at several yaws and scales.

The cases: blocks at several sizes and table portions, irregular ycb boxes at random yaws and scales for which the grid has too
few cells and the fallback engages, a crowded case that fails outright, and goal-distance ratios 0, 0.5 and 1 at the default
minimum.  tests/test_placement.py replays every case on the emulated and the CUDA kernels."""
import gzip
import json
import logging
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
REF = os.environ.get("ROBOGYM_REFERENCE", "/root/reference")
for p in (os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests"), REF, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_placement.json.gz")
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
MODES = {"grid": 1, "uniform": 2, "goal_distance_ratio": 3, "grid_then_uniform": 4}


def _yaw_quat(a):
    return np.array([np.cos(0.5 * a), 0.0, 0.0, np.sin(0.5 * a)])


class _SimView:
    """what get_block_bounding_box / get_mesh_bounding_box read of an MjSim: model arrays and one body's rotation"""

    def __init__(self, m, names, quat):
        from robogym.utils.rotation import quat2mat

        class Model:
            pass

        md = Model()
        md.body_name2id = names["body"].index
        for f, w in (("body_geomadr", 0), ("body_geomnum", 0), ("geom_type", 0), ("geom_dataid", 0), ("mesh_vertadr", 0), ("mesh_vertnum", 0),
                     ("mesh_faceadr", 0), ("mesh_facenum", 0), ("geom_pos", 3), ("geom_quat", 4), ("geom_size", 3), ("mesh_vert", 3), ("mesh_face", 3)):
            a = np.asarray(m[f])
            setattr(md, f, a.reshape(-1, w) if w else a)

        class Data:
            pass

        dt = Data()
        dt.get_body_xmat = lambda name: quat2mat(quat)
        self.model, self.data = md, dt


def main():
    import robogym_b200.mujoco_py_shim as shim
    from robogym_b200 import modelblob
    from robogym_b200 import rearrange_mesh_scene as rms
    from robogym_b200 import rearrange_placement as rp
    from placement_rng import ReplayRandomState

    shim.install()
    logging.disable(logging.WARNING)       # the grid logs every failed trial
    import robogym.envs.rearrange.common.base as base
    import robogym.envs.rearrange.common.utils as U
    from robogym.envs.rearrange.simulation.base import RearrangeSimulationInterface as RSI

    blocks = open(os.path.join(ASSETS, "rearrange_blocks5.rgm"), "rb").read()
    table_pos, table_size, table_height = rp.table_dimensions(blocks)
    ref_table = RSI.compute_table_dimension(table_pos.copy(), table_size.copy())
    table = np.concatenate([table_pos, table_size]).tolist()

    class _Sim:
        max_placement_retry, max_placement_retry_per_object = 100, 20

        def __init__(self, bbox, n, portion):
            self.bbox, self.num_objects, self.used_table_portion = bbox, n, portion

        def get_object_bounding_boxes(self):
            return self.bbox.copy()

        def get_table_dimensions(self):
            return ref_table

        get_table_setting = RSI.get_table_setting

        def get_placement_area(self):
            return RSI.get_placement_area(self)

    grid_valid = []
    orig_grid = base.place_objects_in_grid

    def grid_spy(*a, **k):
        out = orig_grid(*a, **k)
        grid_valid.append(bool(out[1]))
        return out

    base.place_objects_in_grid = grid_spy

    def run(mode, bbox, active, portion, seed, env, epoch, anchor=None, ratio=1.0, dmin=0.06):
        bbox, active = np.asarray(bbox, dtype=np.float64), np.asarray(active, dtype=bool)
        sel = np.nonzero(active)[0]
        sim = _Sim(bbox[sel], len(sel), portion)
        area = sim.get_placement_area()
        rs = ReplayRandomState(seed, env, epoch)
        grid_valid.clear()
        if mode == "grid_then_uniform":
            env_ = type("Env", (), {})()
            env_.mujoco_simulation, env_._random_state = sim, rs
            pl, ok = base.RearrangeEnv._generate_object_placements(env_)
            status = (1 if grid_valid[0] else 2) if ok else 0
        elif mode == "grid":
            pl, ok = U.place_objects_in_grid(bbox[sel], ref_table, area, random_state=rs, max_num_trials=100)
            status = 1 if ok else 0
        elif mode == "uniform":
            pl, ok = U.place_objects_with_no_constraint(bbox[sel], ref_table, area, 100, 20, rs)
            status = 2 if ok else 0
        else:
            pl, ok = U.place_targets_with_goal_distance_ratio(bbox[sel], ref_table, area, np.asarray(anchor, dtype=np.float64)[sel], ratio, dmin, 100, 20, rs)
            status = 3 if ok else 0
        pos = np.zeros((len(bbox), 3))
        if ok:
            pos[sel] = pl
        return dict(mode=mode, bbox=bbox.tolist(), active=active.astype(int).tolist(), table=table, area=list(area.offset) + list(area.size), portion=portion,
                    seed=seed, env=env, epoch=epoch, anchor=None if anchor is None else np.asarray(anchor).tolist(), ratio=ratio, dmin=dmin,
                    status=status, pos=pos.tolist())

    rng = np.random.RandomState(20261016)
    cases = []
    # blocks: several sizes, yaws and table portions; some slots inactive (parked blocks)
    for size in (0.0254, 0.04, 0.06):
        for portion in (1.0, 0.6, 0.4):
            for mode in ("grid_then_uniform", "grid", "uniform"):
                n = 5
                yaw = rng.uniform(-np.pi, np.pi, n)
                bbox = np.array([U.rotate_bounding_box((np.zeros(3), np.full(3, size) * rng.uniform(0.8, 1.2)), _yaw_quat(a)) for a in yaw])
                active = rng.rand(n) < 0.8
                active[0] = True
                cases.append(run(mode, bbox, active, portion, int(rng.randint(1 << 31)), int(rng.randint(4096)), int(rng.randint(16))))
    # irregular ycb boxes: random draws, yaws and scales of the library objects (the grid's cells are too few: the fallback engages)
    b8, bt = (open(os.path.join(ASSETS, n + ".rgm"), "rb").read() for n in ("rearrange_ycb8", "rearrange_ycb8_tcp"))
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    boxes = []
    for trial in range(6):
        draw = rng.randint(0, len(lib.entries), 8)
        scale = rng.uniform(0.7, 1.5, 8)
        yaw = rng.uniform(-np.pi, np.pi, 8)
        c = rms.compact_model(b8, lib, draw, scale)
        m, names = modelblob.unpack(c), modelblob.unpack_names(c)
        bb = np.array([U.get_mesh_bounding_box(_SimView(m, names, _yaw_quat(yaw[k])), f"object{k}") for k in range(8)])
        if trial < 2:
            boxes.append(dict(kind="mesh", draw=draw.tolist(), scale=scale.tolist(), yaw=yaw.tolist(), bbox=bb.tolist()))
        for portion in (1.0, 0.8):
            active = np.ones(8, dtype=bool)
            if trial % 2:
                active[rng.randint(8)] = False
            cases.append(run("grid_then_uniform", bb, active, portion, int(rng.randint(1 << 31)), int(rng.randint(4096)), int(rng.randint(16))))
            cases.append(run("uniform", bb, active, portion, int(rng.randint(1 << 31)), int(rng.randint(4096)), int(rng.randint(16))))
    # crowded: eight large blocks in the smallest area fail outright
    big = np.array([[np.zeros(3), np.full(3, 0.1)]] * 8)
    cases.append(run("grid_then_uniform", big, np.ones(8, dtype=bool), 0.4, 7, 3, 0))
    # goals pulled toward their objects: ratios 0, 0.5 and 1 at the default minimum
    for ratio in (0.0, 0.5, 1.0):
        for size in (0.0254, 0.05):
            bbox = np.array([[np.zeros(3), np.full(3, size)]] * 5)
            active = np.ones(5, dtype=bool)
            obj = run("uniform", bbox, active, 1.0, int(rng.randint(1 << 31)), 5, 0)
            assert obj["status"] == 2
            cases.append(run("goal_distance_ratio", bbox, active, 1.0, int(rng.randint(1 << 31)), 5, 1, anchor=obj["pos"], ratio=ratio))
    # placement areas: 1 to 8 objects at several table portions
    areas = []
    for n in range(1, 9):
        for portion in (1.0, 0.8, 0.6, 0.4):
            a = RSI.get_placement_area(_Sim(None, n, portion))
            areas.append(dict(num_objects=n, portion=portion, area=list(a.offset) + list(a.size)))
    # block boxes at several sizes and yaws, on the shim
    mb, nb = modelblob.unpack(blocks), modelblob.unpack_names(blocks)
    for k, yaw in enumerate((0.0, 0.3, -1.2, 2.5, np.pi / 4)):
        boxes.append(dict(kind="block", body=f"object{k % 5}", yaw=yaw,
                          bbox=np.array(U.get_block_bounding_box(_SimView(mb, nb, _yaw_quat(yaw)), f"object{k % 5}")).tolist()))
    doc = dict(table=table, table_height=float(table_height), cases=cases, areas=areas, boxes=boxes,
               source="robogym v1.0.0 common/base.py _generate_object_placements, common/utils.py placement functions and bounding boxes, "
                      "simulation/base.py get_placement_area; replay RandomState of tests/placement_rng.py")
    with open(OUT, "wb") as f:
        f.write(gzip.compress(json.dumps(doc).encode(), mtime=0))
    st = [c["status"] for c in cases]
    print(f"{OUT}: {len(cases)} cases (status counts {np.bincount(st, minlength=4).tolist()}), {len(areas)} areas, {len(boxes)} boxes")


if __name__ == "__main__":
    main()
