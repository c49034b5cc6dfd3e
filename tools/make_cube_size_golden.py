"""Record what the reference's full-cube size modifier does to the model into tests/golden/reference_cube_size.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_cube_size_golden.py`.  The unmodified
`PerpendicularCubeSizeModifier` (robogym/envs/dactyl/common/mujoco_modifiers.py:8-66, the modifier behind
`RandomizedPerpendicularCubeSizeWrapper`) runs on the mujoco_py shim, on the committed dactyl_full_perpendicular model with the fp64
oracle as engine.  For every multiplier s it records which body_pos rows, geom_rbound entries and mesh_vert rows differ from the
original model afterwards, and their values; tests/test_mesh_scale.py replays that against FullCubeRandomizer(cube_size_range=...)."""
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
REF = os.environ["ROBOGYM_REFERENCE"]
for p in (os.path.join(ROOT, "tests", "stubs"), os.path.join(ROOT, "tests"), REF, ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_cube_size.json.gz")
MULTIPLIERS = (0.95, 1.0, 1.05)


def _changed_rows(a, b):
    return [int(i) for i in np.nonzero(np.any(np.asarray(a).reshape(len(b), -1) != np.asarray(b).reshape(len(b), -1), axis=1))[0]]


def main():
    import robogym_b200.mujoco_py_shim as shim

    shim.install()
    from oracle_engine import OracleEngine

    shim.set_engine_factory(OracleEngine)
    from robogym.envs.dactyl.common.mujoco_modifiers import PerpendicularCubeSizeModifier

    from robogym_b200 import mjcf, modelblob

    blob = open(os.path.join(ROOT, "robogym_b200", "assets", "dactyl_full_perpendicular.rgm"), "rb").read()
    sim = shim.MjSim(shim.PyMjModel(mjcf.CompiledModel.from_blob(blob, modelblob.unpack_names(blob))))
    model = sim.model
    bp0, rb0, mv0 = model.body_pos.copy(), model.geom_rbound.copy(), model.mesh_vert.copy()
    mod = PerpendicularCubeSizeModifier("cube:")
    mod.initialize(sim)
    rec = dict(multipliers=list(MULTIPLIERS), runs=[])
    for s in MULTIPLIERS:
        mod(s)
        bodies = _changed_rows(model.body_pos, bp0)
        geoms = _changed_rows(model.geom_rbound, rb0)
        verts = _changed_rows(model.mesh_vert, mv0)
        rec["runs"].append(dict(
            s=s,
            bodies=bodies, body_pos=np.asarray(model.body_pos)[bodies].ravel().tolist(),
            geoms=geoms, geom_rbound=np.asarray(model.geom_rbound)[geoms].ravel().tolist(),
            mesh_vert_rows=[min(verts), max(verts) + 1] if verts else [], n_mesh_vert_rows=len(verts),
            mesh_vert=np.asarray(model.mesh_vert)[verts].ravel().tolist()))
        print("s=%.2f: %d bodies, %d geoms, %d mesh vertices changed" % (s, len(bodies), len(geoms), len(verts)))
    # the modifier edits in place from its saved originals: the last call leaves the model scaled, restore for good measure
    mod(1.0)
    assert np.array_equal(model.body_pos, bp0) and np.array_equal(model.geom_rbound, rb0) and np.array_equal(model.mesh_vert, mv0)
    with open(OUT, "wb") as f:      # mtime=0: the same record gives the same bytes
        f.write(gzip.compress(json.dumps(rec, separators=(",", ":")).encode(), compresslevel=9, mtime=0))
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
