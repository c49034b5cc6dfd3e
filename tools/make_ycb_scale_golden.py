"""Record what the reference builds for scaled YCB objects into tests/golden/reference_ycb_scale.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_ycb_scale_golden.py`.  For a few objects
of the committed rearrange_ycb8 scene and a few scales s, the reference's own `make_mesh_object(name, files, s)`
(robogym/envs/rearrange/common/utils.py:250-281, the document MeshRearrangeSim.make_objects_xml writes for every object) is
composed with the reference's MujocoXML, given the scene's default material (as tools/compose_reference_xml.py does for
rearrange_ycb8) and compiled by robogym_b200.mjcf from the reference's STL files.  Recorded per object and scale: the part geom
rows and the body rows of the compiled object, a digest of every scaled hull (vertex count, mean, per-axis min / max, mean
squared norm), and the extents of the combined raw mesh (numpy over the STL triangles, what trimesh's `extents` measures).
tests/test_object_scale.py checks compact_model, BatchedMeshScene and ObjectLibrary against these numbers."""
import glob
import gzip
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
import compose_reference_xml as ref  # noqa: E402

for p in (os.path.join(ROOT, "tests", "stubs"), ref.REF, ROOT):   # tests/stubs: trimesh (center_mass of the combined mesh)
    if p not in sys.path:
        sys.path.insert(0, p)

OUT = os.path.join(ROOT, "tests", "golden", "reference_ycb_scale.json.gz")
# slot of the committed rearrange_ycb8 scene (tools/compose_reference_xml.py: YCB_SCENE) -> directory; 025_mug has 29 parts
OBJECTS = ((0, "003_cracker_box"), (1, "011_banana"), (2, "025_mug"))
SCALES = (0.7, 1.0, 1.45)
GEOM_FIELDS = ("geom_pos", "geom_quat", "geom_size", "geom_rbound", "geom_aabb")
BODY_FIELDS = ("body_mass", "body_inertia", "body_ipos", "body_iquat")


def hull_digest(v):
    v = np.asarray(v, dtype=np.float64).reshape(-1, 3)
    return dict(n=len(v), mean=v.mean(0).tolist(), lo=v.min(0).tolist(), hi=v.max(0).tolist(), r2=float((v * v).sum(1).mean()))


def compile_object(files, s):
    X = ref.mujoco_xml_cls()         # installs the mujoco_py stub the reference's modules import
    from robogym.envs.rearrange.common.utils import make_mesh_object

    from robogym_b200 import mjcf

    xml = X().add_default_compiler_directive()
    obj = make_mesh_object("object0", files, s)
    obj.set_objects_attrs(dict(geom=dict(condim="6", margin=0.00005), joint=dict(damping="0.01", armature="0.001")))
    xml.append(obj)
    cm = mjcf.compile_mjcf(xml.xml_string())
    return cm.m, cm.names


def main():
    import trimesh

    stl_root = os.path.join(ref.REF, "robogym", "assets", "stls")
    rec = dict(scales=list(SCALES), objects=[])
    for slot, d in OBJECTS:
        files = sorted(glob.glob(os.path.join(stl_root, "ycb", d, "*.stl")))
        raw = np.concatenate([trimesh.load(f).vertices for f in files])
        o = dict(slot=slot, name=d, nparts=len(files), extents=(raw.max(0) - raw.min(0)).tolist(), runs=[])
        for s in SCALES:
            m, names = compile_object(files, s)
            b = names["body"].index("object0")
            geoms = np.nonzero(np.asarray(m["geom_bodyid"]) == b)[0]
            run = dict(s=s)
            for f in GEOM_FIELDS:
                run[f] = np.asarray(m[f]).reshape(m["ngeom"], -1)[geoms].tolist()
            for f in BODY_FIELDS:
                run[f] = np.asarray(m[f]).reshape(m["nbody"], -1)[b].tolist()
            hulls = []
            for g in geoms:
                mid = int(m["geom_dataid"][g])
                va, nv = int(m["mesh_vertadr"][mid]), int(m["mesh_vertnum"][mid])
                hulls.append(hull_digest(np.asarray(m["mesh_vert"]).reshape(-1, 3)[va:va + nv]))
            run["hulls"] = hulls
            o["runs"].append(run)
            print(f"{d} s={s}: {len(geoms)} parts, mass {run['body_mass'][0]:.6g}")
        rec["objects"].append(o)
    with open(OUT, "wb") as f:      # mtime=0: the same record gives the same bytes
        f.write(gzip.compress(json.dumps(rec, separators=(",", ":")).encode(), compresslevel=9, mtime=0))
    print(OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()
