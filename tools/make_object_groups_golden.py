"""Record the reference's object groups, group attributes and initial yaws into tests/golden/reference_object_groups.json.gz.

Needs a checkout of openai/robogym v1.0.0: `ROBOGYM_REFERENCE=<checkout> python tools/make_object_groups_golden.py`.  It imports
the reference on the mujoco_py shim (as tools/make_layout_goals_golden.py does) and runs the reference's OWN methods on
instances of its environment classes made without their constructors, carrying only what the methods read: `_random_state`,
`parameters`, `constants` and `mujoco_simulation.num_objects` (MESH_FILES is the class's own):

- `_sample_random_object_groups`: RearrangeEnv's (sample_group_counts), DuplicateBlockRearrangeEnv's (one group), the
  dedupe_objects=True overrides of WordBlocksEnv, ChessboardRearrangeEnv and TableSettingRearrangeEnv, and
  HoldoutRearrangeEnv's fixed counts;
- `_sample_group_attributes`: RearrangeEnv's (materials, random colours, size scales), BlockRearrangeEnv's palette,
  MeshRearrangeEnv's grey colours and mesh draw, YcbRearrangeEnv's `_sample_object_meshes` with and without replacement and
  with a `mesh_names` subset, and the dedupe environments' fixed tables;
- `_sample_default_quaternions`.

Random numbers come from the replay RandomState of tests/object_groups_rng.py (draw d at the groups' counter (d, 0, 6, epoch),
object j's yaw at (j, 1, 6, epoch)).  The tool also checks on numpy's own legacy RandomState that `choice` over a single
material name consumes no random numbers, which the kernel's one-material case relies on."""
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

OUT = os.path.join(ROOT, "tests", "golden", "reference_object_groups.json.gz")
MATERIALS = ["default", "painted_wood", "rubber-ball", "tangram"]
YCB_SUBSET = ["003_cracker_box", "004_sugar_box", "005_tomato_soup_can", "006_mustard_bottle", "007_tuna_fish_can", "008_pudding_box",
              "009_gelatin_box", "010_potted_meat_can", "011_banana", "013_apple", "019_pitcher_base"]


def one_material_draws_nothing():
    """numpy's legacy choice(names, size) with one name is randint over a one-value range: no random numbers drawn"""
    rs = np.random.RandomState(5)
    before = rs.get_state()[1].copy(), rs.get_state()[2]
    assert list(rs.choice(["default"], size=3)) == ["default"] * 3
    after = rs.get_state()[1], rs.get_state()[2]
    return bool(np.array_equal(before[0], after[0]) and before[1] == after[1])


def main():
    import robogym_b200.mujoco_py_shim as shim
    from object_groups_rng import GroupsReplayRandomState

    shim.install()
    logging.disable(logging.WARNING)
    from robogym.envs.rearrange.blocks import BlockRearrangeEnv, BlockRearrangeEnvParameters
    from robogym.envs.rearrange.blocks_duplicate import DuplicateBlockRearrangeEnv
    from robogym.envs.rearrange.chessboard import ChessboardRearrangeEnv
    from robogym.envs.rearrange.common.base import RearrangeEnvConstants
    from robogym.envs.rearrange.common.mesh import MeshRearrangeEnvConstants, MeshRearrangeEnvParameters
    from robogym.envs.rearrange.common.utils import load_material_args
    from robogym.envs.rearrange.holdout import HoldoutRearrangeEnv
    from robogym.envs.rearrange.table_setting import TableSettingRearrangeEnv
    from robogym.envs.rearrange.wordblocks import WordBlocksEnv, WordBlocksEnvConstants, WordBlocksEnvParameters
    from robogym.envs.rearrange.ycb import YcbRearrangeEnv, YcbRearrangeEnvConstants

    assert one_material_draws_nothing()
    material_args = {m: load_material_args(m) for m in MATERIALS}

    class Replay(GroupsReplayRandomState):
        """keeps the yaws _sample_default_quaternions draws"""

        def uniform(self, low=0.0, high=1.0, size=None):
            v = super().uniform(low, high, size)
            if self.row == 1:
                self.yaw = np.array(v, dtype=np.float64).reshape(-1)
            return v

    def run(kind, cls, params, constants, n, seed, env, epoch, **meta):
        rs = Replay(seed, env, epoch)
        e = object.__new__(cls)
        e._random_state, e.parameters, e.constants = rs, params, constants
        e.mujoco_simulation = SimpleNamespace(num_objects=n)
        groups = e._sample_random_object_groups()
        attrs = e._sample_group_attributes(len(groups))
        draws = rs.draws[0]
        rs.yaws()
        quat = e._sample_default_quaternions()
        counts = [int(g.count) for g in groups]
        ids = [list(map(int, g.object_ids)) for g in groups]
        assert sum(counts) == n and [i for r in ids for i in r] == list(range(n)), (kind, counts, ids)
        case = dict(kind=kind, n=n, seed=seed, env=env, epoch=epoch, counts=counts, draws=draws, yaw=rs.yaw.tolist(), quat=np.asarray(quat).tolist(),
                    material=None, color=None, scale=None, mesh=None, **meta)
        if "material_args" in attrs:
            names = meta["material_names"]
            case["material"] = [next(i for i, m in enumerate(names) if material_args[m] == a) for a in attrs["material_args"]]
        if "color" in attrs:
            case["color"] = np.asarray(attrs["color"], dtype=np.float64).tolist()
        if "scale" in attrs:
            case["scale"] = np.asarray(attrs["scale"], dtype=np.float64).tolist()
        if meta.get("candidates") is not None:                 # (chessboard's and table_setting's meshes are fixed)
            case["mesh"] = [meta["candidates"].index(f) for f in attrs["mesh_files"]]
        case.pop("candidates", None)
        return case

    def ycb_candidates(mesh_names):
        files = YcbRearrangeEnv.MESH_FILES
        cand = [f for d, f in files.items() if mesh_names is None or d in mesh_names]
        return sorted(cand)

    rng = np.random.RandomState(2024)
    cases = []
    env_id = iter(range(10 ** 6))

    def ids():
        return int(rng.randint(1 << 31)), next(env_id) % 40, int(rng.randint(1 << 16))

    # blocks: 1..8 objects at the default lambda range and two others; one and several materials; scales
    for lam in ((0.1, 5.0), (0.5, 1.0), (2.0, 8.0)):
        for n in range(1, 9):
            for mats in (["default"], MATERIALS):
                for sc in ((0.0, 0.0), (0.3, 0.5)) if lam == (0.1, 5.0) else ((0.0, 0.0),):
                    p = BlockRearrangeEnvParameters()
                    p.simulation_params.num_objects = n
                    p.material_names = list(mats)
                    p.object_scale_low, p.object_scale_high = sc
                    c = RearrangeEnvConstants(sample_lam_low=lam[0], sample_lam_high=lam[1])
                    seed, env, epoch = ids()
                    cases.append(run("blocks", BlockRearrangeEnv, p, c, n, seed, env, epoch, lam=list(lam), material_names=list(mats), scale_range=list(sc),
                                     group_mode="random", color_mode="palette"))
    # blocks_duplicate: the random counts drawn, one group
    for n in range(1, 9):
        p = BlockRearrangeEnvParameters()
        p.simulation_params.num_objects = n
        p.material_names = ["default"]
        seed, env, epoch = ids()
        cases.append(run("blocks_duplicate", DuplicateBlockRearrangeEnv, p, RearrangeEnvConstants(), n, seed, env, epoch, lam=[0.1, 5.0],
                         material_names=["default"], scale_range=[0.0, 0.0], group_mode="single", color_mode="palette"))
    # the dedupe environments (their colour tables, and table_setting's scales and meshes, are fixed: no draws)
    for mats in (["default"], MATERIALS):
        p = WordBlocksEnvParameters()
        p.simulation_params.num_objects = 6
        p.material_names = list(mats)
        seed, env, epoch = ids()
        cases.append(run("wordblocks", WordBlocksEnv, p, WordBlocksEnvConstants(), 6, seed, env, epoch, lam=[0.1, 5.0], material_names=list(mats),
                         scale_range=[0.0, 0.0], group_mode="dedupe", color_mode="fixed"))
        for cls, n in ((ChessboardRearrangeEnv, 4), (TableSettingRearrangeEnv, 5)):
            p = MeshRearrangeEnvParameters()
            p.simulation_params.num_objects = n
            p.material_names = list(mats)
            p.object_scale_low, p.object_scale_high = 0.2, 0.3
            seed, env, epoch = ids()
            kind = "chessboard" if cls is ChessboardRearrangeEnv else "table_setting"
            cases.append(run(kind, cls, p, MeshRearrangeEnvConstants(), n, seed, env, epoch, lam=[0.1, 5.0], material_names=list(mats),
                             scale_range=[0.2, 0.3], group_mode="dedupe", color_mode="fixed"))
    # holdout: the task's fixed counts, no attributes
    for counts in ([1], [2, 1, 3], [1, 1, 1, 1], [4, 4], [3]):
        n = sum(counts)
        p = SimpleNamespace(simulation_params=SimpleNamespace(num_objects=n, task_object_configs=[SimpleNamespace(count=c) for c in counts]))
        seed, env, epoch = ids()
        cases.append(run("holdout", HoldoutRearrangeEnv, p, RearrangeEnvConstants(), n, seed, env, epoch, fixed_counts=list(counts), group_mode="fixed",
                         color_mode="none"))
    # ycb: with and without replacement, a mesh_names subset, grey colours, one and several materials
    for replace in (True, False):
        for mesh_names in (None, YCB_SUBSET):
            for grey in (False, True):
                for n in (1, 3, 5, 8):
                    mats = MATERIALS if n == 5 else ["default"]
                    p = MeshRearrangeEnvParameters(mesh_names=None if mesh_names is None else list(mesh_names))
                    p.simulation_params.num_objects = n
                    p.material_names = list(mats)
                    p.object_scale_low, p.object_scale_high = 0.5, 0.5
                    c = YcbRearrangeEnvConstants(sample_with_replacement=replace, use_grey_colors=grey)
                    cand = ycb_candidates(mesh_names)
                    seed, env, epoch = ids()
                    cases.append(run("ycb", YcbRearrangeEnv, p, c, n, seed, env, epoch, lam=[0.1, 5.0], material_names=list(mats), scale_range=[0.5, 0.5],
                                     group_mode="random", color_mode="grey" if grey else "random", n_candidates=len(cand), replace=replace,
                                     mesh_names=mesh_names, candidates=cand))
    out = dict(cases=cases, palette=np.asarray(BlockRearrangeEnv.OBJECT_COLORS, dtype=np.float64).tolist(), one_material_draws_nothing=True)
    open(OUT, "wb").write(gzip.compress(json.dumps(out).encode(), mtime=0))
    kinds = {}
    for c in cases:
        kinds[c["kind"]] = kinds.get(c["kind"], 0) + 1
    print(OUT, len(cases), "cases", kinds)


if __name__ == "__main__":
    main()
