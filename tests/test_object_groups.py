"""The object groups of a rearrange reset on the CPU tier (rg_object_groups; robogym_b200/rearrange_groups.py): the reference's
group counts, group attributes and initial yaws, from the kernel's code on its emulation build (tests/emu/rg_emu_groups.cpp).

The fixture tests/golden/reference_object_groups.json.gz holds the reference's own results (tools/make_object_groups_golden.py)
for blocks, blocks_duplicate, the dedupe environments, holdout and ycb, drawn from the same Philox counters as the kernel through
the replay RandomState of tests/object_groups_rng.py.  Counts, group ids, materials, meshes, colours and yaws are compared
exactly; scales and quaternions go through exp / cos / sin, whose last bits differ between libraries, so they are compared
within 1e-15 relative."""
import ctypes
import gzip
import json
import os
import subprocess

import numpy as np
import pytest

import pyemu_groups as pg
from object_groups_rng import GroupsReplayRandomState
from placement_rng import bounded, philox, u53
from robogym_b200 import engine, rearrange_groups as rgr

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_object_groups.json.gz")
NOBJ = 8


@pytest.fixture(scope="module")
def golden():
    return json.loads(gzip.decompress(open(GOLDEN, "rb").read()))


def close(a, b, rel=1e-15):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and bool((np.abs(a - b) <= rel * np.maximum(np.abs(b), 1e-300)).all())


def case_args(c, palette):
    """the rg_object_groups arguments that reproduce a fixture case"""
    kw = dict(lam=c.get("lam", rgr.LAM), n_materials=len(c.get("material_names") or ["default"]), scale_range=c.get("scale_range", (0.0, 0.0)))
    kw["group_mode"] = c["group_mode"]
    kw["color_mode"] = {"palette": "palette", "random": "random"}.get(c["color_mode"], "grey")
    if kw["color_mode"] == "palette":
        kw["palette"] = np.array(palette)
    if c["group_mode"] == "fixed":
        fc = np.zeros(NOBJ, np.int32)
        fc[:len(c["fixed_counts"])] = c["fixed_counts"]
        kw["fixed_counts"] = fc
    if c.get("n_candidates"):
        kw["n_candidates"], kw["replace"] = c["n_candidates"], c["replace"]
    return kw


def per_slot(c, values):
    """a per-group list as one value per object"""
    return [v for v, k in zip(values, c["counts"]) for _ in range(k)]


def emulated_case(c, palette):
    """one fixture case as environment c["env"] of a batch holding it alone there: (outputs, the batch's other rows untouched)"""
    nenv = c["env"] + 1
    kw = case_args(c, palette)
    if "fixed_counts" in kw:
        kw["fixed_counts"] = np.tile(kw["fixed_counts"], (nenv, 1))
    mask = np.zeros(nenv, np.uint8); mask[-1] = 1
    fill = pg.empty_outputs(nenv, NOBJ, np.random.RandomState(c["env"]))
    before = {k: v.copy() for k, v in fill.items()}
    active = np.full(nenv, c["n"])
    out = pg.call(nenv, NOBJ, active, c["seed"], c["epoch"], mask=mask, out=fill, **kw)
    untouched = all(np.array_equal(out[k][:-1], before[k][:-1]) for k in out)
    return {k: v[-1] for k, v in out.items()}, untouched


# ---------------------------------------------------------------------------------------------- CPU
def test_replay_draws_read_their_documented_counters():
    rs = GroupsReplayRandomState(9, 4, 2)
    r = [philox((d, 0, 6, 2), 9, 4) for d in range(12)]
    assert rs.uniform(0.5, 2.0) == 0.5 + 1.5 * u53(r[0][0], r[0][1])
    assert rs.randint(0, 5) == bounded(r[1][0], 4) and rs.randint(3, 4) == 3 and rs.draws[0] == 2      # a one-value range: no draw
    assert np.array_equal(rs.random((1, 2)), [[u53(*r[2][:2]), u53(*r[3][:2])]])
    idx = list(range(4))
    for s in range(3):
        i = 3 - s
        j = bounded(r[4 + s][0], i)
        idx[i], idx[j] = idx[j], idx[i]
    assert np.array_equal(rs.permutation(4), idx) and rs.draws[0] == 7
    p = np.array([0.5, 0.3, 0.2])
    u = u53(*r[7][:2])
    assert rs.choice([1, 2, 3], p=p) == 1 + int(np.searchsorted(np.cumsum(p) / np.cumsum(p)[-1], u, side="right"))
    rs.yaws()
    y = [philox((j, 1, 6, 2), 9, 4) for j in range(3)]
    assert np.array_equal(rs.uniform(0.0, 2 * np.pi, size=3), 2 * np.pi * np.array([u53(*w[:2]) for w in y])) and rs.draws == [8, 3]


def test_emulated_kernel_reproduces_every_reference_case(golden):
    for i, c in enumerate(golden["cases"]):
        got, untouched = emulated_case(c, golden["palette"])
        n, tag = c["n"], (i, c["kind"], c["n"])
        assert untouched, tag
        assert got["ngroups"] == len(c["counts"]), tag
        assert np.array_equal(got["count"][:n], per_slot(c, c["counts"])), (tag, got["count"], c["counts"])
        assert np.array_equal(got["group"][:n], per_slot(c, range(len(c["counts"])))), tag
        assert (got["group"][n:] == -1).all() and (got["count"][n:] == 0).all() and (got["material"][n:] == -1).all() and (got["mesh"][n:] == -1).all()
        assert not got["rgba"][n:].any() and not got["scale"][n:].any() and not got["yaw"][n:].any() and not got["quat"][n:].any()
        assert np.array_equal(got["yaw"][:n], c["yaw"]), tag
        assert close(got["quat"][:n], c["quat"]), (tag, np.abs(got["quat"][:n] - np.array(c["quat"])).max())
        if c["material"] is not None:
            assert np.array_equal(got["material"][:n], per_slot(c, c["material"])), tag
        if c["color"] is not None and c["color_mode"] in ("palette", "random", "grey"):
            assert np.array_equal(got["rgba"][:n], per_slot(c, c["color"])), tag
        if c["scale"] is not None and c["kind"] != "table_setting":       # (table_setting's scales are a fixed table)
            assert close(got["scale"][:n], per_slot(c, c["scale"])), (tag, got["scale"][:n], c["scale"])
        if c["mesh"] is not None:
            assert np.array_equal(got["mesh"][:n], per_slot(c, c["mesh"])), tag
        else:
            assert (got["mesh"] == -1).all()


def test_fixture_covers_the_requested_cases(golden):
    cases, kinds = golden["cases"], {c["kind"] for c in golden["cases"]}
    assert {"blocks", "blocks_duplicate", "wordblocks", "chessboard", "table_setting", "holdout", "ycb"} <= kinds
    blocks = [c for c in cases if c["kind"] == "blocks"]
    assert {c["n"] for c in blocks} == set(range(1, 9)) and len({tuple(c["lam"]) for c in blocks}) == 3
    assert any(c["scale_range"] != [0.0, 0.0] for c in blocks) and {len(c["material_names"]) for c in blocks} == {1, 4}
    assert any(len(c["counts"]) > 1 and max(c["counts"]) > 1 for c in blocks)                     # duplicates drawn
    ycb = [c for c in cases if c["kind"] == "ycb"]
    assert {c["replace"] for c in ycb} == {True, False} and {c["color_mode"] for c in ycb} == {"grey", "random"}
    assert {c["mesh_names"] is None for c in ycb} == {True, False} and {c["n_candidates"] for c in ycb} == {79, 11}
    assert any(len(set(c["mesh"])) < len(c["mesh"]) for c in ycb if c["replace"])               # a repeated mesh with replacement
    assert all(len(set(c["mesh"])) == len(c["mesh"]) for c in ycb if not c["replace"])
    assert any(len(c["material_names"]) > 1 and len(set(c["material"])) > 1 for c in cases if c["material"])
    assert golden["one_material_draws_nothing"]


def _batch(seed, nenv=300, nobj=NOBJ):
    rng = np.random.RandomState(seed)
    active = rng.randint(0, nobj + 1, nenv)
    fixed = np.zeros((nenv, nobj), np.int32)
    for e in range(nenv):
        left, k = active[e], 0
        while left:
            fixed[e, k] = rng.randint(1, left + 1); left -= fixed[e, k]; k += 1
    return rng, active, fixed


MODES = [dict(group_mode="random", color_mode="palette", palette=np.array(rgr.BLOCK_COLORS, float), n_materials=3, scale_range=(0.2, 0.4)),
         dict(group_mode="dedupe", color_mode="grey"),
         dict(group_mode="single", color_mode="random", lam=(0.5, 1.0)),
         dict(group_mode="fixed", color_mode="random", n_materials=2),
         dict(group_mode="random", color_mode="random", scale_range=(0.5, 0.5), n_candidates=79, replace=True),
         dict(group_mode="random", color_mode="grey", n_candidates=11, replace=False, n_materials=4)]


@pytest.mark.parametrize("mode", range(len(MODES)))
def test_emulated_masked_calls_equal_full_ones(mode):
    rng, active, fixed = _batch(3 + mode)
    nenv = len(active)
    kw = dict(MODES[mode])
    if kw["group_mode"] == "fixed":
        kw["fixed_counts"] = fixed
    if kw.get("replace") is False:
        active = np.minimum(active, kw["n_candidates"])
    full = pg.call(nenv, NOBJ, active, 41, 7, **kw)
    mask = rng.rand(nenv) < 0.3
    fill = pg.empty_outputs(nenv, NOBJ, rng)
    before = {k: v.copy() for k, v in fill.items()}
    part = pg.call(nenv, NOBJ, active, 41, 7, mask=mask, out=fill, **kw)
    for k in full:
        assert np.array_equal(part[k][mask], full[k][mask]), k
        assert np.array_equal(part[k][~mask], before[k][~mask]), k
    assert (full["ngroups"] <= active).all() and ((full["ngroups"] > 0) == (active > 0)).all()
    if kw["group_mode"] == "random":
        assert (full["ngroups"] < active).any() and (full["ngroups"][active > 1] > 1).any()


def test_the_yaws_do_not_depend_on_the_group_draws():
    rng, active, fixed = _batch(8)
    a = pg.call(len(active), NOBJ, active, 5, 1, group_mode="random", color_mode="random", n_materials=5)
    b = pg.call(len(active), NOBJ, active, 5, 1, group_mode="dedupe", color_mode="grey")
    assert np.array_equal(a["yaw"], b["yaw"]) and np.array_equal(a["quat"], b["quat"])
    assert not np.array_equal(a["material"], b["material"])


def test_the_abi_refuses_bad_inputs():
    n = np.array([3, 5])
    good = dict(group_mode="random", color_mode="random")
    pg.call(2, 8, n, 0, 0, **good)
    refused = [(dict(nobj=65), "at most 64"),
               (dict(active=np.array([3, 9])), "active counts"), (dict(active=np.array([-1, 2])), "active counts"),
               (dict(lam=(0.1, float("inf"))), "lam"), (dict(lam=(float("nan"), 1.0)), "lam"),
               (dict(scale_range=(float("nan"), 0.0)), "scale"), (dict(scale_range=(0.0, float("inf"))), "scale"),
               (dict(n_materials=0), "n_materials"),
               (dict(color_mode="palette", palette=np.ones((4, 4))), "fewer rows"),
               (dict(n_candidates=0, mesh_mode=1), "candidate"),
               (dict(n_candidates=4, replace=False), "more groups than candidates"),
               (dict(mask=np.ones(3, np.uint8), mask_len=3), "mask"),
               (dict(group_mode="fixed", fixed_counts=np.array([[1, 2, 0, 0, 0, 0, 0, 0], [5, 0, 1, 0, 0, 0, 0, 0]])), "fixed_counts"),
               (dict(group_mode="fixed", fixed_counts=np.array([[1, 1, 0, 0, 0, 0, 0, 0], [5, 0, 0, 0, 0, 0, 0, 0]])), "fixed_counts"),
               (dict(group_mode="fixed", fixed_counts=np.array([[1, 2**31 - 1, 2**31 - 1, 4, 0, 0, 0, 0], [5, 0, 0, 0, 0, 0, 0, 0]])), "fixed_counts"),
               (dict(group_mode="fixed", fixed_counts=np.array([[2, 2, 0, 0, 0, 0, 0, 0], [5, 0, 0, 0, 0, 0, 0, 0]])), "fixed_counts"),
               (dict(group_mode="other"), None)]
    for kw, msg in refused:
        args = dict(good)
        args.update(kw)
        nobj = args.pop("nobj", 8)
        act = args.pop("active", n)
        if msg is None:
            with pytest.raises(KeyError):
                pg.call(2, nobj, act, 0, 0, **args)
            continue
        with pytest.raises(ValueError, match=msg):
            pg.call(2, nobj, act, 0, 0, **args)
    # single: one group whatever the count, so four candidates serve five objects without replacement
    pg.call(2, 8, n, 0, 0, group_mode="single", color_mode="grey", n_candidates=1, replace=False)
    pg.call(2, 8, n, 0, 0, color_mode="palette", palette=np.ones((5, 4)))


def test_the_python_layer_refuses_before_any_launch():
    for kw, msg in ((dict(active=np.array([[1, 0, 1]])), "leading slots"), (dict(active=np.array([2, 3])), "nobj"),
                    (dict(active=np.array([2, 3]), nobj=8, group_mode="fixed"), "fixed_counts"),
                    (dict(active=np.array([2, 3]), nobj=8, color_mode="palette"), "palette"),
                    (dict(active=np.array([2, 3]), nobj=8, color_mode="palette", palette=np.ones((8, 3))), "rgba"),
                    (dict(active=np.array([2, 3]), nobj=8, group_mode="fixed", fixed_counts=np.array([1, 2**31 - 1, 2**31 - 1, 4, 0, 0, 0, 0])),
                     "fixed_counts"),
                    (dict(active=np.array([2, 3]), nobj=70), "at most 64"), (dict(active=np.array([2, 3]), nobj=8, group_mode="x"), "group_mode")):
        a = kw.pop("active")
        with pytest.raises(ValueError, match=msg):
            rgr.object_groups(a, 0, 0, **kw)


def test_struct_mirrors_match_the_header(tmp_path):
    """sizeof / offsetof of rg_groups_in and rg_groups_out from the host compiler equal the ctypes mirrors'"""
    lines, expect = [], {}
    for cname, mirror in (("rg_groups_in", engine.GroupsIn), ("rg_groups_out", engine.GroupsOut)):
        lines.append(f'printf("sizeof {cname} %zu\\n", sizeof({cname}));')
        expect[f"sizeof {cname}"] = ctypes.sizeof(mirror)
        for f, _ in mirror._fields_:
            lines.append(f'printf("offsetof {cname}.{f} %zu\\n", offsetof({cname}, {f}));')
            expect[f"offsetof {cname}.{f}"] = getattr(mirror, f).offset
    src = tmp_path / "mirror.c"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "robogym_b200.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    exe = tmp_path / "mirror"
    subprocess.check_call([os.environ.get("CC", "cc"), "-std=c11", "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)])
    got = dict(line.rsplit(" ", 1) for line in subprocess.check_output([str(exe)]).decode().splitlines())
    assert {k: int(v) for k, v in got.items()} == expect


def test_hand_offs_to_the_reset_stages():
    """the helpers' conventions on the emulation's outputs: identity rotations, unit scales and empty draws past the objects"""
    import torch

    active = np.array([0, 3, 8, 5])
    out = pg.call(4, NOBJ, active, 3, 1, n_candidates=9, replace=False)
    g = rgr.ObjectGroups(**{k: torch.as_tensor(v) for k, v in out.items()})
    slot = np.arange(NOBJ)[None] < active[:, None]
    assert np.array_equal(rgr.active(g).numpy(), slot) and rgr.goal_groups(g) is g.group
    assert np.array_equal(rgr.block_scale(g).numpy(), np.where(slot, out["scale"], 1.0))
    cand = [10, 11, 12, 13, 14, 15, 16, 17, 18]
    assert np.array_equal(rgr.mesh_draw(g, cand).numpy(), np.where(slot, np.array(cand)[np.maximum(out["mesh"], 0)], -1))
    q = rgr.initial_quat(g).numpy()
    assert np.array_equal(q[slot], out["quat"][slot]) and np.array_equal(q[~slot], np.tile([1.0, 0.0, 0.0, 0.0], ((~slot).sum(), 1)))
