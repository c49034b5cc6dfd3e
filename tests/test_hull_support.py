"""Hull support mapping through per-cell candidate lists (robogym_b200/csrc/rg_host.h: rg_host_hull_cells; rg_col.inl:
rg_hull_scan).  The narrow phase scans only the vertices listed for the query direction's cube-map cell; it must return the
vertex a scan of the whole hull returns, bit for bit (lowest vertex id among the fp32 maxima).  Checked in the emulation build
on every hull of every committed asset, group-shared (RG_GRP lanes, as in rg_mpr_batch) and one-lane (rg_support), for random
directions, the hulls' face normals, axis and diagonal directions, and directions on the cells' edges and corners; and a
mesh_vert edit must leave the lists, and the emulated step, exactly as a model loaded with the edited hulls has them."""
import ctypes
import glob
import hashlib
import os
import subprocess

import numpy as np
import pytest

import pyemu
from robogym_b200 import modelblob

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
ASSETS = sorted(glob.glob(os.path.join(ROOT, "robogym_b200", "assets", "*.rgm")))
_lib = None


def lib():
    global _lib
    if _lib is None:
        here = os.path.join(ROOT, "tests", "emu_support")
        subprocess.check_call(["make", "-C", here, "-s"])
        L = ctypes.CDLL(os.path.join(here, "_build", "librg_emu_support.so"))
        L.rge_support_table.restype = ctypes.c_void_p
        L.rge_support_table.argtypes = [ctypes.c_void_p]
        L.rge_support_entries.restype = ctypes.c_void_p
        L.rge_support_entries.argtypes = [ctypes.c_void_p, ctypes.POINTER(ctypes.c_int)]
        L.rge_support_cell.argtypes = [ctypes.c_void_p]
        L.rge_support_scan.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
        L.rge_support_set_vert.argtypes = [ctypes.c_void_p, ctypes.c_void_p]
        L.rge_support_build_seconds.restype = ctypes.c_double
        L.rge_support_build_seconds.argtypes = [ctypes.c_void_p]
        _lib = L
    return _lib


def _batch(blob, m):
    return pyemu.EmuBatch(blob, {k: m[k] for k in modelblob.DIMS}, 1)


def lists(e, nmesh):
    """(table [nmesh][ncell][2], entries [used][4] float32 with the vertex ids in column 3 as int32 bits)"""
    L = lib()
    nc = L.rge_support_ncell()
    tab = np.frombuffer((ctypes.c_int32 * (2 * nmesh * nc)).from_address(L.rge_support_table(e.h)), dtype=np.int32).reshape(nmesh, nc, 2).copy()
    cap = ctypes.c_int()
    p = L.rge_support_entries(e.h, ctypes.byref(cap))
    ent = np.frombuffer((ctypes.c_float * (4 * cap.value)).from_address(p), dtype=np.float32).reshape(-1, 4) if cap.value else np.zeros((0, 4), np.float32)
    used = int(tab[:, :, 1].clip(0).sum())
    return tab, ent[:used].copy()


def scan(e, mesh, dirs):
    d = np.ascontiguousarray(dirs, dtype=np.float32).reshape(-1, 3)
    out = np.zeros((len(d), 4), np.int32)
    lib().rge_support_scan(e.h, mesh, d.ctypes.data, len(d), out.ctypes.data)
    return out


def _hulls():
    """every distinct hull of the committed assets: (asset, blob, model, mesh id)"""
    seen, out = set(), []
    for path in ASSETS:
        blob = open(path, "rb").read()
        m = modelblob.unpack(blob)
        V = m["mesh_vert"].reshape(-1, 3)
        for h in range(m["nmesh"]):
            a, n = int(m["mesh_vertadr"][h]), int(m["mesh_vertnum"][h])
            key = hashlib.sha1(V[a:a + n].astype(np.float32).tobytes()).hexdigest()
            if key not in seen:
                seen.add(key)
                out.append((os.path.basename(path), h))
    return out


def _edge_dirs(N, rng, per_line=64):
    """directions on the cells' edges and corners of every cube face: d_f = +-1 and (u, v) on the grid lines, also scaled"""
    grid = -1.0 + 2.0 * np.arange(N + 1) / N
    uv = [(u, v) for u in grid for v in grid]                                 # corners
    t = rng.uniform(-1, 1, per_line)
    for g in grid:
        uv += [(g, x) for x in t] + [(x, g) for x in t]                       # edges
    uv = np.array(uv)
    out = []
    for f in range(3):
        a, b = (f + 1) % 3, (f + 2) % 3
        for s in (1.0, -1.0):
            d = np.zeros((len(uv), 3))
            d[:, f] = s
            d[:, a], d[:, b] = uv[:, 0], uv[:, 1]
            out.append(d)
    d = np.concatenate(out)
    return np.concatenate([d, 0.37 * d, 1e-3 * d, 3.1 * d]).astype(np.float32)


def test_cell_lookup():
    """rg_hull_cell: face = largest |component| and its sign, then the N x N grid of (d_a, d_b) / |d_f|; -1 (whole-hull scan)
    for zero, tiny, huge and non-finite directions"""
    L = lib()
    N = L.rge_support_celln()
    rng = np.random.RandomState(3)
    d = rng.randn(20000, 3).astype(np.float32)
    got = np.array([L.rge_support_cell(np.ascontiguousarray(x).ctypes.data) for x in d])
    ad = np.abs(d.astype(np.float64))
    f = np.argmax(ad, axis=1)
    r = np.arange(len(d))
    mx = ad[r, f]
    u, v = d[r, (f + 1) % 3] / mx, d[r, (f + 2) % 3] / mx
    i, j = np.floor((u + 1) * N / 2), np.floor((v + 1) * N / 2)
    far = (np.abs((u + 1) * N / 2 - np.round((u + 1) * N / 2)) > 1e-4) & (np.abs((v + 1) * N / 2 - np.round((v + 1) * N / 2)) > 1e-4)
    want = ((2 * f + (d[r, f] < 0)) * N + i) * N + j
    assert far.mean() > 0.99 and np.array_equal(got[far], want[far].astype(int))
    for bad in ([0, 0, 0], [1e-16, -1e-16, 0], [np.nan, 1, 0], [0, np.inf, 1], [2e30, 0, 0]):
        assert L.rge_support_cell(np.array(bad, np.float32).ctypes.data) == -1, bad


@pytest.mark.parametrize("asset,mesh", _hulls(), ids=lambda x: str(x))
def test_cell_scan_matches_whole_hull_scan(asset, mesh):
    blob = open(os.path.join(ROOT, "robogym_b200", "assets", asset), "rb").read()
    m = modelblob.unpack(blob)
    e = _batch(blob, m)
    rng = np.random.RandomState(mesh)
    a, n = int(m["mesh_vertadr"][mesh]), int(m["mesh_vertnum"][mesh])
    fa, fn = int(m["mesh_faceadr"][mesh]), int(m["mesh_facenum"][mesh])
    V = m["mesh_vert"].reshape(-1, 3)[a:a + n].astype(np.float32)
    F = m["mesh_face"].reshape(-1, 3)[fa:fa + fn]
    normals = np.cross(V[F[:, 1]] - V[F[:, 0]], V[F[:, 2]] - V[F[:, 0]]).astype(np.float32)
    axes = np.array([(i, j, k) for i in (-1, 0, 1) for j in (-1, 0, 1) for k in (-1, 0, 1) if (i, j, k) != (0, 0, 0)], np.float32)
    N = lib().rge_support_celln()
    sets = {"random": rng.randn(100000, 3).astype(np.float32), "face normals": np.concatenate([normals, -normals]),
            "axes and diagonals": np.concatenate([axes, 0.01 * axes, 7.0 * axes]), "cell edges and corners": _edge_dirs(N, rng)}
    for name, d in sets.items():
        out = scan(e, mesh, d)
        for col, what in ((0, "group-shared list scan"), (2, "one-lane list scan"), (3, "one-lane whole-hull scan")):
            bad = np.nonzero(out[:, col] != out[:, 1])[0]
            assert len(bad) == 0, (name, what, d[bad[:5]], out[bad[:5]])
    # every list is ascending, holds ids of this hull, and names each vertex with its own coordinates
    tab, ent = lists(e, m["nmesh"])
    ids = ent[:, 3].view(np.int32)
    for off, cnt in tab[mesh]:
        assert cnt >= 1
        k = ids[off:off + cnt]
        assert np.all(np.diff(k) > 0) and k.min() >= 0 and k.max() < n
        assert np.array_equal(ent[off:off + cnt, :3], V[k])


def test_list_sizes_and_build_time():
    """the lists stay short (the scan's point) and their construction cheap at model load"""
    L = lib()
    for path in ASSETS:
        blob = open(path, "rb").read()
        m = modelblob.unpack(blob)
        if m["nmesh"] == 0:
            continue
        e = _batch(blob, m)
        tab, _ = lists(e, m["nmesh"])
        cnt = tab[:, :, 1]
        assert cnt.min() >= 1
        assert cnt.mean() < 0.25 * m["mesh_vertnum"].mean() + 2, (path, cnt.mean())
        assert L.rge_support_build_seconds(e.h) < 10.0


def _aabb(m, verts):
    """geom_aabb of the mesh geoms for edited vertices, as rg_model_set_field("mesh_vert") recomputes it"""
    aabb = m["geom_aabb"].copy().reshape(-1, 6)
    V = verts.reshape(-1, 3)
    for g in range(m["ngeom"]):
        mid = int(m["geom_dataid"][g])
        if m["geom_type"][g] != 7 or mid < 0:
            continue
        a, n = int(m["mesh_vertadr"][mid]), int(m["mesh_vertnum"][mid])
        lo, hi = V[a:a + n].min(0), V[a:a + n].max(0)
        aabb[g, :3], aabb[g, 3:] = 0.5 * (lo + hi), 0.5 * (hi - lo)
    return aabb.reshape(-1)


@pytest.mark.parametrize("asset", ["dactyl_locked", "rearrange_ycb8"])
def test_mesh_vert_edit_rebuilds_lists(asset):
    """mesh_vert edited on a loaded model (what rg_model_set_field does) against a model loaded with the edited hulls: the same
    lists, entry for entry, and the same emulated env-step, bit for bit"""
    blob = open(os.path.join(ROOT, "robogym_b200", "assets", asset + ".rgm"), "rb").read()
    m = modelblob.unpack(blob)
    rng = np.random.RandomState(5)
    verts = m["mesh_vert"] * 1.05 + 1e-5 * rng.randn(m["mesh_vert"].size)
    edited = dict(m, mesh_vert=verts, geom_aabb=_aabb(m, verts))
    blob2 = modelblob.pack(edited, modelblob.unpack_names(blob))
    e1, e2 = _batch(blob, m), _batch(blob2, m)
    v = np.ascontiguousarray(verts, dtype=np.float64)
    lib().rge_support_set_vert(e1.h, v.ctypes.data)
    e1.model_field("geom_aabb", np.float32)[:] = np.asarray(edited["geom_aabb"], dtype=np.float32)
    t1, n1 = lists(e1, m["nmesh"])
    t2, n2 = lists(e2, m["nmesh"])
    _, n0 = lists(_batch(blob, m), m["nmesh"])
    assert np.array_equal(t1, t2) and np.array_equal(n1.view(np.int32), n2.view(np.int32))
    assert t1[:, :, 1].min() >= 1                                    # the rebuilt lists fit: no hull fell back to the whole scan
    assert n0.shape != n1.shape or not np.array_equal(n0, n1)       # and they did change
    mocap = np.nonzero(m["body_mocapid"] >= 0)[0][np.argsort(m["body_mocapid"][m["body_mocapid"] >= 0])]
    for e in (e1, e2):
        e.qpos[:] = m["qpos0"]
        e.ctrl[:] = m["actuator_ctrlrange"].reshape(-1, 2).mean(1)
        if e.mocap_pos is not None:
            e.mocap_pos[:] = m["body_pos"].reshape(-1, 3)[mocap][None]
            e.mocap_quat[:] = m["body_quat"].reshape(-1, 4)[mocap][None]
    ncon = 0
    for _ in range(3):
        e1.step(10, 1)
        e2.step(10, 1)
        assert np.array_equal(e1.qpos, e2.qpos) and np.array_equal(e1.qvel, e2.qvel) and np.array_equal(e1.ncon, e2.ncon)
        ncon += int(e1.ncon[0])
    assert ncon > 0
