"""What an environment computes does not depend on how the step kernel is laid out or launched: bit-identical results across
scratch layouts (rg_make_layout at other capacities), warps per CTA and the two kernel builds, barrier groups, work ordering,
the separating-axis cache carried between launches, subset launches, per-environment model views and batch sizes -- on every
bench scene.

A capacity that is too small may change an environment's results only together with the warning bit that its own overflow
explains: more contacts than the contact capacity (RG_WARN_CONTACT_FULL), more single-row constraints than the row capacity
(RG_WARN_ROWS_FULL), or a contact that touches more dofs than the per-contact capacity (RG_WARN_DOFS_FULL).  Overflow counts
come from the reference run's debug view.

CPU tier: the emulation of the kernel source (tests/emu), which compiles the engine's own rg_make_layout.  GPU tier (-m gpu):
the CUDA path against a one-warp-per-CTA, unordered, unbound launch of the same states."""
import ctypes
import functools
import json
import os
import sys

import numpy as np
import pytest

import pyemu
from helpers import contract_states, full_cube_states, rollout_states
from robogym_b200 import modelblob

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
ASSETS = os.path.join(ROOT, "robogym_b200", "assets")
sys.path.insert(0, os.path.join(HERE, "stubs"))

WARN_CONTACT_FULL, WARN_ROWS_FULL, WARN_DOFS_FULL = 1, 2, 32
# per-environment outputs compared bit for bit (engine names; the emulation calls qacc_warmstart "warm")
OUTPUTS = ("qpos", "qvel", "pid", "qacc_warmstart", "time", "ncon", "contact", "site_xpos", "body_xpos", "body_xquat", "geom_xpos",
           "act_force", "qacc", "sensordata")
# the aliases rg_make_layout takes or skips depending on the capacities (robogym_b200/csrc/rg_step.inl)
ALIASES = {
    "inertia_in_con": lambda L: L["I10"] == L["con"],        # body inertias inside the contact records
    "tile_in_cw": lambda L: L["tileJ"] == L["cw"],           # Hessian tiles inside the contact solver vectors
    "late": lambda L: L["gxpos"] == L["el_i"],               # geom / site positions, tendon forces inside the constraint rows
    "lpos_in_cu": lambda L: L["lpos"] == L["cu"],            # local frames inside the contact solver vectors
    "stage_in_cu": lambda L: L["stage"] == L["cu"],          # narrow-phase staging inside the contact solver vectors
}


def _blob(asset):
    with open(os.path.join(ASSETS, asset + ".rgm"), "rb") as f:
        return f.read()


def _names(asset):
    with open(os.path.join(ASSETS, asset + ".names.json")) as f:
        return json.load(f)


class Scene:
    """one model with its teacher-forcing states.  states[k] = (qpos, qvel, ctrl, pid, warmstart[, mocap_pos, mocap_quat]);
    `edits` are model-wide array edits every run carries; `pairs`: the batch streams per-environment pair lists (a slotted
    model with disabled parts); `grid`: capacity triples (contacts, rows, dofs per contact) of the layout grid; `ref_caps`:
    the reference run's, raised from the bench's (`bench_caps`, 0 = engine default) until nothing overflows."""

    def __init__(self, name, asset, states, nsub, final_forward, ref_caps, grid, bench_nenv, bench_caps, edits=None, blob=None, pairs=False):
        self.name, self.asset, self.states, self.nsub, self.final_forward = name, asset, states, nsub, final_forward
        self.ref_caps, self.grid, self.bench_nenv, self.bench_caps = ref_caps, grid, bench_nenv, bench_caps
        self.edits = edits or {}
        self.blob = blob if blob is not None else _blob(asset)
        self.m = modelblob.unpack(self.blob)
        self.dims = {k: self.m[k] for k in modelblob.DIMS}
        self.pairs = pairs
        self.mesh = int(self.m["nmesh"]) > 0

    @functools.cached_property
    def dof_chains(self):
        """dof ids of every body's chain to the world (its own and its ancestors'), from body_parentid / body_dofadr / body_dofnum"""
        m = self.m
        chains = [frozenset()]
        for b in range(1, m["nbody"]):
            own = range(int(m["body_dofadr"][b]), int(m["body_dofadr"][b]) + int(m["body_dofnum"][b]))
            chains.append(chains[int(m["body_parentid"][b])] | frozenset(own))
        return chains

    def contact_dofs(self, g1, g2):
        """dofs a contact between two geoms moves: the bodies' chains without the part they share (rg_make_constraints)"""
        b1, b2 = int(self.m["geom_bodyid"][g1]), int(self.m["geom_bodyid"][g2])
        return len(self.dof_chains[b1] ^ self.dof_chains[b2])


# ---------------------------------------------------------------------------------------------- scenes and their states
def _locked():
    blob = _blob("dactyl_locked")
    sts, _, _ = contract_states(blob, range(300, 302), 8)
    return Scene("locked", "dactyl_locked", sts, 10, 1, (100, 256, 32),
                 [(20, 40, 8), (20, 64, 16), (24, 64, 12), (32, 64, 16), (48, 96, 24)], 8192, bench_caps=(0, 0, 0))


def _reach():
    blob = _blob("dactyl_reach")
    sts, _, _ = rollout_states(blob, 16, seed=5, action_scale=1.0)
    return Scene("dactyl_reach", "dactyl_reach", sts, 10, 1, (100, 256, 32),
                 [(100, 64, 16), (20, 40, 8), (20, 64, 16), (32, 96, 24)], 8192, bench_caps=(100, 0, 0))


def _full():
    blob = _blob("dactyl_full_perpendicular")
    sts, _ = full_cube_states(blob, 8)
    return Scene("full_perpendicular", "dactyl_full_perpendicular", sts, 10, 1, (128, 384, 32),
                 [(96, 288, 32), (40, 200, 16), (64, 256, 24), (128, 384, 32)], 4096, bench_caps=(96, 288, 32))


def _blocks():
    import test_rearrange_blocks as T

    blob = _blob("rearrange_blocks5")
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    sts, _, eqd = T._rollout(blob, m, names, 12)
    return Scene("rearrange_blocks", "rearrange_blocks5", sts, 20, 1, (100, 256, 32),
                 [(64, 128, 16), (20, 64, 8), (23, 128, 16), (32, 96, 12)], 2048, edits={"eq_data": eqd}, bench_caps=(64, 128, 16))


def _ycb():
    import test_rearrange_ycb as T

    blob = _blob("rearrange_ycb8")
    m, names = modelblob.unpack(blob), modelblob.unpack_names(blob)
    sts, _, eqd, _ = T._rollout(blob, m, names, 8, settle=400)
    return Scene("rearrange_ycb", "rearrange_ycb8", sts, 20, 1, (100, 256, 32),
                 [(64, 128, 16), (20, 128, 16), (23, 128, 16), (24, 64, 8), (32, 48, 12)], 1024, edits={"eq_data": eqd},
                 bench_caps=(64, 128, 16))


def _mesh_scene():
    """the slotted YCB scene (robogym_b200.rearrange_mesh_scene) holding the identity draw: the padded model's own geom_dataid row
    enables the base scene's parts, and every environment streams the pair list derived from it"""
    import test_mesh_scene as T

    from robogym_b200 import rearrange_mesh_scene as rms

    b8, bt = _blob("rearrange_ycb8"), _blob("rearrange_ycb8_tcp")
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    sb = rms.slotted_model(b8, lib)
    sts, _, eqd, _ = T._rollout(b8, lib, lib.identity[0], 8, settle=200)
    return Scene("mesh_scene", None, sts, 20, 1, (100, 256, 32),
                 [(64, 128, 16), (23, 128, 16), (24, 64, 8), (32, 96, 12)], 1024, edits={"eq_data": eqd}, blob=sb, pairs=True,
                 bench_caps=(64, 128, 0))


def _tcp(config):
    """states the dual-simulation workload of bench.py reaches on the emulated kernels (main scene after two env-steps)"""
    import torch

    import bench
    from emu_generic_sim import EmuGenericSim

    cfg = bench.CONFIGS[config]
    blob, sblob = _blob(cfg["asset"]), _blob(cfg["solver_asset"])
    n = 8
    main = EmuGenericSim(blob, n, cfg["nsub"], contact_capacity=cfg["caps"][0], row_capacity=cfg["caps"][1])
    solver = EmuGenericSim(sblob, n, cfg["nsub"])
    gen = torch.Generator(device="cpu")
    gen.manual_seed(3)
    wl = bench.RearrangeTcpWorkload(main, main.model, _names(cfg["asset"]), torch.device("cpu"), gen, cfg["nobj"], cfg["grid"], solver)
    for _ in range(2):
        wl.apply_action(wl.sample_action())
        wl.step_timed()
    e = main.e
    sts = [(e.qpos[k].copy(), e.qvel[k].copy(), e.ctrl[k].copy(), e.pid[k].copy(), e.warm[k].copy(), e.mocap_pos[k, 0].copy(),
            e.mocap_quat[k, 0].copy()) for k in range(n)]
    grid = [(64, 160, 16), (20, 64, 8), (23, 160, 16), (32, 96, 12)]
    return Scene(config, cfg["asset"], sts, cfg["nsub"], wl.ctl.main_forwards, (100, 256, 32), grid, cfg["nenv"], bench_caps=cfg["caps"])


BUILDERS = {
    "locked": _locked,
    "full_perpendicular": _full,
    "rearrange_blocks": _blocks,
    "rearrange_blocks_tcp": lambda: _tcp("rearrange_blocks_tcp"),
    "rearrange_ycb_tcp": lambda: _tcp("rearrange_ycb_tcp"),
    "rearrange_ycb": _ycb,
    "dactyl_reach": _reach,
    "mesh_scene": _mesh_scene,
}


def test_every_bench_config_has_a_scene():
    import bench

    assert set(bench.CONFIGS) <= set(BUILDERS)


@functools.lru_cache(maxsize=None)
def scene(name):
    return BUILDERS[name]()


# ---------------------------------------------------------------------------------------------- comparisons
class Run:
    """the outputs of one run after each of its launches ([nenv, ...] numpy arrays), with the overflow counts of the debug view:
    contacts and single-row constraints of the launch's last forward pass, and the most dofs one of its contacts touches"""

    def __init__(self):
        self.snaps, self.ncon, self.nel, self.dofs = [], [], [], []

    @property
    def out(self):
        return self.snaps[-1]

    def record(self, sc, outputs, dbg):
        self.snaps.append(outputs)
        if dbg is not None:
            o = sc.dims["nv"] * sc.dims["nv"] + 6 * sc.dims["nv"] + sc.dims["ntendon"] + 2 * sc.dims["nu"]   # rg_dbg_size's order
            ncon, nel, con = dbg[:, o].astype(int), dbg[:, o + 1].astype(int), outputs["contact"]
            self.ncon.append(ncon)
            self.nel.append(nel)
            self.dofs.append(np.array([max([sc.contact_dofs(int(c[0]), int(c[1])) for c in con[k, :ncon[k]]] or [0]) for k in range(len(ncon))]))


def _first_difference(a, b, k):
    """the first output of environment k that differs in any bit between two snapshots (contact records: the rows both
    capacities hold), or None"""
    for name in OUTPUTS:
        if name in a:
            x, y = a[name][k], b[name][k]
            if name == "contact":
                x, y = x[:len(y)], y[:len(x)]
            if x.tobytes() != y.tobytes():
                return name
    return None


def assert_identical(ref, var, what, envs=None):
    """every output of every (selected) environment bit for bit"""
    envs = range(len(ref.out["qpos"])) if envs is None else envs
    bad = [(k, d) for k in envs if (d := _first_difference(ref.out, var.out, k))]
    assert not bad, f"{what}: {len(bad)} environments differ from the reference, first (env, output): {bad[:6]}"


def assert_explained(ref, var, caps, what):
    """Launch by launch (one substep each): an environment matches the reference bit for bit up to the launch in which it first
    warns, and that warning is the overflow the reference's same forward pass shows at these capacities.  From there on it
    has lost a contact or a row, and its results may differ."""
    errs = []
    for k in range(len(var.out["warn"])):
        for i, (a, b) in enumerate(zip(ref.snaps, var.snaps)):
            w = int(b["warn"][k])
            if not w:
                if d := _first_difference(a, b, k):
                    errs.append((k, f"{d} differs after launch {i} without a warning"))
                    break
                continue
            cause = {WARN_CONTACT_FULL: ref.ncon[i][k] > caps[0], WARN_ROWS_FULL: ref.nel[i][k] > caps[1],
                     WARN_DOFS_FULL: ref.dofs[i][k] > min(caps[2], 32)}
            bad = [bit for bit, ok in cause.items() if w & bit and not ok]
            if bad or w & ~sum(cause):
                errs.append((k, "warning %d in launch %d, where the reference has %d contacts, %d rows, %d dofs per contact"
                             % (w, i, ref.ncon[i][k], ref.nel[i][k], ref.dofs[i][k])))
            break
    assert not errs, f"{what}: {len(errs)} environments, first (env, finding): {errs[:6]}"


# ---------------------------------------------------------------------------------------------- CPU tier: the emulation
def emu_batch(sc, nenv, caps):
    e = pyemu.EmuBatch(sc.blob, sc.dims, nenv, contact_capacity=caps[0], row_capacity=caps[1], dofs_per_contact=caps[2])
    for k, v in sc.edits.items():
        e.model_field(k, np.float32)[:] = v
    if sc.pairs:
        did = np.asarray(sc.m["geom_dataid"], np.int32)
        lst = np.zeros(sc.m["npair"], np.uint32)
        w = ctypes.c_int()
        n = pyemu.lib().rge_pairs(e.h, did.ctypes.data, lst.ctypes.data, len(lst), ctypes.byref(w))
        assert w.value == 0
        e.use_pairs(lst, n)
    return e


def emu_load(e, states):
    e.time[:] = 0
    e.warn[:] = 0
    for k, st in enumerate(states):
        e.qpos[k], e.qvel[k], e.ctrl[k], e.pid[k], e.warm[k] = [np.asarray(a) for a in st[:5]]
        if e.mocap_pos is not None and len(st) > 5:
            e.mocap_pos[k, 0], e.mocap_quat[k, 0] = st[5], st[6]


def launches(sc, steps, split):
    """(substeps, forwards) of the launches of `steps` env-steps; split: one launch per substep and one for the final forward
    passes, so that the debug view sees every forward pass"""
    one = [(1, 0)] * sc.nsub + [(0, sc.final_forward)] if split else [(sc.nsub, sc.final_forward)]
    return one * steps


def emu_run(sc, caps, e=None, steps=2, split=False):
    """a fresh batch (or `e`) loaded with the scene's states, `steps` env-steps"""
    if e is None:
        e = emu_batch(sc, len(sc.states), caps)
    emu_load(e, sc.states)
    r = Run()
    for nsub, nfwd in launches(sc, steps, split):
        e.step(nsub, nfwd)
        out = {}
        for name in OUTPUTS + ("warn",):
            a = getattr(e, "warm" if name == "qacc_warmstart" else name)
            if a is not None and a.size:
                out[name] = a.copy()
        r.record(sc, out, e.dbg)
    return r


@functools.lru_cache(maxsize=None)
def emu_reference(name, split=False):
    sc = scene(name)
    ref = emu_run(sc, sc.ref_caps, split=split)
    assert int(ref.out["warn"].max()) == 0, f"{name}: the reference capacities {sc.ref_caps} overflow: {ref.out['warn']}"
    return ref


def test_layout_grid_takes_every_alias_both_ways():
    """Across the grid, each of the aliases rg_make_layout takes by capacity is taken on some scene and skipped on some scene,
    so the grid cannot quietly stop covering either side."""
    seen = {a: set() for a in ALIASES}
    for name in BUILDERS:
        sc = scene(name)
        for caps in sc.grid:
            L = pyemu.layout(sc.blob, *caps)
            assert (L["ncon"], L["nel"], L["tile"]) == (caps[0], caps[1], min(caps[2], 32, sc.dims["nv"]))
            for a, taken in ALIASES.items():
                seen[a].add(bool(taken(L)))
    print("aliases taken / not taken across the layout grid:", {a: sorted(v) for a, v in seen.items()})
    assert all(v == {True, False} for v in seen.values()), seen


@pytest.mark.parametrize("name", list(BUILDERS))
def test_emulated_layouts_are_bit_identical_or_warn(name):
    """Two env-steps of the scene's states at every capacity triple of its grid, one launch per substep: each environment either
    matches the reference layout bit for bit or carries the warnings of its own overflow."""
    sc = scene(name)
    ref = emu_reference(name, split=True)
    for caps in sc.grid:
        var = emu_run(sc, caps, split=True)
        assert_explained(ref, var, caps, f"{name} at capacities {caps}")


@pytest.mark.parametrize("name", ["locked", "rearrange_ycb"])
def test_emulated_separating_axis_cache_does_not_change_results(name):
    """A batch that stepped other states for three env-steps (its cache warm with their separations) and is then loaded with the
    test states steps them exactly like a fresh batch."""
    sc = scene(name)
    e = emu_batch(sc, len(sc.states), sc.ref_caps)
    emu_load(e, sc.states[::-1])
    for _ in range(3):
        e.step(sc.nsub, sc.final_forward)
    assert_identical(emu_reference(name), emu_run(sc, sc.ref_caps, e=e), f"{name}, warm separating-axis cache")


# ---------------------------------------------------------------------------------------------- GPU tier: the CUDA path
GPU_OUTPUTS = ("site_xpos", "body_xpos", "body_xquat", "geom_xpos", "act_force", "qacc", "contact", "sensordata", "ncon", "warn")
# per-environment rows bound with the model's own values (what the randomisers edit); geom_dataid as well on the mesh scenes
VIEW_ROWS = ("dof_damping", "geom_friction", "body_mass", "actuator_gainprm")


@pytest.fixture(scope="module")
def gpu():
    import torch

    from robogym_b200 import build, engine

    assert torch.cuda.is_available(), "gpu tests need a CUDA device"
    build.build()
    return torch, engine


@pytest.fixture
def launch_env(monkeypatch):
    """no launch-geometry experiment setting leaks in from outside; the test sets what it varies"""
    for k in ("RG_WARPS_PER_CTA", "RG_BAR_GROUPS", "RG_BALANCE", "RG_CTAS_PER_SM"):
        monkeypatch.delenv(k, raising=False)
    return monkeypatch


@functools.lru_cache(maxsize=None)
def device_model(name):
    from robogym_b200 import engine

    sc = scene(name)
    model = engine.DeviceModel(sc.blob, 0)
    for k, v in sc.edits.items():
        model.set_field(k, v)
    return model


def gpu_batch(gpu, sc, nenv, caps, debug=True):
    torch, engine = gpu
    outs = tuple(o for o in GPU_OUTPUTS if o != "sensordata" or sc.dims["nsensordata"])
    return engine.BatchedSim(device_model(sc.name), nenv, sc.nsub, outputs=outs, debug=debug, contact_capacity=caps[0],
                             row_capacity=caps[1], dofs_per_contact=caps[2])


def gpu_load(gpu, sim, states, idx=None):
    torch, _ = gpu
    f = lambda i: torch.tensor(np.stack([s[i] for s in states]), dtype=torch.float32, device=sim.device)[idx if idx is not None else slice(None)]
    sim.qpos.copy_(f(0)); sim.qvel.copy_(f(1)); sim.ctrl.copy_(f(2)); sim.pid.copy_(f(3)); sim.qacc_warmstart.copy_(f(4))
    sim.time.zero_()
    sim.warn.zero_()
    if sim.mocap_pos is not None and len(states[0]) > 5:
        sim.mocap_pos[:, 0].copy_(f(5)); sim.mocap_quat[:, 0].copy_(f(6))


def gpu_run(gpu, sc, sim, steps=2, mask=None, idx=None, split=False):
    """the scene's states (rows `idx` of them, tiled) loaded into `sim`, `steps` env-steps (of the environments of `mask`);
    split: a snapshot after every launch of one substep (launches()), else after the last launch"""
    torch, _ = gpu
    gpu_load(gpu, sim, sc.states, idx)
    r = Run()
    todo = launches(sc, steps, split)
    for j, (nsub, nfwd) in enumerate(todo):
        sim.step(nsub, nfwd, mask=mask)
        if split or j == len(todo) - 1:
            torch.cuda.synchronize()
            out = {name: getattr(sim, name).cpu().numpy() for name in OUTPUTS + ("warn",)
                   if getattr(sim, name, None) is not None and getattr(sim, name).numel()}
            r.record(sc, out, sim.dbg.cpu().numpy() if split else None)
    return r


def tiled(run, idx):
    """a run's last outputs, environment idx[j] in row j"""
    t = Run()
    t.snaps = [{k: v[idx] for k, v in run.out.items()}]
    return t


def gpu_reference(gpu, launch_env, sc, split=False, caps=None):
    """one warp per CTA, no work ordering, no per-environment rows, the reference capacities (or `caps`)"""
    launch_env.setenv("RG_WARPS_PER_CTA", "1")
    sim = gpu_batch(gpu, sc, len(sc.states), caps or sc.ref_caps)
    sim.set_balance(False)
    assert sim.launch_info()["warps_per_cta"] == 1
    ref = gpu_run(gpu, sc, sim, split=split)
    assert caps or int(ref.out["warn"].max()) == 0, f"{sc.name}: the reference capacities {sc.ref_caps} overflow: {ref.out['warn']}"
    launch_env.delenv("RG_WARPS_PER_CTA")
    return ref


def _show(sc, what, sim):
    print(f"{sc.name} {what}: {sim.launch_info()}")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_cuda_layouts_are_bit_identical_or_warn(gpu, launch_env, name):
    sc = scene(name)
    ref = gpu_reference(gpu, launch_env, sc, split=True)
    for caps in sc.grid:
        sim = gpu_batch(gpu, sc, len(sc.states), caps)
        sim.set_balance(False)
        _show(sc, f"capacities {caps}", sim)
        assert_explained(ref, gpu_run(gpu, sc, sim, split=True), caps, f"{name} at capacities {caps}")


@pytest.mark.gpu
@pytest.mark.parametrize("warps", [2, 3, 7, 12, 13])
@pytest.mark.parametrize("name", list(BUILDERS))
def test_cuda_warps_per_cta_do_not_change_results(gpu, launch_env, name, warps):
    """2, odd counts, 12 (the 168-register build) and 13 (the 128-register build) warps per CTA at the bench's capacities; the
    scene's states and 37 environments (a partial last round at every count) against the one-warp launch"""
    sc = scene(name)
    ref = gpu_reference(gpu, launch_env, sc, caps=sc.bench_caps)
    n = len(sc.states)
    launch_env.setenv("RG_WARPS_PER_CTA", str(warps))
    sim = gpu_batch(gpu, sc, n, sc.bench_caps)
    sim.set_balance(False)
    got = sim.launch_info()["warps_per_cta"]
    if got != warps:
        pytest.skip(f"{name}: {warps} warps of {sim.launch_info()['scratch_bytes_per_env']} B scratch do not fit in shared memory")
    _show(sc, f"{warps} warps per CTA", sim)
    assert_identical(ref, gpu_run(gpu, sc, sim), f"{name}, {warps} warps per CTA")
    idx = np.arange(37) % n
    big = gpu_batch(gpu, sc, 37, sc.bench_caps)
    big.set_balance(False)
    assert big.launch_info()["warps_per_cta"] == warps
    assert_identical(tiled(ref, idx), gpu_run(gpu, sc, big, idx=idx), f"{name}, 37 environments at {warps} warps per CTA")


@pytest.mark.gpu
@pytest.mark.parametrize("groups", [2, 3])
@pytest.mark.parametrize("name", list(BUILDERS))
def test_cuda_barrier_groups_do_not_change_results(gpu, launch_env, name, groups):
    sc = scene(name)
    ref = gpu_reference(gpu, launch_env, sc)
    launch_env.setenv("RG_BAR_GROUPS", str(groups))
    launch_env.setenv("RG_WARPS_PER_CTA", "4")            # (where it fits: a CTA of one warp has one barrier group)
    sim = gpu_batch(gpu, sc, len(sc.states), sc.ref_caps)
    sim.set_balance(False)
    _show(sc, f"{groups} barrier groups", sim)
    assert_identical(ref, gpu_run(gpu, sc, sim), f"{name}, {groups} barrier groups")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_cuda_work_ordering_and_a_warm_cache_do_not_change_results(gpu, launch_env, name):
    """Work ordering on, after three launches on other states (the scene's states in reverse): the slot table is sorted by those
    states' costs and the separating-axis cache holds their separations when the test states are loaded."""
    torch, _ = gpu
    sc = scene(name)
    ref = gpu_reference(gpu, launch_env, sc)
    launch_env.setenv("RG_WARPS_PER_CTA", "4")
    sim = gpu_batch(gpu, sc, len(sc.states), sc.ref_caps)
    sim.set_balance(True)
    gpu_load(gpu, sim, sc.states[::-1])
    for _ in range(3):
        sim.step(final_forward=sc.final_forward)
    _show(sc, "work-ordered after warm-up", sim)
    assert_identical(ref, gpu_run(gpu, sc, sim), f"{name}, work-ordered with a warm cache")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_cuda_subset_launch_matches_the_full_launch(gpu, launch_env, name):
    """step(mask=...) with a scattered selection: the selected environments match the reference, the others are untouched"""
    torch, _ = gpu
    sc = scene(name)
    ref = gpu_reference(gpu, launch_env, sc)
    n = len(sc.states)
    sel = np.zeros(n, bool)
    sel[[k for k in range(n) if k % 3 == 0 or k % 5 == 2]] = True
    sim = gpu_batch(gpu, sc, n, sc.ref_caps, debug=False)
    sim.set_balance(False)
    gpu_load(gpu, sim, sc.states)
    sim.forward()                           # every output row holds something the subset launches must leave alone
    torch.cuda.synchronize()
    before = {k: getattr(sim, k).cpu().numpy().copy() for k in OUTPUTS + ("warn",) if getattr(sim, k, None) is not None and getattr(sim, k).numel()}
    mask = torch.as_tensor(sel, device=sim.device)
    r = gpu_run(gpu, sc, sim, mask=mask)
    assert_identical(ref, r, f"{name}, selected environments of a subset launch", envs=np.nonzero(sel)[0])
    # the state rows were reloaded from the states by gpu_run, the derived outputs still hold the forward pass's
    loaded = dict(qpos=0, qvel=1, pid=3, qacc_warmstart=4)
    for k, v in before.items():
        want = np.stack([np.asarray(s[loaded[k]], np.float32) for s in sc.states]) if k in loaded else v
        assert r.out[k][~sel].tobytes() == want[~sel].tobytes(), f"{name}: the subset launch wrote {k} of an unselected environment"


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_cuda_per_environment_model_views_do_not_change_results(gpu, launch_env, name):
    """Rows equal to the model's own values bound per environment (each warp then steps its own copy of the model view), and on
    the mesh scenes geom_dataid as well (each environment then streams its own pair list): the results of the unbound run."""
    sc = scene(name)
    ref = gpu_reference(gpu, launch_env, sc)
    n = len(sc.states)
    launch_env.setenv("RG_WARPS_PER_CTA", "4")            # several warps, each with its own view copy (where they fit)
    sim = gpu_batch(gpu, sc, n, sc.ref_caps)
    sim.set_balance(False)
    for f in VIEW_ROWS:
        sim.set_param(f, np.repeat(np.asarray(sc.m[f], np.float64).reshape(1, -1), n, axis=0))
    if sc.mesh:
        sim.set_param("geom_dataid", np.repeat(np.asarray(sc.m["geom_dataid"]).reshape(1, -1), n, axis=0))
        sim.update_pairs()
        assert sim.pair_counts() is not None
    _show(sc, "per-environment model views", sim)
    assert_identical(ref, gpu_run(gpu, sc, sim), f"{name}, per-environment rows")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(BUILDERS))
def test_cuda_bench_size_launch_matches_the_small_launch(gpu, launch_env, name):
    """The scene's states tiled over its bench batch (default launch geometry and work ordering): every environment matches the
    one-warp launch of the states themselves."""
    torch, _ = gpu
    sc = scene(name)
    ref = gpu_reference(gpu, launch_env, sc)
    N = sc.bench_nenv
    idx = np.arange(N) % len(sc.states)
    sim = gpu_batch(gpu, sc, N, sc.ref_caps, debug=False)
    _show(sc, f"{N} environments", sim)
    assert_identical(tiled(ref, idx), gpu_run(gpu, sc, sim, idx=idx), f"{name}, {N} environments")
