"""One environment per CTA of W warps (robogym_b200/csrc/rg_cta.cu): the dense loops of the Newton solve spread over the CTA, and
what an environment computes stays bit for bit what the one-warp kernel computes.

CPU tier: the emulation of both builds of the same source (tests/emu/rg_emu_cta.cpp) -- whole env-steps on every output, and the
envelope factorisation and substitutions on random matrices -- and the engine's selection rule from the shared-memory budgets
of tools/residency.py.  GPU tier (-m gpu): the CUDA kernel at every W against the one-warp, one-environment-per-CTA reference of
tests/test_step_invariance.py, at the bench's batch, under a masked subset launch and with per-environment rows and timestep."""
import os
import sys

import numpy as np
import pytest

import pyemu_cta
from test_step_invariance import (BUILDERS, VIEW_ROWS, assert_identical, gpu, gpu_batch, gpu_reference, gpu_run, launch_env,  # noqa: F401
                                  scene, tiled)

ROOT = os.path.abspath(os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
CTA_MIN_NS, CTA_WARPS = 96, 8      # RG_CTA_MIN_NS, RG_CTA_WARPS (robogym_b200/csrc/rg_engine.cu)


# ---------------------------------------------------------------------------------------------- CPU tier: the emulation
def emu_step(coop, sc, warps, steps=2, caps=None):
    """the scene's states, `steps` env-steps through one build of the emulation; every output it writes"""
    L = pyemu_cta.lib(coop)
    L.rgc_set_warps(warps)
    caps = caps or sc.bench_caps
    h = L.rgc_create(sc.blob, len(sc.blob), *caps)
    assert h
    try:
        n, d = len(sc.states), sc.dims
        npid = len(sc.states[0][3])
        f = np.float32
        out = dict(qpos=np.zeros((n, d["nq"]), f), qvel=np.zeros((n, d["nv"]), f), ctrl=np.zeros((n, d["nu"]), f), pid=np.zeros((n, npid), f),
                   warm=np.zeros((n, d["nv"]), f), sensordata=np.zeros((n, max(d["nsensordata"], 1)), f),
                   contact=np.zeros((n, L.rgc_ncon(h), 4), f), ncon=np.zeros(n, np.int32), warn=np.zeros(n, np.int32))
        for k, st in enumerate(sc.states):
            out["qpos"][k], out["qvel"][k], out["ctrl"][k], out["pid"][k], out["warm"][k] = [np.asarray(a) for a in st[:5]]
        ts = np.full(n, sc.m["opt_timestep"][0], f) * (1.0 + 0.01 * np.arange(n, dtype=f))   # per-environment timestep
        p = lambda a: a.ctypes.data
        for _ in range(steps):
            L.rgc_step(h, n, p(out["qpos"]), p(out["qvel"]), p(out["ctrl"]), p(out["pid"]), p(out["warm"]), p(ts),
                       p(out["sensordata"]) if d["nsensordata"] else None, p(out["contact"]), p(out["ncon"]), p(out["warn"]), sc.nsub, sc.final_forward)
        return out
    finally:
        L.rgc_destroy(h)


def assert_same_bytes(a, b, what):
    bad = [k for k in a if a[k].tobytes() != b[k].tobytes()]
    assert not bad, f"{what}: {bad} differ"


@pytest.mark.parametrize("warps", [2, 4, 8])
def test_emulated_cta_step_is_bit_identical_on_full_cube(warps):
    """Two env-steps of the full cube's states at the bench's capacities: every output of the cooperative build equals the
    one-warp build's bytes."""
    sc = scene("full_perpendicular")
    ref = emu_step(False, sc, 1)
    assert int(ref["ncon"].max()) > 20, "the states should exercise the contact blocks of the Hessian"
    assert_same_bytes(ref, emu_step(True, sc, warps), f"full_perpendicular, W={warps}")


@pytest.mark.parametrize("name", ["locked", "rearrange_blocks_tcp"])
def test_emulated_cta_step_is_bit_identical_when_forced(name):
    """The cooperative code is not specific to the full cube: forced on the locked cube and on the elliptic-cone blocks scene of the
    dual-simulation loop, it is bit-identical too."""
    sc = scene(name)
    ref = emu_step(False, sc, 1)
    for warps in (2, 8):
        assert_same_bytes(ref, emu_step(True, sc, warps), f"{name}, W={warps}")


def random_envelope_spd(rng, n):
    """packed lower rows of an SPD matrix whose row i is zero left of env[i] (random, sometimes right after the diagonal), plus a
    right-hand side in row n"""
    env = np.array([0 if i == 0 else int(rng.integers(0, i + 1)) for i in range(n)], np.int32)
    if n > 3:
        env[n // 2] = n // 2                     # a row whose envelope starts at its own column
    B = np.zeros((n, n))
    for i in range(n):
        B[i, env[i]:i + 1] = rng.normal(size=i + 1 - env[i])
        B[i, i] = abs(B[i, i]) + 1.0
    A = B @ B.T                                  # the envelope of B B' is no wider than B's
    for i in range(n):
        A[i, :env[i]] = 0.0
    A += n * np.eye(n)
    rows = [A[i, :i + 1] for i in range(n)] + [rng.normal(size=n)]
    return np.concatenate(rows).astype(np.float32), env


@pytest.mark.parametrize("n", [1, 5, 31, 33, 64, 100, 168])
def test_emulated_cta_factorisation_and_substitutions_are_bit_identical(n):
    """rg_cholesky, rg_chol_back and rg_chol_forward of the cooperative build at W = 2, 4, 8 against the one-warp build on random
    envelope SPD matrices: sizes below 32 and not multiples of 32 W, rows whose envelope starts at or after a column."""
    rng = np.random.default_rng(n)
    a0, env = random_envelope_spd(rng, n)
    b = rng.normal(size=n).astype(np.float32)
    sidx = np.concatenate([np.arange(n), np.arange(n)]).astype(np.int32)

    def run(coop, warps):
        L = pyemu_cta.lib(coop)
        L.rgc_set_warps(warps)
        a, out, fwd = a0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
        L.rgc_chol(n, a.ctypes.data, env.ctypes.data, b.ctypes.data, sidx.ctypes.data, out.ctypes.data, fwd.ctypes.data)
        return dict(factor=a, solution=out, forward=fwd)

    ref = run(False, 1)
    assert np.isfinite(ref["solution"]).all()
    for warps in (2, 4, 8):
        assert_same_bytes(ref, run(True, warps), f"n={n}, W={warps}")


def test_selection_rule_from_the_shared_memory_budgets():
    """The engine takes the cooperative kernel where the one-warp layout holds a single environment per SM and the solver is large:
    the full cube, and none of the other bench scenes."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import residency

    picked = {}
    for asset in ("dactyl_full_perpendicular", "dactyl_locked", "dactyl_reach", "rearrange_blocks5", "rearrange_blocks5_tcp", "rearrange_ycb8",
                  "rearrange_ycb8_tcp"):
        b = residency.budget(asset, residency.CAPS.get(asset, (0, 0, 0)))
        with open(os.path.join(ROOT, "robogym_b200", "assets", asset + ".rgm"), "rb") as f:
            blob = f.read()
        h = pyemu_cta.lib(False).rgc_create(blob, len(blob), 0, 0, 0)
        ns = pyemu_cta.lib(False).rgc_ns(h)
        pyemu_cta.lib(False).rgc_destroy(h)
        picked[asset] = b["warps_per_cta"] == 1 and ns >= CTA_MIN_NS
    assert picked == {a: a == "dactyl_full_perpendicular" for a in picked}, picked


# ---------------------------------------------------------------------------------------------- GPU tier: the CUDA kernel
def _cta_run(gpu, launch_env, sc, warps, nenv=None, idx=None, mask=None, caps=None, rows=False):
    launch_env.setenv("RG_WARPS_PER_ENV", str(warps))
    sim = gpu_batch(gpu, sc, nenv or len(sc.states), caps or sc.ref_caps)
    info = sim.launch_info()
    assert info["warps_per_env"] == warps and info["warps_per_cta"] == 1, info
    if rows:
        for name in VIEW_ROWS:
            if sc.m[name].size:
                sim.set_param(name, np.repeat(np.asarray(sc.m[name], np.float64).reshape(1, -1), sim.nenv, axis=0))
    run = gpu_run(gpu, sc, sim, mask=mask, idx=idx)
    launch_env.delenv("RG_WARPS_PER_ENV")
    return run


def _reference(gpu, launch_env, sc, caps=None):
    launch_env.setenv("RG_WARPS_PER_ENV", "1")
    ref = gpu_reference(gpu, launch_env, sc, caps=caps)
    launch_env.delenv("RG_WARPS_PER_ENV")
    return ref


@pytest.mark.gpu
def test_engine_selects_the_cta_kernel_for_the_full_cube_only(gpu, launch_env):
    launch_env.delenv("RG_WARPS_PER_ENV", raising=False)
    for name in ("full_perpendicular", "locked", "rearrange_blocks"):
        sc = scene(name)
        info = gpu_batch(gpu, sc, sc.bench_nenv, sc.bench_caps, debug=False).launch_info()
        assert (info["warps_per_env"] == CTA_WARPS) == (name == "full_perpendicular"), (name, info)


@pytest.mark.gpu
@pytest.mark.parametrize("warps", [2, 4, 8, 16])
def test_cta_kernel_is_bit_identical_on_full_cube(gpu, launch_env, warps):
    """every output of the full cube's states after two env-steps, at each W, equals the one-warp reference"""
    sc = scene("full_perpendicular")
    assert_identical(_reference(gpu, launch_env, sc), _cta_run(gpu, launch_env, sc, warps), f"W={warps}")


@pytest.mark.gpu
def test_cta_kernel_at_bench_batch_subset_and_rows(gpu, launch_env):
    """W = 8 at the bench's batch (tiled states), under a masked subset launch, and with per-environment model rows bound"""
    torch, _ = gpu
    sc = scene("full_perpendicular")
    ref = _reference(gpu, launch_env, sc, caps=sc.bench_caps)
    n = sc.bench_nenv
    idx = np.arange(n) % len(sc.states)
    assert_identical(tiled(ref, idx), _cta_run(gpu, launch_env, sc, 8, nenv=n, idx=idx, caps=sc.bench_caps), "batch 4096")
    mask = torch.zeros(n, dtype=torch.bool, device="cuda")
    mask[::3] = True
    sub = _cta_run(gpu, launch_env, sc, 8, nenv=n, idx=idx, mask=mask, caps=sc.bench_caps)
    assert_identical(tiled(ref, idx), sub, "masked subset", envs=range(0, n, 3))
    assert_identical(ref, _cta_run(gpu, launch_env, sc, 8, caps=sc.bench_caps, rows=True), "per-environment rows")


@pytest.mark.gpu
def test_cta_kernel_per_environment_timestep(gpu, launch_env):
    torch, _ = gpu
    sc = scene("full_perpendicular")
    runs = []
    for warps in (1, 8):
        launch_env.setenv("RG_WARPS_PER_ENV", str(warps))
        sim = gpu_batch(gpu, sc, len(sc.states), sc.ref_caps)
        ts = sim.enable_per_env_timestep()
        ts.copy_(torch.full_like(ts, float(sc.m["opt_timestep"][0])) * (1.0 + 0.01 * torch.arange(len(ts), device=ts.device)))
        runs.append(gpu_run(gpu, sc, sim))
    launch_env.delenv("RG_WARPS_PER_ENV")
    assert_identical(runs[0], runs[1], "per-environment timestep")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in BUILDERS if n != "full_perpendicular"])
def test_cta_kernel_forced_on_other_scenes_is_bit_identical(gpu, launch_env, name):
    sc = scene(name)
    assert_identical(_reference(gpu, launch_env, sc), _cta_run(gpu, launch_env, sc, 8), f"{name} forced to W=8")
