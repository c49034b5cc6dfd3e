"""The robot's part of the rearrange reset (rearrange_arm.BatchedTcpArmController.initialize_sim_state /
randomize_initial_position, rg_arm_phase, rg_arm_sample_actions), CPU tier: the random action's draws in the kernel source's
emulation against the numpy replay, the C ABI's argument checks and struct layouts, and the step loop on the fp64 stand-ins.
The CUDA kernel is checked in tests/test_robot_reset_gpu.py."""
import ctypes
import gzip
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import pyemu_arm
from robogym_b200 import engine
from robot_reset_rng import initial_action

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.join(HERE, "..")
sys.path.insert(0, os.path.join(HERE, "stubs"))


def test_emulated_draws_equal_the_replay_and_do_not_depend_on_the_mask():
    for seed, epoch in ((0, 0), (12345, 7), (2 ** 32 - 1, 2 ** 31)):
        full = pyemu_arm.sample(40, 6, seed, epoch)
        assert np.array_equal(full, np.stack([initial_action(seed, e, epoch, 6) for e in range(40)]))
        mask = np.arange(40) % 3 == 1
        part = pyemu_arm.sample(40, 6, seed, epoch, mask)
        assert np.array_equal(part[mask], full[mask]) and not part[~mask].any()
    # gym 0.15.3 Box.sample for the bounded float32 box [-1, 1]: low + (high - low) * u in float64, then float32
    # (the cast can reach the closed upper bound: u = 1 - 2^-53 gives 1.0f)
    u = np.array([0.0, 0.25, 1.0 - 2 ** -53])
    assert np.array_equal((-1.0 + 2.0 * u).astype(np.float32), np.float32([-1.0, -0.5, 1.0]))
    a = pyemu_arm.sample(4096, 5, 3, 1)
    assert (np.abs(a) <= 1).all() and abs(float(a.mean())) < 0.02 and a.std() > 0.55


def _tables():
    T = engine.ArmTables()
    T.narm = 6
    for j in range(6):
        T.arm_qpos_main[j], T.arm_qpos_solver[j], T.arm_act_main[j] = j, j, j
        T.lo_lim[j], T.hi_lim[j] = -6.0, 6.0
    T.grip_qpos_main, T.grip_qpos_solver, T.grip_act_main, T.grip_act_solver = 6, 6, 6, 0
    T.tcp_body, T.nweld, T.weld_mocap[0], T.weld_body[0] = 9, 1, 0, 9
    T.ndof, T.euler_index[0], T.euler_index[1], T.dof_joint[0], T.dof_joint[1] = 2, 0, 2, -1, 5
    T.align_axis = -1
    T.speed[0], T.speed[1], T.max_position_change, T.grip_lo, T.grip_hi, T.grip_half = 0.3, 1.0, 0.1, 0.0, 0.8, 0.4
    return T


def _phase(T, phases=engine.ARM_PRESOLVE, nenv=4, width=6, mask_len=None, main=(34, 7, 20, 0), solver=(8, 1, 12, 1)):
    L = engine.lib()
    m, s = engine.ArmSim(*main), engine.ArmSim(*solver)
    mask = ctypes.c_void_p(1) if mask_len is not None else None     # never read: the call is refused before any launch
    rc = L.rg_arm_phase(ctypes.byref(T), phases, nenv, ctypes.byref(m), ctypes.byref(s), None, width, mask, mask_len or 0, None)
    return rc, L.rg_last_error().decode()


@pytest.mark.skipif(not os.path.exists(engine.LIB_PATH), reason="needs the built library")
def test_abi_refuses_bad_tables_masks_and_widths():
    rc, msg = _phase(_tables())
    assert rc != 0 and "null" in msg                      # a well-formed call without rows gets as far as the pointers
    for field, idx, bad, what in (("arm_qpos_main", 2, 34, "arm_qpos_main"), ("arm_qpos_solver", 0, 8, "arm_qpos_solver"), ("arm_act_main", 5, 7, "arm_act_main"),
                                  ("tcp_body", None, 12, "tcp_body"), ("tcp_body", None, 0, "tcp_body"), ("weld_mocap", 0, 1, "weld_mocap"),
                                  ("weld_body", 0, -1, "weld_body"), ("grip_act_solver", None, 1, "gripper actuator"), ("grip_qpos_main", None, -1, "gripper qpos"),
                                  ("dof_joint", 1, 6, "dof_joint"), ("euler_index", 1, 0, "euler_index"), ("align_axis", None, 3, "align_axis")):
        T = _tables()
        if idx is None:
            setattr(T, field, bad)
        else:
            getattr(T, field)[idx] = bad
        rc, msg = _phase(T)
        assert rc != 0 and what in msg, (field, msg)
    rc, msg = _phase(_tables(), mask_len=3)
    assert rc != 0 and "mask" in msg
    for width in (5, 7):
        rc, msg = _phase(_tables(), width=width)
        assert rc != 0 and "action width" in msg
    rc, msg = _phase(_tables(), phases=engine.ARM_SYNC, width=5)     # phases without the action do not read its width
    assert rc != 0 and "null" in msg
    for phases in (0, 32):
        assert _phase(_tables(), phases=phases)[0] != 0
    L = engine.lib()
    assert L.rg_arm_sample_actions(4, 9, 0, 0, None, 0, ctypes.c_void_p(1), None) != 0 and "action_dim" in L.rg_last_error().decode()
    assert L.rg_arm_sample_actions(4, 6, 0, 0, ctypes.c_void_p(1), 5, ctypes.c_void_p(1), None) != 0 and "mask" in L.rg_last_error().decode()


def test_struct_mirrors_match_the_header(tmp_path):
    lines, expect = [], {}
    for cname, mirror in (("rg_arm_tables", engine.ArmTables), ("rg_arm_sim", engine.ArmSim)):
        lines.append(f'printf("sizeof {cname} %zu\\n", sizeof({cname}));')
        expect[f"sizeof {cname}"] = ctypes.sizeof(mirror)
        for f, _ in mirror._fields_:
            lines.append(f'printf("offsetof {cname}.{f} %zu\\n", offsetof({cname}, {f}));')
            expect[f"offsetof {cname}.{f}"] = getattr(mirror, f).offset
    for i, e in enumerate(("RG_ARM_SYNC", "RG_ARM_GRIP", "RG_ARM_SEAT", "RG_ARM_PRESOLVE", "RG_ARM_POSTSOLVE")):
        lines.append(f'printf("{e} %d\\n", (int){e});')
        expect[e] = getattr(engine, e[3:])
    src, exe = tmp_path / "arm_layout.c", tmp_path / "arm_layout"
    src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "robogym_b200.h"\nint main(void) {\n' + "\n".join(lines) + "\nreturn 0;\n}\n")
    subprocess.run([os.environ.get("CC", "cc"), "-std=c11", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout
    assert {k: int(v) for k, v in (line.rsplit(" ", 1) for line in out.splitlines())} == expect


def _golden():
    with gzip.open(os.path.join(HERE, "golden", "reference_robot_reset.json.gz"), "rt") as f:
        return json.load(f)["cases"]


MODES = {"TCP_ROLL_YAW": dict(dof_dims=("roll", "pitch")), "TCP_WRIST": dict(dof_dims=("pitch",), align_axis="pitch")}


def load(sim, st, rows=slice(None)):
    """a recorded simulation state (tools/make_robot_reset_golden.py) into rows of a BatchedSim or a stand-in"""
    t = sim.torch
    for name, key in (("qpos", "qpos"), ("qvel", "qvel"), ("ctrl", "ctrl"), ("pid", "pid"), ("qacc_warmstart", "warm"), ("mocap_pos", "mocap_pos"),
                      ("mocap_quat", "mocap_quat"), ("body_xpos", "body_xpos"), ("body_xquat", "body_xquat")):
        dst = getattr(sim, name, None)
        if dst is not None and key in st:
            dst[rows] = t.as_tensor(np.asarray(st[key]), dtype=dst.dtype).to(dst.device).reshape(dst.shape[1:])


def controller(c, make_sim):
    """both simulations of case `c` from make_sim(blob, nsub) and the controller of its mode"""
    from helpers import golden_model
    from robogym_b200.rearrange_arm import BatchedTcpArmController

    main = make_sim(golden_model("rearrange_blocks5_tcp", c["main_model"])[0], c["nsub_main"])
    solver = make_sim(golden_model("rearrange_solver_arm", c["solver_model"])[0], c["nsub_solver"])
    ctl = BatchedTcpArmController(main, solver, float(np.float32(0.1)), reset_controller_error=c["reset_controller_error"], **MODES[c["mode"]])
    return main, solver, ctl


def errors(sim, rec, n=None):
    """largest |difference| of qpos, ctrl and mocap pose against a recorded record (row 0, or every row)"""
    out = {}
    for k in ("qpos", "ctrl", "mocap_pos", "mocap_quat"):
        v = getattr(sim, k, None)
        if v is None or k not in rec:
            continue
        got = v.detach().cpu().numpy().astype(np.float64).reshape(v.shape[0], -1)
        out[k] = float(np.abs(got - np.asarray(rec[k])[None]).max())
    return out


def test_fixture_covers_the_cases():
    cases = _golden()
    assert {(c["mode"], c["reset_controller_error"], c["n_random_initial_steps"]) for c in cases} >= {
        ("TCP_ROLL_YAW", True, 10), ("TCP_ROLL_YAW", False, 10), ("TCP_WRIST", True, 10), ("TCP_ROLL_YAW", True, 1), ("TCP_ROLL_YAW", True, 0)}
    for c in cases:
        n = c["n_random_initial_steps"]
        assert c["action"] == initial_action(c["seed"], c["env"], c["epoch"], 3 + len(MODES[c["mode"]]["dof_dims"]) + 1).astype(np.float64).tolist()
        assert c["n_main_steps"] == (n + 100 if n >= 1 else 0)
        assert [a["step"] for a in c["after"]] == ([n] + [n + 10 * k for k in range(1, 11)] if n >= 1 else [])


@pytest.mark.parametrize("index", range(5))
def test_stand_ins_replay_the_reference_initialize_sim_state(index):
    """initialize_sim_state on the fp64 stand-ins from the state the reference had before _initialize_sim_state: both
    simulations land on the reference's state after it to 1e-9"""
    from oracle_generic_sim import OracleGenericSim

    c = _golden()[index]
    main, solver, ctl = controller(c, lambda blob, nsub: OracleGenericSim(blob, 1, nsub))
    load(main, c["init_before"]["main"]); load(solver, c["init_before"]["solver"])
    ctl.initialize_sim_state()
    for sim, key in ((main, "main"), (solver, "solver")):
        e = errors(sim, c["init_after"][key])
        assert max(e.values()) < 1e-9, (key, e)
    assert not main.qvel.any() and not solver.qvel.any()


@pytest.mark.parametrize("index", range(5))
def test_stand_ins_replay_the_reference_random_initial_position(index):
    """hold_initial_action with the replayed draw on the fp64 stand-ins, from the state the reference had before
    _randomize_robot_initial_position: the main arm after the held steps, and both simulations after the last zero-action
    step, to 1e-9"""
    import torch

    from oracle_generic_sim import OracleGenericSim

    c = _golden()[index]
    n = c["n_random_initial_steps"]
    a = torch.tensor([c["action"]], dtype=torch.float32)
    main, solver, ctl = controller(c, lambda blob, nsub: OracleGenericSim(blob, 1, nsub))
    load(main, c["before"]["main"]); load(solver, c["before"]["solver"])
    if n < 1:
        ctl.hold_initial_action(a, None, n)
        for sim, key in ((main, "main"), (solver, "solver")):
            assert max(errors(sim, c["before"][key]).values()) == 0
        return
    for _ in range(n):                              # the held steps alone: hold_initial_action's first loop
        ctl._step(a, None, 1, False)
    assert errors(main, c["after"][0]["main"])["qpos"] < 1e-9
    load(main, c["before"]["main"]); load(solver, c["before"]["solver"])
    ctl.hold_initial_action(a, None, n)
    for sim, key in ((main, "main"), (solver, "solver")):
        e = errors(sim, c["after"][-1][key])
        assert max(e.values()) < 1e-9, (key, e)
    assert int(main.warn.max()) == 0


def test_stand_ins_refuse_masks_and_device_draws():
    from oracle_generic_sim import OracleGenericSim

    c = _golden()[0]
    main, solver, ctl = controller(c, lambda blob, nsub: OracleGenericSim(blob, 2, nsub))
    load(main, c["init_before"]["main"]); load(solver, c["init_before"]["solver"])
    before = main.qpos.clone()
    with pytest.raises(ValueError):
        ctl.initialize_sim_state(np.array([True, False]))
    assert main.qpos.equal(before)                  # refused before anything was written
    with pytest.raises(ValueError):
        ctl.sample_initial_action(1, 0)
    with pytest.raises(ValueError):
        ctl.hold_initial_action(main.qpos[:, :6].float(), np.ones(2, bool))
