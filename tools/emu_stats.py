"""Algorithmic counters of the kernel logic (CPU emulation build with -DRG_STATS) on the bench workload.

Tells where the per-substep work goes (Newton iterations, refactorisations, line-search evaluations, MPR pairs,
support calls, climb steps) without a GPU.  Development tool: python tools/emu_stats.py [nenv] [env_steps]"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "emu"))
EMU = os.path.join(ROOT, "tests", "emu")
OUT = os.path.join(EMU, "_build", "librg_emu_stats.so")


def build():
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    subprocess.check_call(["g++", "-O2", "-fPIC", "-std=c++17", "-ffp-contract=off", "-DRG_STATS", *os.environ.get("RG_EMU_FLAGS", "").split(), "-shared", "-o", OUT, os.path.join(EMU, "rg_emu.cpp")])


def main():
    nenv = int(sys.argv[1]) if len(sys.argv) > 1 else 16
    steps = int(sys.argv[2]) if len(sys.argv) > 2 else 20
    build()
    import pyemu
    pyemu._LIB = OUT
    pyemu.subprocess = type("S", (), {"check_call": staticmethod(lambda *a, **k: 0)})
    from robogym_b200 import modelblob
    blob = open(os.path.join(ROOT, "robogym_b200", "assets", "dactyl_locked.rgm"), "rb").read()
    names = json.load(open(os.path.join(ROOT, "robogym_b200", "assets", "dactyl_locked.names.json")))
    m = modelblob.unpack(blob)
    dims = {k: m[k] for k in modelblob.DIMS}
    e = pyemu.EmuBatch(blob, dims, nenv)
    L = pyemu.lib()
    L.rge_stats.argtypes = [ctypes.c_void_p]
    nu = m["nu"]
    cr = m["actuator_ctrlrange"].reshape(-1, 2)
    # control = P qpos_hand (relative actions, robot_interface.py:247-278)
    P = np.zeros((nu, m["nq"]))
    for i in range(nu):
        tid = int(m["actuator_trnid"][i])
        if m["actuator_trntype"][i] == 0:
            P[i, m["jnt_qposadr"][tid]] = 1
        else:
            for w in range(m["tendon_adr"][tid], m["tendon_adr"][tid] + m["tendon_num"][tid]):
                P[i, m["jnt_qposadr"][int(m["wrap_objid"][w])]] = m["wrap_prm"][w]
    rng = np.random.RandomState(0)
    e.qpos[:] = m["qpos0"]
    e.ctrl[:] = cr.mean(1)
    for _ in range(20):
        e.step(10, 1)
    e.qpos[:, 0:3] += 0.005 * rng.randn(nenv, 3)
    q = rng.randn(nenv, 4)
    e.qpos[:, 3:7] = q / np.linalg.norm(q, axis=1, keepdims=True)
    buf = (ctypes.c_longlong * 192)()
    L.rge_stats(buf)
    base = np.array(buf[:])
    for _ in range(steps):
        a = rng.uniform(-1, 1, (nenv, nu))
        e.ctrl[:] = np.clip(e.qpos @ P.T + a * (cr[:, 1] - cr[:, 0]) / 2, cr[:, 0], cr[:, 1])
        e.step(10, 1)
    L.rge_stats(buf)
    s = np.array(buf[:]) - base
    x = s[136:152]
    fw = x[0]
    print("forwards", fw, "on palm", float((e.site_xpos[:, names["site"].index("cube:center"), 2] > 0.04).mean()), "warn", int(e.warn.max()))
    lab = ["forwards", "newton iterations", "refactorisations", "line-search evals", "mpr batch trips", "broad survivors", "obb survivors", "contacts", "rows(el)", "mpr iterations",
           "exit:gradient", "exit:alpha", "exit:improvement"]
    for k, l in enumerate(lab):
        print("%-22s %10d  per forward %.3f" % (l, x[k], x[k] / fw))
    print("support calls per forward %.2f, hull vertices visited %.2f, mpr pairs %.2f (hits %.2f)" % (s[0] / fw, s[1] / fw, s[2] / fw, s[3] / fw))
    h = s[8:136].reshape(2, 64)
    print("mpr iteration histogram (miss):", h[0][:24])
    print("mpr iteration histogram (hit): ", h[1][:40])
    ih = s[152:168]
    fh = s[168:184]
    print("rows whose active state flipped between consecutive refactorisations of a solve, histogram:", fh, " single-row flips/refactor %.2f, contact-edge flips/refactor %.2f" % (x[13] / max(x[15], 1), x[14] / max(x[15], 1)))
    print("newton iterations per solve, histogram:", ih[:12], " P(>=5) = %.3f, P(>=6) = %.3f" % (ih[5:].sum() / ih.sum(), ih[6:].sum() / ih.sum()))


if __name__ == "__main__":
    main()
