"""Shared test helpers: oracle rollouts that produce teacher-forcing states."""
import numpy as np

from oracle import pyoracle


def oracle_pair(blob):
    om = pyoracle.OracleModel(blob)
    return om, pyoracle.OracleData(om)


def rollout_states(blob, n_states, seed=1, settle=20, nsub=10, action_scale=0.3):
    """Roll the oracle with smoothed random position targets; return (states, after, model dims).

    states[k] = (qpos, qvel, ctrl, pid, warmstart) BEFORE env-step k, after[k] = (qpos, qvel, ncon) AFTER it."""
    om, d = oracle_pair(blob)
    nu = om.dim("nu")
    cr = om.field("actuator_ctrlrange").reshape(-1, 2)
    rng = np.random.RandomState(seed)
    d.ctrl[:] = cr.mean(1)
    for _ in range(settle):
        d.env_step(nsub)
    states, after = [], []
    for _ in range(n_states):
        a = rng.uniform(-1, 1, nu)
        d.ctrl[:] = np.clip(d.ctrl + action_scale * a * (cr[:, 1] - cr[:, 0]) / 2, cr[:, 0], cr[:, 1])
        states.append((d.qpos.copy(), d.qvel.copy(), d.ctrl.copy(), d.userdata[:3 * nu].copy(), d.qacc_warmstart.copy()))
        d.env_step(nsub)
        after.append((d.qpos.copy(), d.qvel.copy(), int(d.ncon[0])))
    return states, after, om


def control_matrix(m):
    """P with ctrl = P qpos for position actuators (joint -> 1, fixed tendon -> its joint coefficients):
    hand_interface.py:245-266 read off the compiled transmissions."""
    nu = m["nu"]
    P = np.zeros((nu, m["nq"]))
    for i in range(nu):
        tid = int(m["actuator_trnid"][i])
        if m["actuator_trntype"][i] == 0:
            P[i, m["jnt_qposadr"][tid]] = 1.0
        else:
            for w in range(m["tendon_adr"][tid], m["tendon_adr"][tid] + m["tendon_num"][tid]):
                P[i, m["jnt_qposadr"][int(m["wrap_objid"][w])]] = m["wrap_prm"][w]
    return P


def contract_states(blob, seeds, per_seed, settle=20, nsub=10):
    """SURVEY.md 8(d) cfg 2 workload on the oracle: per seed, settle 20 env-steps, jitter the cube position (N(0, 0.005^2))
    and draw a uniform random cube orientation, then full-range relative actions a ~ U(-1,1): ctrl = clip(P qpos + a*range/2)
    (robogym/robot/robot_interface.py:247-278).  Returns teacher-forcing states and the oracle's result after each env-step."""
    from robogym_b200 import modelblob

    m = modelblob.unpack(blob)
    P = control_matrix(m)
    states, after, om = [], [], None
    for seed in seeds:
        om, d = oracle_pair(blob)
        nu = om.dim("nu")
        cr = om.field("actuator_ctrlrange").reshape(-1, 2)
        rng = np.random.RandomState(seed)
        d.ctrl[:] = cr.mean(1)
        for _ in range(settle):
            d.env_step(nsub)
        d.qpos[0:3] += 0.005 * rng.randn(3)
        q = rng.randn(4)
        d.qpos[3:7] = q / np.linalg.norm(q)
        for _ in range(per_seed):
            a = rng.uniform(-1, 1, nu)
            d.ctrl[:] = np.clip(P @ d.qpos + a * (cr[:, 1] - cr[:, 0]) / 2, cr[:, 0], cr[:, 1])
            states.append((d.qpos.copy(), d.qvel.copy(), d.ctrl.copy(), d.userdata[:3 * nu].copy(), d.qacc_warmstart.copy()))
            d.env_step(nsub)
            after.append((d.qpos.copy(), d.qvel.copy(), int(d.ncon[0])))
    return states, after, om


def full_cube_states(blob, n=16):
    """dactyl/full_perpendicular on the oracle: 5 settling env-steps at mid-range targets, then n env-steps of smoothed random
    targets.  Returns (states, after) like rollout_states."""
    om, d = oracle_pair(blob)
    nu = om.dim("nu")
    cr = om.field("actuator_ctrlrange").reshape(-1, 2)
    rng = np.random.RandomState(3)
    d.ctrl[:] = cr.mean(1)
    for _ in range(5):
        d.env_step(10)
    states, after = [], []
    for _ in range(n):
        a = rng.uniform(-1, 1, nu)
        d.ctrl[:] = np.clip(d.ctrl + 0.3 * a * (cr[:, 1] - cr[:, 0]) / 2, cr[:, 0], cr[:, 1])
        states.append((d.qpos.copy(), d.qvel.copy(), d.ctrl.copy(), d.userdata[:3 * nu].copy(), d.qacc_warmstart.copy()))
        d.env_step(10)
        after.append((d.qpos.copy(), d.qvel.copy(), int(d.ncon[0])))
    return states, after


def live_indices(om, names):
    """qpos / qvel indices excluding the free-falling, collision-less target cube
    (robogym/envs/dactyl/locked.py:89-96; masked from observations, observation/mujoco.py:46,60)."""
    jq, jv = om.field("jnt_qposadr"), om.field("jnt_dofadr")
    jt = om.field("jnt_type")
    iq, iv = [], []
    for j, name in enumerate(names["joint"]):
        if name.startswith("target:"):
            continue
        nq, nv = {0: (7, 6), 1: (4, 3), 2: (1, 1), 3: (1, 1)}[int(jt[j])]
        iq += list(range(jq[j], jq[j] + nq))
        iv += list(range(jv[j], jv[j] + nv))
    return iq, iv


def reference_golden(name):
    """tests/golden/reference_<name>.json.gz: what the original robogym code returned (tools/make_reference_goldens.py)"""
    import gzip
    import json
    import os

    with gzip.open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_%s.json.gz" % name), "rt") as f:
        return json.load(f)


def golden_model(asset, overrides):
    """(blob, unpacked model, names) of a committed asset with the recorded differences of the reference environment's own
    compiled model written over it"""
    import os

    from robogym_b200 import modelblob

    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "robogym_b200", "assets", asset + ".rgm"), "rb") as f:
        base = f.read()
    m, names = modelblob.unpack(base), modelblob.unpack_names(base)
    for k, v in overrides.items():
        m[k][...] = np.asarray(v, dtype=m[k].dtype)
    return modelblob.pack(m, names), m, names


def step_errors(q_new, v_new, after, iq, iv):
    eq = np.array([np.abs(q_new[k][iq] - after[k][0][iq]).max() for k in range(len(after))])
    ev = np.array([np.abs(v_new[k][iv] - after[k][1][iv]).max() for k in range(len(after))])
    return eq, ev
