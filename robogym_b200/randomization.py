"""Per-environment domain randomisation sampled on the device (SURVEY.md 8(f) row 2, parameter set of 5.6).

The reference randomises by wrapping ONE env in a stack of gym wrappers that write `sim.model.<array>` before every
episode and call `mj_setConst` in the following reset (robogym/envs/dactyl/locked.py:263-277 lists the stack).  Here
the same distributions are drawn for `n` environments at once as `[n, count]` tensors and handed to the engine's
per-environment parameter rows (`BatchedSim.set_param` -> `rg_batch_bind_param`), including the constants that
`mj_setConst` would recompute from a changed inertia (`BatchedConstants`).

| sampler                | reference wrapper (robogym/wrappers/...)                                   |
|------------------------|-----------------------------------------------------------------------------|
| body_inertia           | randomizations.RandomizedBodyInertiaWrapper (72-92): x U(0.5, 1.5) per body  |
| geom_friction          | dactyl RandomizedRobotFrictionWrapper / cube.RandomizedCubeFrictionWrapper (95-173): one multiplier per friction column, robot and cube geoms separately |
| opt_gravity            | randomizations.RandomizedGravityWrapper (176-191): + 0.4 N(0, 1) per axis    |
| dof_damping            | dactyl.RandomizedRobotDampingWrapper (dactyl.py:153-160): x logU(1/1.5, 1.5) per robot dof |
| actuator Kp            | dactyl.RandomizedRobotKpWrapper (dactyl.py:163-170): x logU(0.5, 2) per robot actuator |
| jnt_range + ctrlrange  | randomizations.RandomizedJointLimitWrapper (593-670)                         |
| tendon_range           | randomizations.RandomizedTendonRangeWrapper (673-717)                        |
| cube size              | cube.RandomizedCubeSizeWrapper (cube.py:12-52): x U(0.95, 1.05)              |
| full cube size         | parametric.RandomizedPerpendicularCubeSizeWrapper (parametric.py:24-38): cubelet body_pos, named cubelet geom_rbound, cubelet hull mesh_scale x U(0.95, 1.05), then set_const on the device (FullCubeRandomizer(cube_size_range=...)) |
| phasespace sites       | dactyl.RandomizedPhasespaceFingersWrapper (dactyl.py:14-60): + N(0, sigma) per site |
| timestep (per step)    | randomizations.RandomizedTimestepWrapper (194-311)                           |
| wind (per step)        | cube.RandomizedWindWrapper (cube.py:56-85)                                   |
"""
import math

import numpy as np

from . import mjcf

JNT_FREE, JNT_BALL = 0, 1


class BatchedConstants:
    """mj_setConst for a batch of body_inertia rows: dof_invweight0, body_invweight0, tendon_invweight0, opt_meaninertia.

    At qpos0 the mass matrix is affine in the principal inertias: M = M_rest + sum_b sum_k I[b,k] w[b,k] w[b,k]^T with
    w[b,k] = (k-th principal axis of body b in the world)^T Jrot_b, so a batch of inertias needs one einsum, one batched
    inverse and three contractions (same formulas as mjcf.set_const, which is the single-model host version)."""

    def __init__(self, m, torch, device, dtype):
        self.torch = torch
        nb, nv = m["nbody"], m["nv"]
        M, (xpos, xquat, jaxis, janchor) = mjcf.mass_matrix(m, m["qpos0"])
        W = np.zeros((nb, 3, nv))
        JP = np.zeros((nb, 3, nv))
        JR = np.zeros((nb, 3, nv))
        inertia = m["body_inertia"].reshape(-1, 3).astype(float)
        Mrest = M.copy()
        for b in range(1, nb):
            R = mjcf.quat2mat(mjcf.quat_mul(xquat[b], m["body_iquat"].reshape(-1, 4)[b]))
            com = xpos[b] + mjcf.rot_vec(xquat[b], m["body_ipos"].reshape(-1, 3)[b])
            jp, jr = mjcf.body_jacobian(m, xpos, xquat, jaxis, janchor, b, com)
            JP[b], JR[b] = jp, jr
            W[b] = R.T @ jr
            for k in range(3):
                Mrest -= inertia[b, k] * np.outer(W[b, k], W[b, k])
        t = lambda a: torch.as_tensor(np.asarray(a), dtype=dtype, device=device)
        self.Mrest, self.W, self.JP, self.JR = t(Mrest), t(W), t(JP), t(JR)
        # averaging matrix for ball / free-joint dof triplets
        A = np.eye(nv)
        for j in range(m["njnt"]):
            ty, a = int(m["jnt_type"][j]), int(m["jnt_dofadr"][j])
            groups = [(a, a + 3)] if ty == JNT_BALL else ([(a, a + 3), (a + 3, a + 6)] if ty == JNT_FREE else [])
            for lo, hi in groups:
                A[lo:hi, :] = 0
                A[lo:hi, lo:hi] = 1.0 / 3.0
        self.avg = t(A)
        self.movable = t((np.asarray(m["body_weldid"]) != 0).astype(float))
        self.movable[0] = 0
        # tendon Jacobians at qpos0 (fixed tendons from their coefficients, spatial ones from the compile-time geometry)
        nt = m["ntendon"]
        Jt = np.zeros((nt, nv))
        if nt:
            _, Jsp = mjcf.tendon_eval(m, m["qpos0"])
            for i in range(nt):
                if mjcf.tendon_length_fixed(m, m["qpos0"], i) is not None:
                    for w in range(m["tendon_adr"][i], m["tendon_adr"][i] + m["tendon_num"][i]):
                        Jt[i, m["jnt_dofadr"][m["wrap_objid"][w]]] += m["wrap_prm"][w]
                else:
                    Jt[i] = Jsp[i]
        self.Jt = t(Jt)

    def derive(self, body_inertia):
        """body_inertia [n, nbody*3] -> dict of [n, count] rows."""
        torch = self.torch
        n = body_inertia.shape[0]
        I = body_inertia.reshape(n, -1, 3).to(self.W.dtype)
        M = self.Mrest.unsqueeze(0) + torch.einsum("ebk,bkm,bkn->emn", I, self.W, self.W)
        Minv = torch.linalg.inv(M)
        diag = torch.diagonal(Minv, dim1=1, dim2=2)
        out = {}
        out["opt_meaninertia"] = torch.diagonal(M, dim1=1, dim2=2).mean(dim=1, keepdim=True)
        out["dof_invweight0"] = diag @ self.avg.T
        tp = torch.einsum("bim,emn,bin->eb", self.JP, Minv, self.JP) / 3.0
        tr = torch.einsum("bim,emn,bin->eb", self.JR, Minv, self.JR) / 3.0
        biw = torch.stack([torch.clamp(tp, min=mjcf.MINVAL), torch.clamp(tr, min=mjcf.MINVAL)], dim=2) * self.movable.view(1, -1, 1)
        out["body_invweight0"] = biw.reshape(n, -1)
        if self.Jt.shape[0]:
            out["tendon_invweight0"] = torch.clamp(torch.einsum("tm,emn,tn->et", self.Jt, Minv, self.Jt), min=mjcf.MINVAL)
        return out


def joint_limit_rule(torch, orig, noise, relative_std=0.15):
    """RandomizedJointLimitWrapper._set_field (randomizations.py:615-640) on [n, njoint, 2] tensors:
    each bound moves by N(0,1) * relative_std * width, a bound that sits at 0 never crosses 0, width >= 0.1 %."""
    lo0, hi0 = orig[..., 0], orig[..., 1]
    width = hi0 - lo0
    d = noise * (width * relative_std).unsqueeze(-1)
    minw = width * 0.001
    # case A: low == 0 and high > 0
    loA = torch.clamp(lo0 + d[..., 0], min=0.0)
    hiA = torch.maximum(loA + minw, hi0 + d[..., 1])
    # case B: low < 0 and high == 0
    hiB = torch.clamp(hi0 + d[..., 1], max=0.0)
    loB = torch.minimum(hiB - minw, lo0 + d[..., 0])
    # otherwise
    loC = lo0 + d[..., 0]
    hiC = torch.maximum(loC + minw, hi0 + d[..., 1])
    A = (lo0 == 0.0) & (hi0 > 0)
    B = (lo0 < 0) & (hi0 == 0.0)
    lo = torch.where(A, loA, torch.where(B, loB, loC))
    hi = torch.where(A, hiA, torch.where(B, hiB, hiC))
    return torch.stack([lo, hi], dim=-1)


def tendon_range_rule(torch, orig, noise, relative_std=0.15):
    """RandomizedTendonRangeWrapper._set_field (randomizations.py:687-714)."""
    width = orig[..., 1] - orig[..., 0]
    d = noise * (width * relative_std).unsqueeze(-1)
    lo = torch.clamp(orig[..., 0] + d[..., 0], min=0.0)
    hi = torch.maximum(lo + width * 0.001, orig[..., 1] + d[..., 1])
    return torch.stack([lo, hi], dim=-1)


# The per-episode rules sample() draws.  The per-step rules (RandomizedTimestepWrapper, cube.RandomizedWindWrapper) are run by the
# environments through timestep_state / next_timestep and wind_state / next_wind, and are not listed.  "set_constants" is
# CubeEnv._reset's set_constants() (cube_env.py:343-349): the constants mj_setConst derives from the drawn inertias.
LOCKED_RULES = ("body_inertia", "robot_friction", "cube_friction", "gravity", "joint_limit", "tendon_range", "phasespace",
                "robot_damping", "robot_kp", "cube_size", "set_constants")
# dactyl/reach's stack (reach.py:226-240): RandomizedActionLatency and the observation noise live in the environment.  Its reset
# never calls set_constants() (RobotEnv._reset is `pass`), so the derived constants keep the model's values.
REACH_RULES = ("body_inertia", "robot_friction", "gravity", "phasespace", "robot_damping", "robot_kp")
CUBE_RULES = ("cube_friction", "cube_size")


class LockedRandomizer:
    """The randomisation stack of dactyl/locked (locked.py:263-277), drawn for n environments at once.  `rules` names the
    wrappers of another dactyl stack (REACH_RULES); the cube's rules are skipped on a model without a cube."""

    EPISODE_PARAMS = ("body_inertia", "geom_friction", "opt_gravity", "dof_damping", "actuator_gainprm", "jnt_range",
                      "actuator_ctrlrange", "tendon_range", "geom_size", "geom_rbound", "geom_aabb", "site_pos",
                      "dof_invweight0", "body_invweight0", "tendon_invweight0", "opt_meaninertia")

    def __init__(self, m, names, rand, torch, device, dtype, hand_prefix="robot0:", cube_prefix="cube:", rules=LOCKED_RULES):
        self.torch, self.rand, self.m = torch, rand, m
        self.device, self.dtype = device, dtype
        t = lambda a, dt=dtype: torch.as_tensor(np.asarray(a), dtype=dt, device=device)
        self.orig = {k: t(m[k]).reshape(1, -1) for k in self.EPISODE_PARAMS if k in m}
        gn, jn, an, sn = names["geom"], names["joint"], names["actuator"], names["site"]
        idx = lambda lst, pred: t([i for i, nme in enumerate(lst) if nme is not None and pred(nme)], torch.long)
        self.robot_geoms = idx(gn, lambda s: s.startswith(hand_prefix))
        self.cube_geoms = idx(gn, lambda s: s.startswith(cube_prefix))
        robot_j = [j for j, nme in enumerate(jn) if nme is not None and nme.startswith(hand_prefix)]
        self.robot_joints = t(robot_j, torch.long)
        self.robot_dofs = t([d for d in range(m["nv"]) if int(m["dof_jntid"][d]) in set(robot_j)], torch.long)
        self.robot_acts = idx(an, lambda s: s.startswith(hand_prefix))
        self.cube_middle = gn.index(cube_prefix + "middle") if cube_prefix + "middle" in gn else None   # the locked cube is one box geom
        from .batched_env import FINGERTIP_SITES, REFERENCE_SITES
        self.tip_sites = t([sn.index(hand_prefix + s) for s in FINGERTIP_SITES], torch.long)
        self.ref_sites = t([sn.index(hand_prefix + s) for s in REFERENCE_SITES], torch.long)
        # joint -> actuator coupling of RandomizedJointLimitWrapper (randomizations.py:645-664)
        self.act_of_joint = []
        for j in robot_j:
            an_j = jn[j].replace(":", ":A_")
            if an_j not in an:
                continue
            other = jn.index(jn[j].replace("FJ1", "FJ0")) if an_j.endswith("FJ1") else -1
            self.act_of_joint.append((j, an.index(an_j), other))
        # the wrapper perturbs actuated_joint_range (robogym/utils/dactyl_utils.py:4-14): jnt_range clipped to the
        # control range of the actuator that drives the joint -- for ALL joints (its default joint_names)
        jr0 = np.array(m["jnt_range"], dtype=float).reshape(-1, 2).copy()
        cr0 = np.asarray(m["actuator_ctrlrange"], dtype=float).reshape(-1, 2)
        for a, nme in enumerate(an):
            j = jn.index(nme.replace("A_", ""))
            jr0[j, 0] = max(jr0[j, 0], cr0[a, 0])
            jr0[j, 1] = max(jr0[j, 0], min(jr0[j, 1], cr0[a, 1]))
        self.joint_limits0 = t(jr0).unsqueeze(0)
        self.constants = BatchedConstants(m, torch, device, dtype)
        self.timestep0 = float(m["opt_timestep"][0])
        self.nsub_dt = None
        has_cube = cube_prefix + "middle" in names["body"]
        self.rules = tuple(r for r in rules if has_cube or r not in CUBE_RULES)
        if has_cube:
            self.cube_body = names["body"].index(cube_prefix + "middle")
            self.cube_mass = float(m["body_mass"][self.cube_body])

    def _logu(self, lo, hi, n, k):
        return self.torch.exp(self.rand.uniform(math.log(lo), math.log(hi), n, k))

    # ------------------------------------------------------------ per-episode parameters
    def sample(self, n, noises=None):
        """dict name -> [n, count] rows.  `noises` (tests) overrides individual draws by name."""
        torch, m, o = self.torch, self.m, self.orig
        nz = noises or {}
        draw = lambda key, fn: nz[key].to(self.dtype) if key in nz else fn()
        out = {}
        on = self.rules
        nb = m["nbody"]
        if "body_inertia" in on:
            out["body_inertia"] = (o["body_inertia"].reshape(1, nb, 3) * draw("inertia", lambda: self.rand.uniform(0.5, 1.5, n, nb)).unsqueeze(2)).reshape(n, -1)
        if "robot_friction" in on or "cube_friction" in on:
            fr = o["geom_friction"].reshape(1, -1, 3).repeat(n, 1, 1)
            if "robot_friction" in on:
                rm = draw("robot_friction", lambda: torch.stack([self.rand.uniform(a, b, n, 1)[:, 0] for a, b in ((0.7, 1.3), (0.5, 1.5), (0.5, 1.5))], dim=1))
                fr[:, self.robot_geoms] = fr[:, self.robot_geoms] * rm.unsqueeze(1)
            if "cube_friction" in on:
                cm = draw("cube_friction", lambda: torch.stack([self.rand.uniform(a, b, n, 1)[:, 0] for a, b in ((0.5, 1.5), (0.2, 5.0), (0.2, 5.0))], dim=1))
                fr[:, self.cube_geoms] = fr[:, self.cube_geoms] * cm.unsqueeze(1)
            out["geom_friction"] = fr.reshape(n, -1)
        if "gravity" in on:
            out["opt_gravity"] = o["opt_gravity"] + 0.4 * draw("gravity", lambda: self.rand.randn(n, 3))
        if "robot_damping" in on:
            damp = o["dof_damping"].repeat(n, 1)
            damp[:, self.robot_dofs] = damp[:, self.robot_dofs] * draw("damping", lambda: self._logu(1 / 1.5, 1.5, n, int(self.robot_dofs.numel())))
            out["dof_damping"] = damp
        if "robot_kp" in on:
            gain = o["actuator_gainprm"].reshape(1, m["nu"], -1).repeat(n, 1, 1)
            gain[:, self.robot_acts, 0] = gain[:, self.robot_acts, 0] * draw("kp", lambda: self._logu(0.5, 2.0, n, int(self.robot_acts.numel())))
            out["actuator_gainprm"] = gain.reshape(n, -1)
        if "joint_limit" in on:
            # joint limits (robot joints) and the control ranges that follow them
            nj = m["njnt"]
            jr = joint_limit_rule(torch, self.joint_limits0.repeat(n, 1, 1), draw("joint_limit", lambda: self.rand.randn(n, nj * 2).reshape(n, nj, 2)))
            out["jnt_range"] = jr.reshape(n, -1)
            cr = o["actuator_ctrlrange"].reshape(1, -1, 2).repeat(n, 1, 1)
            for j, a, other in self.act_of_joint:
                if other >= 0:
                    cr[:, a, 0] = torch.minimum(jr[:, other, 0], jr[:, j, 0])
                    cr[:, a, 1] = jr[:, other, 1] + jr[:, j, 1]
                else:
                    cr[:, a] = jr[:, j]
            out["actuator_ctrlrange"] = cr.reshape(n, -1)
        if "tendon_range" in on:
            nt = m["ntendon"]
            out["tendon_range"] = tendon_range_rule(torch, o["tendon_range"].reshape(1, nt, 2).repeat(n, 1, 1),
                                                    draw("tendon_range", lambda: self.rand.randn(n, nt * 2).reshape(n, nt, 2))).reshape(n, -1)
        # cube size: geom_size of cube:middle and the bounds the broad phase derives from it
        if "cube_size" in on and self.cube_middle is not None:
            scale = draw("cube_size", lambda: self.rand.uniform(0.95, 1.05, n, 1))
            gs = o["geom_size"].reshape(1, -1, 3).repeat(n, 1, 1)
            gs[:, self.cube_middle] = gs[:, self.cube_middle] * scale
            out["geom_size"] = gs.reshape(n, -1)
            rb = o["geom_rbound"].repeat(n, 1)
            rb[:, self.cube_middle] = gs[:, self.cube_middle].norm(dim=1)
            out["geom_rbound"] = rb
            ab = o["geom_aabb"].reshape(1, -1, 6).repeat(n, 1, 1)
            ab[:, self.cube_middle, 3:6] = gs[:, self.cube_middle]
            out["geom_aabb"] = ab.reshape(n, -1)
        self._extra_rules(n, draw, out)
        if "phasespace" in on:
            # phasespace marker sites
            sp = o["site_pos"].reshape(1, -1, 3).repeat(n, 1, 1)
            sp[:, self.tip_sites] += 0.003 * draw("tip_noise", lambda: self.rand.randn(n, 15).reshape(n, 5, 3))
            sp[:, self.ref_sites] += 0.001 * draw("ref_noise", lambda: self.rand.randn(n, 9).reshape(n, 3, 3))
            out["site_pos"] = sp.reshape(n, -1)
        if "set_constants" in on and "body_inertia" in out:
            out.update(self.constants.derive(out["body_inertia"]))
        return out

    def _extra_rules(self, n, draw, out):
        """hook for the scenes that add wrappers to the locked stack"""

    def apply(self, sim, params, idx=None):
        """Write sampled rows into the simulator's per-environment parameter tensors (all rows, or rows `idx`)."""
        for name, rows in params.items():
            cur = getattr(sim, "_params", {}).get(name)
            if cur is None:
                full = self.orig[name].repeat(sim.nenv, 1).to(rows.dtype) if name in self.orig else None
                if idx is None:
                    full = rows
                else:
                    full[idx] = rows
                sim.set_param(name, full)
            else:
                sim.set_param(name, rows, idx=idx)     # through set_param: world-attached body / geom / site rows keep the fp32 world shift

    # ------------------------------------------------------------ per-step randomisation
    def timestep_state(self, n):
        """RandomizedTimestepWrapper._set_field (randomizations.py:242-262): per-episode lambdas, side and flip probabilities."""
        torch = self.torch
        side = torch.where(self.rand.uniform(0.0, 1.0, n, 1)[:, 0] < 0.5, -torch.ones(n, dtype=self.dtype, device=self.device), torch.ones(n, dtype=self.dtype, device=self.device))
        return dict(pos_lambda=self.rand.uniform(1250.0, 10000.0, n, 1)[:, 0], neg_lambda=self.rand.uniform(1250.0, 10000.0, n, 1)[:, 0], side=side,
                    p_flip_pos=self.rand.uniform(0.0, 1.0, n, 1)[:, 0], p_flip_neg=self.rand.uniform(0.0, 1.0, n, 1)[:, 0])

    def next_timestep(self, st):
        """RandomizedTimestepWrapper.step (randomizations.py:270-311) -> per-env opt.timestep for the next env-step."""
        torch = self.torch
        n = st["side"].shape[0]
        u = self.rand.uniform(0.0, 1.0, n, 1)[:, 0]
        flip = torch.where(st["side"] > 0, u > st["p_flip_pos"], u > st["p_flip_neg"])
        st["side"] = torch.where(flip, -st["side"], st["side"])
        lam = torch.where(st["side"] > 0, st["pos_lambda"], st["neg_lambda"])
        e = -torch.log(torch.clamp(1.0 - self.rand.uniform(0.0, 1.0, n, 1)[:, 0], min=1e-12)) / lam      # Exp(1/lambda)
        t0 = self.timestep0
        neg = st["side"] < 0
        frac = e / t0
        e = torch.where(neg, torch.clamp(t0 * (frac / (1 + frac)), 0.0, t0 / 2), e)
        return t0 + st["side"] * e

    def wind_state(self, n, env_step_dt, max_mean_time_between=0.8):
        """RandomizedWindWrapper.reset (cube.py:62-73): per-episode hit probability, log-uniform."""
        hi = env_step_dt / max_mean_time_between
        return dict(hit_prob=self._logu(0.01 * hi, hi, n, 1)[:, 0])

    def next_wind(self, st, xfrc, force_std=1.0):
        """RandomizedWindWrapper.step (cube.py:75-85) on the [nenv, nbody, 6] xfrc_applied tensor, in place."""
        n = xfrc.shape[0]
        f = xfrc[:, self.cube_body, :3]
        f *= 0.99
        hit = self.rand.uniform(0.0, 1.0, n, 1)[:, 0] < st["hit_prob"]
        gust = self.rand.randn(n, 3) * self.cube_mass * force_std
        xfrc[:, self.cube_body, :3] = self.torch.where(hit.unsqueeze(1), gust.to(xfrc.dtype), f)
        return xfrc


class FullCubeRandomizer(LockedRandomizer):
    """The randomisation stack of dactyl/full_perpendicular (robogym/envs/dactyl/full_perpendicular.py:425-440): the locked stack
    (body inertias, robot / cube friction, gravity, robot damping, Kp, joint limits, tendon ranges, phasespace marker offsets, per-step
    timestep, wind on `cube:middle`) plus `RandomizedFaceDampingWrapper` (wrappers/face.py:4-9: the damping of the cube's face-driver and
    cubelet joints times a log-uniform factor in [1/3, 3] per dof).  Cube friction applies to every named cube geom (25 cubelets + the core sphere)
    (`RandomizedCubeFrictionWrapper` takes every geom whose name starts with "cube:").

    `cube_size_range=(lo, hi)` adds `RandomizedPerpendicularCubeSizeWrapper` (wrappers/parametric.py:24-38) with the edits of its
    `PerpendicularCubeSizeModifier` (envs/dactyl/common/mujoco_modifiers.py:8-66): one s ~ U(lo, hi) per environment, drawn after every
    other draw, scales the original `body_pos` of the 26 `cube:cubelet:*` bodies, the `geom_rbound` of the 25 NAMED cubelet geoms (the
    reference leaves one cubelet geom unnamed, and its bounding sphere unscaled), and the cubelet hull `cube:rounded_cube` through the
    engine's per-environment `mesh_scale` row.  Masses and inertias keep their values.  As the reference calls `set_constants()` after
    its modifiers (cube_env.py:343-349), `apply()` then recomputes dof_invweight0 / body_invweight0 / tendon_invweight0 /
    opt_meaninertia on the device (`BatchedSim.set_const`) from each environment's own rows: `BatchedConstants` assumes the shared model's
    geometry.  `None` (default) leaves the cube at its nominal size and every row as without the argument."""

    def __init__(self, m, names, rand, torch, device, dtype, hand_prefix="robot0:", cube_prefix="cube:", cube_size_range=None):
        super().__init__(m, names, rand, torch, device, dtype, hand_prefix, cube_prefix)
        jn = names["joint"]
        face_j = {j for j, nme in enumerate(jn) if nme is not None and (nme.startswith(cube_prefix + "cubelet:driver:") or nme.startswith(cube_prefix + "cubelet:rot"))}
        self.face_dofs = torch.as_tensor([d for d in range(m["nv"]) if int(m["dof_jntid"][d]) in face_j], dtype=torch.long, device=device)
        self.cube_size_range = None if cube_size_range is None else (float(cube_size_range[0]), float(cube_size_range[1]))
        if self.cube_size_range is not None:
            lo, hi = self.cube_size_range
            if not (0.0 < lo <= hi and math.isfinite(hi)):
                raise ValueError(f"cube_size_range must satisfy 0 < low <= high < inf, got {cube_size_range}")
            pre = cube_prefix + "cubelet:"
            sel = lambda lst: torch.as_tensor([i for i, nme in enumerate(lst) if nme is not None and nme.startswith(pre)], dtype=torch.long, device=device)
            self.cubelet_bodies = sel(names["body"])
            self.cubelet_geoms = sel(names["geom"])
            self.cube_mesh = names["mesh"].index(cube_prefix + "rounded_cube")
            self.orig["body_pos"] = torch.as_tensor(np.asarray(m["body_pos"]), dtype=dtype, device=device).reshape(1, -1)
            self.orig["mesh_scale"] = torch.ones(1, m["nmesh"], dtype=dtype, device=device)

    def _extra_rules(self, n, draw, out):
        damp = out["dof_damping"]
        damp[:, self.face_dofs] = damp[:, self.face_dofs] * draw("face_damping", lambda: self._logu(1 / 3.0, 3.0, n, int(self.face_dofs.numel())))

    def sample(self, n, noises=None):
        out = super().sample(n, noises)
        if self.cube_size_range is None:
            return out
        nz = noises or {}
        s = nz["cube_size"].to(self.dtype) if "cube_size" in nz else self.rand.uniform(*self.cube_size_range, n, 1)   # last draw of the episode
        o = self.orig
        bp = o["body_pos"].reshape(1, -1, 3).repeat(n, 1, 1)
        bp[:, self.cubelet_bodies] = bp[:, self.cubelet_bodies] * s.reshape(n, 1, 1)
        out["body_pos"] = bp.reshape(n, -1)
        rb = o["geom_rbound"].repeat(n, 1)
        rb[:, self.cubelet_geoms] = rb[:, self.cubelet_geoms] * s.reshape(n, 1)
        out["geom_rbound"] = rb
        ms = o["mesh_scale"].repeat(n, 1)
        ms[:, self.cube_mesh] = s.reshape(n)
        out["mesh_scale"] = ms
        return out

    def apply(self, sim, params, idx=None):
        super().apply(sim, params, idx)
        if self.cube_size_range is not None:
            # set_constants() after the modifiers: the scaled cubelet offsets move the bodies' centres of mass
            mask = None
            if idx is not None:
                mask = self.torch.zeros(sim.nenv, dtype=self.torch.uint8, device=sim.device)
                mask[self.torch.as_tensor(idx, device=sim.device)] = 1
            sim.set_const(mask=mask)
