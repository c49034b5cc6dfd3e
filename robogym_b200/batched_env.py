"""Batched host facade for the ShadowHand + cube step loop (SURVEY.md 8(f) row 1; rows a6-a9 of 8(a)).

Torch restatements, over `[nenv, ...]` tensors, of the per-environment numpy code that surrounds
`SimulationInterface.step()` in the reference -- so that 8192 environments do not need 8192 Python
`RobotEnv` objects:

* `denormalize_position_control`  <- robogym/robot/robot_interface.py:247-278 with
  `joint_positions_to_control` = POSITION_TO_CONTROL_MATRIX @ qpos (robot/shadow_hand/hand_interface.py:400-405);
  the 20x24 matrix is read off the compiled model's actuator transmissions (joint -> 1, fixed tendon -> its
  joint coefficients), which reproduces hand_interface.py:245-266.
* `observe`                       <- MuJoCoObservation (robot/shadow_hand/mujoco/mujoco_shadow_hand.py:21-46),
  get_relative_positions (robot/shadow_hand/hand_forward_kinematics.py:39-50), cube observations
  (envs/dactyl/observation/cube.py:8-29).
* `on_palm`                       <- envs/dactyl/common/cube_utils.py:17-23 / wrappers/cube.py:153-156.
* `fingers_occluded`              <- utils/sensor_utils.py:18-38 (contacts with dist < -1e-4 on the occlusion boxes).

Everything here is elementwise / small-matmul torch on the device the state tensors live on; the
physics stays in `engine.BatchedSim`.  tests/test_batched_facade.py checks each function against the
reference's own code driven through the mujoco_py shim.
"""
import numpy as np

FINGERTIP_SITES = ["S_fftip", "S_mftip", "S_rftip", "S_lftip", "S_thtip"]
REFERENCE_SITES = ["phasespace_ref0", "phasespace_ref1", "phasespace_ref2"]
WRAP_JOINT, TRN_JOINT, TRN_TENDON = 1, 0, 3


class ShadowHandCubeFacade:
    def __init__(self, model, names, device, hand_prefix="robot0:", cube_prefix="cube:", max_position_change=None, dtype=None):
        import torch

        self.torch = torch
        dtype = dtype or torch.float32
        m = model
        t = lambda a, dt=dtype: torch.as_tensor(np.asarray(a), dtype=dt, device=device)
        jn = names["joint"]
        hand = [j for j, n in enumerate(jn) if n is not None and n.startswith(hand_prefix)]
        self.hand_qpos_idx = t([m["jnt_qposadr"][j] for j in hand], torch.long)
        self.hand_qvel_idx = t([m["jnt_dofadr"][j] for j in hand], torch.long)
        col = {j: k for k, j in enumerate(hand)}
        P = np.zeros((m["nu"], len(hand)))
        for i in range(m["nu"]):
            tid = int(m["actuator_trnid"][i])
            if m["actuator_trntype"][i] == TRN_JOINT:
                P[i, col[tid]] = 1.0
            else:
                for w in range(m["tendon_adr"][tid], m["tendon_adr"][tid] + m["tendon_num"][tid]):
                    assert m["wrap_type"][w] == WRAP_JOINT, "actuated tendons are fixed tendons"
                    P[i, col[int(m["wrap_objid"][w])]] = m["wrap_prm"][w]
        self.P = t(P)
        cr = m["actuator_ctrlrange"].reshape(-1, 2)
        self.ctrl_lo, self.ctrl_hi = t(cr[:, 0]), t(cr[:, 1])
        self.max_position_change = max_position_change
        fr = m["actuator_forcerange"].reshape(-1, 2)
        self.force_lo, self.force_hi = t(fr[:, 0]), t(fr[:, 1])
        sn = names["site"]
        self.tip_sites = t([sn.index(hand_prefix + s) for s in FINGERTIP_SITES], torch.long)
        self.ref_sites = t([sn.index(hand_prefix + s) for s in REFERENCE_SITES], torch.long)
        # a model without a cube (dactyl/reach) has no cube observations and no on-palm test
        self.has_cube = cube_prefix + "center" in sn
        self.cube_center = sn.index(cube_prefix + "center") if self.has_cube else None
        cube_t = [j for j, n in enumerate(jn) if n is not None and n.startswith(cube_prefix + "cube_t")]
        cube_r = [j for j, n in enumerate(jn) if n == cube_prefix + "cube_rot"]
        self.cube_pos_idx = t([m["jnt_qposadr"][j] for j in cube_t], torch.long)
        a = int(m["jnt_qposadr"][cube_r[0]]) if cube_r else 0
        self.cube_quat_idx = t(list(range(a, a + 4)) if cube_r else [], torch.long)
        self.occlusion_geoms = t([g for g, n in enumerate(names["geom"]) if n is not None and n.endswith("occlusion")], torch.long)

    # ---- a6: action -> ctrl
    def joint_positions_to_control(self, qpos):
        return qpos[:, self.hand_qpos_idx] @ self.P.T

    def denormalize_position_control(self, action, qpos=None, relative_action=True, ctrlrange=None):
        """`ctrlrange` ([nenv, nu, 2], optional): per-environment control ranges (joint-limit randomisation)."""
        torch = self.torch
        lo, hi = (self.ctrl_lo, self.ctrl_hi) if ctrlrange is None else (ctrlrange[..., 0], ctrlrange[..., 1])
        return self._denormalize(action, qpos, relative_action, lo, hi)

    def _denormalize(self, action, qpos, relative_action, ctrl_lo, ctrl_hi):
        torch = self.torch
        base = 0.5 * (ctrl_hi - ctrl_lo)
        if relative_action:
            center = self.joint_positions_to_control(qpos)
            rng = torch.clamp(base, max=self.max_position_change) if self.max_position_change else base
        else:
            center = 0.5 * (ctrl_hi + ctrl_lo)
            rng = base
        return torch.minimum(torch.maximum(center + action * rng, ctrl_lo), ctrl_hi)

    # ---- a7: observations
    def fingertip_relative_positions(self, site_xpos):
        torch = self.torch
        tips = site_xpos[:, self.tip_sites] - site_xpos[:, self.ref_sites[1]].unsqueeze(1)
        ref = site_xpos[:, self.ref_sites] - site_xpos[:, self.ref_sites[1]].unsqueeze(1)
        e0 = ref[:, 0] / ref[:, 0].norm(dim=1, keepdim=True)
        e2 = ref[:, 2] / ref[:, 2].norm(dim=1, keepdim=True)
        ort = torch.cross(e0, e2, dim=1)
        basis = torch.stack([e0, ort, e2], dim=2)          # columns, like np.transpose([e0, ort, e2])
        return torch.bmm(tips, basis)

    def fingertip_absolute_positions(self, site_xpos):
        """MujocoShadowhandAbsoluteFingertipsObservation (envs/dactyl/observation/shadow_hand.py:40-58): [nenv, 15]"""
        return site_xpos[:, self.tip_sites].reshape(site_xpos.shape[0], -1)

    def observe(self, qpos, qvel, site_xpos, act_force=None):
        torch = self.torch
        obs = dict(
            hand_angle=qpos[:, self.hand_qpos_idx],
            hand_velocity=qvel[:, self.hand_qvel_idx],
            fingertip_pos=self.fingertip_relative_positions(site_xpos).reshape(qpos.shape[0], -1),
            qpos=qpos, qvel=qvel,
        )
        if self.has_cube:
            quat = qpos[:, self.cube_quat_idx]
            obs["cube_pos"] = qpos[:, self.cube_pos_idx]          # get_qpos("cube_position"): slide-joint coordinates
            # robogym.utils.rotation.quat_normalize (rotation.py:281-286) only canonicalises the sign (w >= 0)
            obs["cube_quat"] = quat * torch.where(quat[:, :1] < 0, -torch.ones_like(quat[:, :1]), torch.ones_like(quat[:, :1]))
        if act_force is not None:
            # normalize_by_limits (robot/shadow_hand/hand_utils.py:21-28): x / hi for x >= 0, |x| / lo otherwise
            obs["actuator_force"] = torch.where(act_force >= 0, act_force / self.force_hi, act_force.abs() / self.force_lo)
        return obs

    # ---- a8 / a9
    def on_palm(self, site_xpos, height=0.04):
        return site_xpos[:, self.cube_center, 2] > height

    def fingers_occluded(self, contact, ncon, dist_cutoff=-1e-4):
        """contact: [nenv, K, 4] = (geom1, geom2, dist, dim) rows as written by the engine; returns [nenv, 5] bools."""
        torch = self.torch
        K = contact.shape[1]
        valid = (torch.arange(K, device=contact.device).unsqueeze(0) < ncon.unsqueeze(1)) & (contact[:, :, 2] < dist_cutoff)
        g1, g2 = contact[:, :, 0].long(), contact[:, :, 1].long()
        occ = self.occlusion_geoms.view(1, 1, -1)
        hit = ((g1.unsqueeze(2) == occ) | (g2.unsqueeze(2) == occ)) & valid.unsqueeze(2)
        return hit.any(dim=1)
