#!/usr/bin/env python
"""rearrange/ycb at batch 1024 on the slotted model (robogym_b200.rearrange_mesh_scene), four arms: the base scene's draw in every
environment and a random draw per environment, each with every object at scale 1 and with every object at its own scale, the
reference's randomised size scale exp(U(-0.5, 0.5)) (sample_object_size_scales, ObjectLibrary.object_scales), i.e.
per-environment scaled rows and a bound geom_mesh_scale row.  The scaled arms hold the same draws as the unscaled ones.  Prints one JSON line per arm and round: env-steps/s (one env-step = 20 substeps + forward),
environments resident per SM (warps per CTA, one CTA per SM), shared memory per CTA, mean active pairs per environment, the
warning bits raised, and the card's power limit and SM clock; then one summary line per arm (median and spread over the
alternated rounds, environments that needed a bad-state reset).

The reset is tools/mesh_scene_bench.py's: mocap weld at identity, the arm at its start pose, the mocap body on the tool centre
point, the gripper command at its upper limit, and the objects resting on the table by their (scaled) lowest hull points,
unrotated, here on a 3 x 3 grid 0.32 m x 0.57 m wide whose cell below the arm stays empty, so that objects up to 1.65 x their
size stay apart and clear of the arm.  The mocap target stays where it is, so the timed steps hold the scene at rest.

    python tools/ycb_scale_bench.py [--nenv 1024] [--steps 20] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
TABLE_TOP = 0.453 + 0.03324
ARM_INIT = np.deg2rad(np.array([135.0, -90.0, 135.0, -100.0, -240.0, 135.0]))   # robogym/robot/ur16e/arm_interface.py:27
# bench.py's rearrange_ycb capacities, with room for one contact per resting part (a random draw rests up to 217 parts)
CAPS = dict(contact_capacity=256, row_capacity=128, dofs_per_contact=16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nenv", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch

    from robogym_b200 import build, engine, modelblob
    from robogym_b200 import rearrange_mesh_scene as rms

    build.build()
    blob = lambda n: open(os.path.join(ROOT, "robogym_b200", "assets", n + ".rgm"), "rb").read()
    b8, bt = blob("rearrange_ycb8"), blob("rearrange_ycb8_tcp")
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    sb = rms.slotted_model(b8, lib)
    names = modelblob.unpack_names(sb)
    n = args.nenv
    slots_xy = [[1.22 + 0.32 * (k % 3), 0.20 + 0.57 * (k // 3)] for k in range(1, 9)]
    rng = np.random.RandomState(0)
    draws = {"identity": np.array([lib.identity[0]] * n), "random": rng.randint(0, len(lib.entries), (n, 8))}
    size = rms.sample_object_size_scales(n, 8, 0.5, 0.5, generator=torch.Generator(device="cuda:0").manual_seed(0))
    arms = {}
    for d, draw in draws.items():
        arms[d] = (draw, None)
        arms[d + "_scaled"] = (draw, lib.object_scales(draw, size))

    def make(arm):
        model = engine.DeviceModel(sb, 0)
        sim = engine.BatchedSim(model, n, 20, outputs=("ncon", "warn", "body_xpos", "body_xquat"), **CAPS)
        m = model.host
        eq = np.array(m["eq_data"], dtype=np.float64).reshape(-1, 7)
        eq[0] = [0, 0, 0, 1, 0, 0, 0]                                           # gym reset_mocap_welds
        model.set_field("eq_data", eq.reshape(-1))
        sim.qpos[:, :6] = torch.tensor(ARM_INIT, dtype=torch.float32, device=sim.device)
        for k in range(8):                                                      # out of the way while the tool pose is read
            a = int(m["jnt_qposadr"][names["joint"].index(f"object{k}:joint")])
            sim.qpos[:, a:a + 3] = torch.tensor([1.0 + 0.25 * (k % 4), 1.1 + 0.3 * (k // 4), 0.75], device=sim.device)
        sc = rms.BatchedMeshScene(sim, lib)
        sc.set_objects(*arms[arm])
        sim.forward()
        tcp = names["body"].index("robot0:gripper_tcp")
        sim.mocap_pos[:, 0].copy_(sim.body_xpos[:, tcp]); sim.mocap_quat[:, 0].copy_(sim.body_xquat[:, tcp])   # reset_mocap2body_xpos
        sim.ctrl.copy_(torch.tensor(m["actuator_ctrlrange"].reshape(-1, 2)[:, 1], dtype=torch.float32, device=sim.device).expand_as(sim.ctrl))
        sc.place(torch.tensor(slots_xy, device=sim.device).expand(n, 8, 2), np.zeros((n, 8)), TABLE_TOP)
        pairs = float(sim.pair_counts().float().mean())
        sim.qvel.zero_(); sim.pid.zero_(); sim.qacc_warmstart.zero_(); sim.warn.zero_()
        for _ in range(args.warmup):
            sim.step()
        torch.cuda.synchronize()
        return sim, pairs

    def clocks():
        try:
            return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                                  capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.SubprocessError):
            return "unknown"

    sims = {arm: make(arm) for arm in arms}
    rates = {arm: [] for arm in sims}
    for r in range(args.rounds):
        for arm, (sim, pairs) in sims.items():
            times = []
            for _ in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); sim.step(); b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b) / 1e3)
            info = sim.launch_info()
            rates[arm].append(n / statistics.median(times))
            print(json.dumps(dict(arm=arm, round=r, nenv=n, env_steps_per_s=round(n / statistics.median(times), 1), contact_capacity=sim.contact_capacity,
                                  envs_per_sm=info["warps_per_cta"], ctas=info["ctas"], smem_bytes=info["smem_bytes"],
                                  mean_active_pairs=round(pairs, 1), warn_bits=int(sim.warn.max()), gpu=clocks())), flush=True)
    for arm, x in rates.items():
        warn = sims[arm][0].warn
        print(json.dumps(dict(arm=arm, summary=True, env_steps_per_s_median=round(statistics.median(x), 1), min=round(min(x), 1),
                              max=round(max(x), 1), rounds=len(x), envs_with_bad_state_reset=int(((warn & 4) != 0).sum()),
                              warn_bits_any=int(warn.max()))), flush=True)


if __name__ == "__main__":
    main()
