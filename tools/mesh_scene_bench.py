#!/usr/bin/env python
"""rearrange/ycb at batch 1024 three ways: the plain rearrange_ycb8 batch, the slotted model (robogym_b200.rearrange_mesh_scene)
holding the same draw in every environment, and the slotted model with a random draw per environment.  Prints one JSON line
per variant and round: env-steps/s (one env-step = 20 substeps + forward), environments resident per SM (warps per CTA, one
CTA per SM), mean active pairs per environment, the warning bits raised, and the card's power limit and SM clock; then one
summary line per variant (median and spread over the alternated rounds).

Every variant starts from bench.py's rearrange reset: the mocap weld reset to identity, the arm at its start pose, the mocap
body on the tool centre point, the gripper command at its upper limit, and the objects resting on the table in front of the arm
by their lowest hull points, unrotated, on a grid that keeps any two library objects apart.  The mocap target then stays where
it is, so the timed steps hold the scene at rest; no environment may need a bad-state reset (warning bit 2).

    python tools/mesh_scene_bench.py [--nenv 1024] [--steps 20] [--rounds 3]
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
CAPS = dict(contact_capacity=64, row_capacity=128, dofs_per_contact=16)         # bench.py's rearrange_ycb capacities


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
    n = args.nenv
    # a 3 x 3 grid on the table (x 0.84..2.06, y 0.01..1.54), centre cell empty, wide enough that no two of the library's
    # objects overlap whatever the draw: the largest half extents are 0.11 m along x and 0.20 m along y
    slots_xy = [[1.25 + 0.30 * (k % 3), 0.30 + 0.44 * (k // 3)] for k in (0, 1, 2, 3, 5, 6, 7, 8)]
    rng = np.random.RandomState(0)
    yaw = np.zeros((n, 8))                       # objects unrotated, as the tests place them
    random_draw = rng.randint(0, len(lib.entries), (n, 8))

    def make(variant):
        model = engine.DeviceModel(b8 if variant == "plain" else sb, 0)
        # random draws rest up to 217 parts on the table (one contact each, the base draw 59): bench.py's 64 contacts would drop
        # most of them and let objects sink, so that arm gets room for every resting part
        caps = dict(CAPS, contact_capacity=256) if variant == "slotted_random" else CAPS
        sim = engine.BatchedSim(model, n, 20, outputs=("ncon", "warn", "body_xpos", "body_xquat"), **caps)
        m, names = model.host, modelblob.unpack_names(b8 if variant == "plain" else sb)
        eq = np.array(m["eq_data"], dtype=np.float64).reshape(-1, 7)
        eq[0] = [0, 0, 0, 1, 0, 0, 0]                                           # gym reset_mocap_welds
        model.set_field("eq_data", eq.reshape(-1))
        sim.qpos[:, :6] = torch.tensor(ARM_INIT, dtype=torch.float32, device=sim.device)
        for k in range(8):                                                      # out of the way while the tool pose is read
            a = int(m["jnt_qposadr"][names["joint"].index(f"object{k}:joint")])
            sim.qpos[:, a:a + 3] = torch.tensor([1.0 + 0.25 * (k % 4), 1.1 + 0.3 * (k // 4), 0.75], device=sim.device)
        if variant != "plain":
            sc = rms.BatchedMeshScene(sim, lib)
            sc.set_objects(np.array([lib.identity[0]] * n) if variant == "slotted_identity" else random_draw)
        sim.forward()
        tcp = names["body"].index("robot0:gripper_tcp")
        sim.mocap_pos[:, 0].copy_(sim.body_xpos[:, tcp]); sim.mocap_quat[:, 0].copy_(sim.body_xquat[:, tcp])   # reset_mocap2body_xpos
        sim.ctrl.copy_(torch.tensor(m["actuator_ctrlrange"].reshape(-1, 2)[:, 1], dtype=torch.float32, device=sim.device).expand_as(sim.ctrl))
        if variant == "plain":
            for k in range(8):
                a = int(m["jnt_qposadr"][names["joint"].index(f"object{k}:joint")])
                sim.qpos[:, a:a + 2] = torch.tensor(slots_xy[k], device=sim.device)
                sim.qpos[:, a + 2] = TABLE_TOP - lib.entries[lib.identity[0][k]].lowest_point() + 1e-3
                h = torch.tensor(0.5 * yaw[:, k], dtype=torch.float32, device=sim.device)
                sim.qpos[:, a + 3] = torch.cos(h); sim.qpos[:, a + 4:a + 6] = 0.0; sim.qpos[:, a + 6] = torch.sin(h)
            pairs = float(m["npair"])
        else:
            sc.place(torch.tensor(slots_xy, device=sim.device).expand(n, 8, 2), yaw, TABLE_TOP)
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

    sims = {v: make(v) for v in ("plain", "slotted_identity", "slotted_random")}
    rates = {v: [] for v in sims}
    for r in range(args.rounds):
        for v, (sim, pairs) in sims.items():
            times = []
            for _ in range(args.steps):
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(); sim.step(); b.record()
                torch.cuda.synchronize()
                times.append(a.elapsed_time(b) / 1e3)
            info = sim.launch_info()
            rates[v].append(n / statistics.median(times))
            print(json.dumps(dict(variant=v, round=r, nenv=n, env_steps_per_s=round(n / statistics.median(times), 1), contact_capacity=sim.contact_capacity,
                                  envs_per_sm=info["warps_per_cta"], ctas=info["ctas"], smem_bytes=info["smem_bytes"],
                                  mean_active_pairs=round(pairs, 1), warn_bits=int(sim.warn.max()), gpu=clocks())), flush=True)
    for v, x in rates.items():
        warn = sims[v][0].warn
        print(json.dumps(dict(variant=v, summary=True, env_steps_per_s_median=round(statistics.median(x), 1), min=round(min(x), 1),
                              max=round(max(x), 1), rounds=len(x), envs_with_bad_state_reset=int(((warn & 4) != 0).sum()),
                              warn_bits_any=int(warn.max()))), flush=True)


if __name__ == "__main__":
    main()
