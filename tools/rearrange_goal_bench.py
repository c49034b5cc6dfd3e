#!/usr/bin/env python
"""Goal evaluation and goal orientations on the device (robogym_b200.rearrange_goal): BatchedRearrangeGoal.evaluate
(rg_rearrange_goal) and goal_orientations (rg_goal_orientations).

Workloads:
- blocks: evaluate on 2048 environments of rearrange_blocks5_tcp, 5 blocks, rot_dist_type mod90, two groups of duplicates
  ([0, 0, 1, 1, 1]) so the greedy matching runs;
- ycb: evaluate on 1024 environments of rearrange_ycb8_tcp, 8 slots (10 % padded), rot_dist_type full, distinct objects;
- orientations: goal_orientations("block") for 2048 x 5 slots.
The evaluations read the sims' body_xpos / body_xquat rows in place; those rows hold random object poses, half of them near
their goals (the kernel's work does not depend on how the poses came about).

Times are CUDA events around `--iters` calls after `--warmup` untimed ones; the workloads alternate round by round and each
figure is the median of `--rounds`.  A call's time includes its host-side launch.  Prints one JSON line per workload with the
card's name, power limit and SM clock read in the same run; compare with one env-step of the same batch from
`bench.py --config rearrange_blocks_tcp` / `rearrange_ycb_tcp`.

    python tools/rearrange_goal_bench.py [--iters 200] [--warmup 20] [--rounds 5]
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


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _batch(torch, asset, nenv, nobj, groups, mode, rng):
    from robogym_b200 import engine, rearrange_goal as rg, rearrange_placement as rp

    blob = open(os.path.join(ROOT, "robogym_b200", "assets", asset + ".rgm"), "rb").read()
    model = engine.DeviceModel(blob, 0)
    sim = engine.BatchedSim(model, nenv, 10, outputs=("body_xpos", "body_xquat"))
    bodies = [model.name2id("body", f"object{k}") for k in range(nobj)]
    table = rp.table_dimensions(model)
    top = table[2]
    gp = np.stack([rng.uniform(1.0, 1.6, (nenv, nobj)), rng.uniform(0.3, 1.2, (nenv, nobj)), np.full((nenv, nobj), top + 0.03)], -1)
    gq = rng.normal(size=(nenv, nobj, 4))
    near = rng.rand(nenv, nobj) < 0.5
    pos = np.where(near[..., None], gp + rng.normal(scale=0.02, size=gp.shape), rng.uniform(0.8, 1.8, gp.shape))
    quat = np.where(near[..., None], gq + rng.normal(scale=0.05, size=gq.shape), rng.normal(size=gq.shape))
    b = torch.as_tensor(bodies, device=sim.device)
    sim.body_xpos[:, b] = torch.as_tensor(pos, dtype=torch.float32, device=sim.device)
    sim.body_xquat[:, b] = torch.as_tensor(quat, dtype=torch.float32, device=sim.device)
    goal = rg.BatchedRearrangeGoal(sim, bodies, groups, table, rot_dist_type=mode)
    goal.set_goal(torch.as_tensor(gp), torch.as_tensor(gq))
    return goal


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()

    import torch
    from robogym_b200 import build, rearrange_goal as rg

    build.build()
    rng = np.random.RandomState(0)
    blocks = _batch(torch, "rearrange_blocks5_tcp", 2048, 5, np.array([0, 0, 1, 1, 1]), "mod90", rng)
    ycb_groups = np.tile(np.arange(8), (1024, 1))
    ycb_groups[rng.rand(1024, 8) < 0.1] = -1
    ycb = _batch(torch, "rearrange_ycb8_tcp", 1024, 8, ycb_groups, "full", rng)
    base = torch.as_tensor(rng.normal(size=(2048, 5, 4)), device="cuda:0")
    active = torch.ones(2048, 5, dtype=torch.bool, device="cuda:0")
    work = {"blocks_evaluate_2048x5_mod90": blocks.evaluate, "ycb_evaluate_1024x8_full": ycb.evaluate,
            "goal_orientations_block_2048x5": lambda: rg.goal_orientations(base, active, 1, 2, mode="block")}
    for fn in work.values():
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in work}
    for _ in range(args.rounds):
        for k, fn in work.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for _ in range(args.iters):
                fn()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b) / args.iters)
    card = _card()
    info = blocks.evaluate()
    torch.cuda.synchronize()
    for k, v in times.items():
        print(json.dumps(dict(workload=k, ms_median=round(statistics.median(v), 4), ms_min=round(min(v), 4), ms_max=round(max(v), 4), iters=args.iters,
                              rounds=args.rounds, card=card)), flush=True)
    print(json.dumps(dict(check="blocks", achieved=int(info["goal_achieved"].sum()), mean_num_success=float(info["num_success"].mean()))), flush=True)


if __name__ == "__main__":
    main()
