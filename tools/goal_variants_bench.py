#!/usr/bin/env python
"""The reference's other goal generators on the device (robogym_b200.rearrange_placement stack_goals, pick_and_place_goals,
train_goals, reach_goals: rg_place_objects then rg_goal_modify), each next to one env-step of the same batch.

Workloads:
- blocks: 2048 environments of rearrange_blocks5, 5 blocks of half size U(0.02, 0.05), 2 to 5 active (reach: one);
- ycb: 1024 environments of the slotted rearrange_ycb8 model, 8 slots with random draws (10 % empty slots), their rotated
  bounding boxes at random yaws (reach: one active slot).

For every generator the JSON line gives the whole call (placement, modifier and the host-side checks, which read the active
counts back) and the rg_goal_modify launch alone.  Times are CUDA events around `--iters` calls after `--warmup` untimed ones,
median of `--rounds`; one env-step is the batch's sim.step() (10 substeps + forward for blocks, 20 for ycb) on the scene placed
by object_placements (as tools/placement_bench.py times it).  Prints one JSON
line per workload with the card's name, power limit and SM clock read in the same run.

    python tools/goal_variants_bench.py [--iters 20] [--warmup 3] [--rounds 3]
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
ARM_INIT = np.deg2rad(np.array([135.0, -90.0, 135.0, -100.0, -240.0, 135.0]))
CAPS = dict(contact_capacity=256, row_capacity=128, dofs_per_contact=16)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _time(torch, fn, iters, warmup, rounds):
    for _ in range(warmup):
        fn()
    out = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b) / iters)
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch

    from robogym_b200 import build, engine
    from robogym_b200 import rearrange_mesh_scene as rms
    from robogym_b200 import rearrange_placement as rp
    from robogym_b200.rearrange_scene import BatchedBlockScene

    build.build()
    card = _card()
    blob = lambda n: open(os.path.join(ROOT, "robogym_b200", "assets", n + ".rgm"), "rb").read()
    rng = np.random.RandomState(0)
    T = lambda x: torch.as_tensor(x, device="cuda:0")
    yawq = lambda y: T(np.stack([np.cos(0.5 * y), 0 * y, 0 * y, np.sin(0.5 * y)], -1))

    workloads = []
    bmodel = engine.DeviceModel(blob("rearrange_blocks5"), 0)
    bsim = engine.BatchedSim(bmodel, 2048, 10, outputs=("ncon", "warn"))
    bs = BatchedBlockScene(bsim)
    bs.set_blocks(rng.uniform(0.02, 0.05, (2048, bs.nobj)))
    workloads.append(("blocks", bsim, bs, rp.table_dimensions(bmodel)))
    b8, bt = blob("rearrange_ycb8"), blob("rearrange_ycb8_tcp")
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    model = engine.DeviceModel(rms.slotted_model(b8, lib), 0)
    sim = engine.BatchedSim(model, 1024, 20, outputs=("ncon", "warn"), **CAPS)
    sc = rms.BatchedMeshScene(sim, lib)
    draw = rng.randint(0, len(lib.entries), (1024, 8))
    draw[rng.rand(1024, 8) < 0.1] = -1
    sc.set_objects(draw, np.ones((1024, 8)))
    sim.qpos[:, :6] = T(ARM_INIT).float()
    workloads.append(("ycb", sim, sc, rp.table_dimensions(model)))

    for name, s, scene, table in workloads:
        n, nobj = s.nenv, len(scene.bodies)
        yaw = rng.uniform(-np.pi, np.pi, (n, nobj))
        bbox = scene.bounding_boxes(yawq(yaw))
        act = rng.rand(n, nobj) < 0.6
        act[np.arange(n), rng.randint(nobj, size=n)] = True
        act[np.arange(n), (act.argmax(1) + rng.randint(1, nobj, size=n)) % nobj] = True
        if name == "ycb":
            act &= draw >= 0
            act[(act.sum(1) < 2), :2] = True
        one = np.zeros((n, nobj), bool)
        one[np.arange(n), rng.randint(nobj, size=n)] = True
        active, single = T(act), T(one)
        area, area1 = rp.placement_area(table, act.sum(1), 1.0), rp.placement_area(table, 1, 1.0)
        seed = rp.PlacementSeed(1)
        osz = T(rng.uniform(0.02, 0.05, n))
        anchor, _ = rp.object_placements(bbox, active, table, area, *seed.next())
        if name == "ycb":
            scene.place(anchor[..., :2], T(yaw), table[2])
        else:
            scene.place(anchor[..., :2], T(yaw), anchor[..., 2], active=active)
        out = torch.zeros(n, nobj, 3, dtype=torch.float64, device="cuda:0")
        calls = dict(
            stack=(lambda: rp.stack_goals(bbox, active, table, area, *seed.next(), osz, out=out),
                   lambda: rp._modify("stack", out, active.to(torch.uint8), *seed.next(), None, object_size=osz, fixed_order=False)),
            pick_and_place=(lambda: rp.pick_and_place_goals(bbox, active, table, area, *seed.next(), out=out),
                            lambda: rp._modify("lift", out, active.to(torch.uint8), *seed.next(), None, height_range=(0.05, 0.25))),
            train=(lambda: rp.train_goals(bbox, active, table, area, *seed.next(), anchor, 0.5, 0.3, 0.4, object_size=osz, out=out),
                   lambda: rp._modify("train", out, active.to(torch.uint8), *seed.next(), None, object_size=osz, ratio=0.5, height_range=(0.05, 0.25),
                                      pickup=0.3, stacking=0.4)),
            reach=(lambda: rp.reach_goals(bbox, single, table, area1, *seed.next(), 0.1, out=out),
                   lambda: rp._modify("reach", out, single.to(torch.uint8), *seed.next(), None, target_height=0.1)))
        res = dict(workload=name, nenv=n, objects=nobj, card=card)
        for k, (whole, modify) in calls.items():
            res[k + "_ms"] = round(_time(torch, whole, args.iters, args.warmup, args.rounds), 4)
            res[k + "_modify_ms"] = round(_time(torch, modify, args.iters, args.warmup, args.rounds), 4)
        res["env_step_ms"] = round(_time(torch, s.step, max(args.iters // 4, 2), args.warmup, args.rounds), 4)
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
