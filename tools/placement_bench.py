#!/usr/bin/env python
"""Reset-time placement on the device (robogym_b200.rearrange_placement): rotated bounding boxes (rg_batch_body_aabb) plus
grid_then_uniform placement (rg_place_objects), each next to one env-step of the same batch.

Workloads:
- ycb: 1024 environments of the slotted rearrange_ycb8 model, 8 slots, random draws (5 % empty slots), per-slot scales
  U(0.7, 1.3) and random yaws;
- blocks: 2048 environments of rearrange_blocks5, 5 blocks of random half size U(0.02, 0.05), random yaws, 80 % active;
- masked: a re-placement of 5 % of the environments of each batch (boxes and placement under the mask).

Times are CUDA events around `--iters` launches after `--warmup` untimed ones, median of `--rounds`; one env-step is the
batch's sim.step() (20 substeps + forward for ycb, 10 for blocks) on the placed scene.  ycb environments no algorithm could
place are redrawn and placed again under a mask, as a user would (the reference's safe_reset_env), before the env-step is
timed; the status counts are those of the first placement.  Prints one JSON line per workload with the card's name,
power limit and SM clock read in the same run.

    python tools/placement_bench.py [--iters 20] [--warmup 3] [--rounds 3]
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
    return statistics.median(out), min(out), max(out)


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

    # ycb: 1024 x 8 slots
    b8, bt = blob("rearrange_ycb8"), blob("rearrange_ycb8_tcp")
    lib = rms.ObjectLibrary.from_blobs(b8, bt)
    sb = rms.slotted_model(b8, lib)
    n = 1024
    draw = rng.randint(0, len(lib.entries), (n, 8))
    draw[rng.rand(n, 8) < 0.05] = -1
    model = engine.DeviceModel(sb, 0)
    sim = engine.BatchedSim(model, n, 20, outputs=("ncon", "warn"), **CAPS)
    sc = rms.BatchedMeshScene(sim, lib)
    scale = rng.uniform(0.7, 1.3, (n, 8))
    sc.set_objects(draw, scale)
    sim.qpos[:, :6] = T(ARM_INIT).float()
    yaw = rng.uniform(-np.pi, np.pi, (n, 8))
    workloads = [("ycb", sim, sc, yaw, T(draw >= 0), rp.table_dimensions(model), None)]
    # blocks: 2048 x 5
    bmodel = engine.DeviceModel(blob("rearrange_blocks5"), 0)
    bsim = engine.BatchedSim(bmodel, 2048, 10, outputs=("ncon", "warn"))
    bs = BatchedBlockScene(bsim)
    bs.set_blocks(rng.uniform(0.02, 0.05, (2048, bs.nobj)))
    workloads.append(("blocks", bsim, bs, rng.uniform(-np.pi, np.pi, (2048, bs.nobj)), T(rng.rand(2048, bs.nobj) < 0.8), rp.table_dimensions(bmodel), 8 * 2048 * bs.nobj))

    for name, s, scene, yaw, active, table, points in workloads:
        quat = yawq(yaw)
        area = rp.placement_area(table, active.sum(1).cpu().numpy(), 1.0)
        seed = rp.PlacementSeed(1)
        mask = T(rng.rand(s.nenv) < 0.05)
        out = torch.zeros(s.nenv, active.shape[1], 3, dtype=torch.float64, device="cuda:0")
        res = {}

        def boxes():
            res["bbox"] = scene.bounding_boxes(quat)

        def place(m=None):
            pos, st = rp.object_placements(res["bbox"], active, table, area, *seed.next(), mask=m, out=out)
            res["status"] = st

        def reset(m=None):
            res["bbox"] = scene.bounding_boxes(quat, mask=m)
            place(m)

        boxes()
        place()
        torch.cuda.synchronize()
        st = res["status"].cpu().numpy()
        # the env-step runs on the placed scene: redraw the environments no algorithm could place, and place them again
        rounds = 0
        while name == "ycb" and (res["status"] == 0).any() and rounds < 20:
            bad = (res["status"] == 0).cpu().numpy()
            draw[bad] = np.where(draw[bad] >= 0, rng.randint(0, len(lib.entries), draw[bad].shape), -1)
            scene.set_objects(draw, scale)
            res["bbox"] = scene.bounding_boxes(quat, mask=T(bad))
            _, st2 = rp.object_placements(res["bbox"], active, table, area, *seed.next(), mask=T(bad), out=out)
            res["status"] = torch.where(T(bad), st2, res["status"])
            rounds += 1
        still_invalid = int((res["status"] == 0).sum())
        if name == "ycb":
            points = int(sum(lib.entries[d].hulls[j].vert.shape[0] for d in draw.reshape(-1) if d >= 0 for j in range(lib.entries[d].nparts)))
        boxes()
        if name == "ycb":
            scene.place(out[..., :2], T(yaw), table[2])
        else:
            scene.place(out[..., :2], T(yaw), out[..., 2], active=active)
        t_box = _time(torch, boxes, args.iters, args.warmup, args.rounds)
        t_place = _time(torch, place, args.iters, args.warmup, args.rounds)
        t_reset = _time(torch, reset, args.iters, args.warmup, args.rounds)
        t_masked = _time(torch, lambda: reset(mask), args.iters, args.warmup, args.rounds)
        t_step = _time(torch, s.step, max(args.iters // 4, 2), args.warmup, args.rounds)
        print(json.dumps(dict(workload=name, nenv=s.nenv, objects=int(active.shape[1]), points_boxed=points, card=card,
                              boxes_ms=round(t_box[0], 4), placement_ms=round(t_place[0], 4), reset_ms=round(t_reset[0], 4),
                              reset_spread_ms=[round(t_reset[1], 4), round(t_reset[2], 4)], masked_5pct_reset_ms=round(t_masked[0], 4),
                              env_step_ms=round(t_step[0], 4), reset_over_env_step=round(t_reset[0] / t_step[0], 3),
                              status_counts=np.bincount(st, minlength=4).tolist(), redraw_rounds=rounds,
                              still_invalid=still_invalid)), flush=True)


if __name__ == "__main__":
    main()
