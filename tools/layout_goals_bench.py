#!/usr/bin/env python
"""The reference's layout goal generators on the device (robogym_b200.rearrange_placement domino_goals, attached_goals,
fixed_goals: rg_layout_goals), each next to one env-step of rearrange_blocks5_tcp at the same batch size.

Workload: 2048 environments x 8 slots.  Dominoes: object_size U(0.015, 0.035), eccentricity U(1, 4.5), 1 to 8 active,
distance_mul U(2, 5), the default placement area of the active count (so some environments need many retries and some
exhaust MAX_RETRY = 1000); attached blocks: 8 of 8 active; fixed layouts: wordblocks' placements on 6 of 8 slots.

For every kind the JSON line gives the whole call (the wrapper's checks, which read the active counts back, and the launch)
and the rg_layout_goals launch alone.  Times are CUDA events around `--iters` calls after `--warmup` untimed ones, median of
`--rounds`; the env-step is sim.step() (10 substeps) of a rearrange_blocks5_tcp batch of 2048.  Dominoes also report how many
retry rounds (32 retries each) their slowest and their median environment took.  Prints one JSON line with the card's name,
power limit and SM clock read in the same run.

    python tools/layout_goals_bench.py [--iters 20] [--warmup 3] [--rounds 3]
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
    from robogym_b200 import rearrange_placement as rp

    build.build()
    card = _card()
    n, nobj = 2048, 8
    rng = np.random.RandomState(0)
    T = lambda x: torch.as_tensor(x, device="cuda:0")
    model = engine.DeviceModel(open(os.path.join(ROOT, "robogym_b200", "assets", "rearrange_blocks5_tcp.rgm"), "rb").read(), 0)
    sim = engine.BatchedSim(model, n, 10, outputs=("ncon", "warn"), contact_capacity=64, row_capacity=160)
    table = rp.table_dimensions(model)

    size, ecc = rng.uniform(0.015, 0.035, n), rng.uniform(1.0, 4.5, n)
    hs = (size[:, None] * np.stack([1.0 / ecc, np.ones(n), ecc], 1))[:, None].repeat(nobj, 1)
    bbox = T(np.stack([np.zeros((n, nobj, 3)), hs], 2))
    act = np.arange(nobj)[None] < rng.randint(1, nobj + 1, n)[:, None]
    active, full = T(act), T(np.ones((n, nobj), bool))
    area, area8 = T(rp.placement_area(table, act.sum(1), 1.0)), T(rp.placement_area(table, nobj, 1.0))
    osz, mul = T(size), T(rng.uniform(2.0, 5.0, n))
    words = np.array([[0.5, 0.05], [0.5, 0.2], [0.5, 0.35], [0.5, 0.65], [0.5, 0.8], [0.5, 0.95], [0.0, 0.0], [0.0, 0.0]])
    six = T(np.arange(nobj)[None].repeat(n, 0) < 6)
    seed = rp.PlacementSeed(1)
    out = (torch.zeros(n, nobj, 3, dtype=torch.float64, device="cuda:0"), torch.zeros(n, nobj, 4, dtype=torch.float64, device="cuda:0"))
    st = torch.zeros(n, dtype=torch.int32, device="cuda:0")
    ptr, lib = engine.ptr, engine.lib()
    tab = np.concatenate([np.asarray(table[0], dtype=np.float64), np.asarray(table[1], dtype=np.float64)])
    rel = T(np.broadcast_to(words, (n, nobj, 2)).copy())
    u8 = lambda a: a.to(torch.uint8).contiguous()
    stream = lambda: engine.current_stream(torch, torch.device("cuda:0"))

    def launch(kind, a, ar, s_, e_):
        engine._check(lib.rg_layout_goals(n, nobj, rp.LAYOUT[kind], ptr(bbox), ptr(a), tab.ctypes.data, ptr(ar), ptr(osz), ptr(mul), ptr(rel), 1000, s_, e_,
                                          None, ptr(out[0]), ptr(out[1]), ptr(st), None, None, stream()))

    a_dom, a_full, a_six = u8(active), u8(full), u8(six)
    calls = dict(
        domino=(lambda: rp.domino_goals(bbox, active, table, area, *seed.next(), osz, mul, out=out),
                lambda: launch("domino", a_dom, area, *seed.next())),
        attached=(lambda: rp.attached_goals(bbox, full, table, area8, *seed.next(), osz, out=out),
                  lambda: launch("attached", a_full, area8, *seed.next())),
        fixed=(lambda: rp.fixed_goals(bbox, six, table, area8, words, out=out),
               lambda: launch("fixed", a_six, area8, 0, 0)))
    res = dict(workload="blocks", nenv=n, objects=nobj, card=card)
    for k, (whole, kernel) in calls.items():
        res[k + "_ms"] = round(_time(torch, whole, args.iters, args.warmup, args.rounds), 4)
        res[k + "_kernel_ms"] = round(_time(torch, kernel, args.iters, args.warmup, args.rounds), 4)
    _, _, status, _, retry = rp.domino_goals(bbox, active, table, area, *seed.next(), osz, mul, details=True)
    r = retry.cpu().numpy()
    rounds = np.where(r >= 0, r // 32 + 1, (1000 + 31) // 32)
    res.update(domino_placed=round(float((status == 1).float().mean()), 4), domino_rounds_max=int(rounds.max()), domino_rounds_median=float(np.median(rounds)))
    res["env_step_ms"] = round(_time(torch, sim.step, max(args.iters // 4, 2), args.warmup, args.rounds), 4)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
