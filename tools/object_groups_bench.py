#!/usr/bin/env python
"""The object groups of a rearrange reset on the device (robogym_b200.rearrange_groups.object_groups: rg_object_groups), next
to one env-step of the same batch.

Workloads: 2048 environments x 5 blocks (rearrange_blocks5_tcp: 1 to 5 objects, random groups, the blocks' palette, scale
range (0.1, 0.1)) and 1024 environments x 8 YCB slots (rearrange_ycb8_tcp: 1 to 8 objects, random groups, random colours,
scale range (0.5, 0.5), 79 mesh candidates with replacement).

For each the JSON line gives the whole call (the Python wrapper: host arrays of the counts and the ObjectGroups outputs
allocated, then the C ABI), the C ABI call alone into preallocated outputs (the copy of the host inputs, the kernel and the
stream-ordered free), and the rg_groups_kernel alone (torch.profiler's CUDA time of the kernel, in a run of its own after
the timed ones).  Times are CUDA events around `--iters` calls after `--warmup` untimed ones, median of `--rounds`; the
env-step is sim.step() of the workload's model at the same batch size.  Prints one JSON line per workload with the card's name,
power limit and SM clock read in the same run.

    python tools/object_groups_bench.py [--iters 50] [--warmup 5] [--rounds 3]
"""
import argparse
import ctypes
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


def _kernel_ms(torch, fn, iters):
    """mean CUDA time of rg_groups_kernel over `iters` calls, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(iters):
            fn()
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if "rg_groups_kernel" in e.name]
    us = [getattr(e, "device_time", None) or getattr(e, "cuda_time", 0.0) for e in ev]
    return float(np.mean(us)) / 1000.0 if us else float("nan")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch

    from robogym_b200 import build, engine
    from robogym_b200 import rearrange_groups as rgr
    from robogym_b200 import rearrange_placement as rp

    build.build()
    card = _card()
    lib = engine.lib()
    for name, asset, n, nobj, kw in (
            ("blocks", "rearrange_blocks5_tcp", 2048, 5, dict(color_mode="palette", palette=rgr.BLOCK_COLORS, scale_range=(0.1, 0.1))),
            ("ycb", "rearrange_ycb8_tcp", 1024, 8, dict(color_mode="random", scale_range=(0.5, 0.5), mesh_candidates=list(range(79))))):
        rng = np.random.RandomState(0)
        active = rng.randint(1, nobj + 1, n)
        seed = rp.PlacementSeed(3)
        g = rgr.object_groups(active, *seed.next(), nobj=nobj, **kw)
        torch.cuda.synchronize()

        # the C ABI alone, into g's outputs
        c = engine.GroupsIn()
        act = np.ascontiguousarray(active, dtype=np.int32)
        pal = np.ascontiguousarray(np.asarray(rgr.BLOCK_COLORS, dtype=np.float64))
        c.nenv, c.nobj, c.active = n, nobj, act.ctypes.data
        c.group_mode, c.lam_low, c.lam_high, c.n_materials = rgr.GROUP_MODES["random"], rgr.LAM[0], rgr.LAM[1], 1
        c.color_mode = rgr.COLOR_MODES[kw["color_mode"]]
        if kw["color_mode"] == "palette":
            c.palette, c.n_palette = pal.ctypes.data, len(pal)
        c.scale_low, c.scale_high = kw["scale_range"]
        c.mesh_mode, c.n_candidates = (1, 79) if "mesh_candidates" in kw else (0, 0)
        o = engine.GroupsOut(**{k: engine.ptr(x) for k, x in g._asdict().items()})
        stream = engine.current_stream(torch, torch.device("cuda:0"))

        def abi():
            c.seed, c.epoch = seed.next()
            engine._check(lib.rg_object_groups(ctypes.byref(c), None, n, ctypes.byref(o), stream))

        res = dict(workload=name, nenv=n, objects=nobj, card=card)
        res["call_ms"] = round(_time(torch, lambda: rgr.object_groups(active, *seed.next(), nobj=nobj, **kw), args.iters, args.warmup, args.rounds), 4)
        res["abi_ms"] = round(_time(torch, abi, args.iters, args.warmup, args.rounds), 4)
        model = engine.DeviceModel(open(os.path.join(ROOT, "robogym_b200", "assets", asset + ".rgm"), "rb").read(), 0)
        sim = engine.BatchedSim(model, n, 10, outputs=("ncon", "warn"), contact_capacity=64,
                                row_capacity=160 if name == "blocks" else 128)
        res["env_step_ms"] = round(_time(torch, sim.step, max(args.iters // 10, 2), 2, args.rounds), 4)
        res["kernel_ms"] = round(_kernel_ms(torch, abi, args.iters), 4)
        res["call_over_step"] = round(res["call_ms"] / res["env_step_ms"], 4)
        print(json.dumps(res), flush=True)
        del sim, model


if __name__ == "__main__":
    main()
