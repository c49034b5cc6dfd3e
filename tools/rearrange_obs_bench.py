"""Time BatchedRearrangeObservation.observe() (rg_rearrange_obs) against one env-step of the same batch and against the torch-op
assembly of the same keys.

Workloads: rearrange_blocks5_tcp with 2048 environments (5 blocks) and rearrange_ycb8_tcp with 1024 environments (5 of 8 slots
active, masks on), random states as tests/test_rearrange_obs.py builds them.  Arms per workload: `observe` (one launch),
`torch_ops` (the tests' tensor-op restatement of the object, goal and robot keys: a subset of what observe writes, without
contacts or masks), and `step` (sim.step(): 10 substeps and a forward, the env-step the observation follows).  Times are CUDA
events around `--iters` calls after `--warmup` untimed ones, host launch included; the arms alternate round by round and each
figure is the median of `--rounds`.  Prints one JSON line per arm with the card, its power limit and maximum SM clock.

    python tools/rearrange_obs_bench.py [--iters 200] [--warmup 20] [--rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    import torch

    from test_rearrange_obs import _batch, _restate

    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    card = _card()
    arms = {}
    for name, asset, nenv, mask in (("blocks", "rearrange_blocks5_tcp", 2048, False), ("ycb", "rearrange_ycb8_tcp", 1024, True)):
        sim, goal, obs_fn = _batch(asset, nenv, 5, 1, mask)
        arms[f"{name}/observe"] = (lambda o=obs_fn: o.observe(), args.iters)
        arms[f"{name}/torch_ops"] = (lambda s=sim, g=goal, o=obs_fn: _restate(s, g, o), args.iters)
        arms[f"{name}/step"] = (lambda s=sim: s.step(), max(1, args.iters // 10))
    times = {k: [] for k in arms}
    for fn, n in arms.values():
        for _ in range(args.warmup):
            fn()
    torch.cuda.synchronize()
    for _ in range(args.rounds):
        for k, (fn, n) in arms.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            for _ in range(n):
                fn()
            b.record()
            torch.cuda.synchronize()
            times[k].append(a.elapsed_time(b) / n)
    for k, v in times.items():
        print(json.dumps(dict(workload=k, ms_median=round(statistics.median(v), 4), ms_min=round(min(v), 4), ms_max=round(max(v), 4),
                              iters=arms[k][1], rounds=args.rounds, card=card)), flush=True)


if __name__ == "__main__":
    main()
