"""Env-steps/s of dactyl/full_perpendicular at the bench's batch with one warp per environment against one environment per CTA of
W warps (RG_WARPS_PER_ENV), alternated in one process for several rounds, CUDA events around each step, and every arm's outputs
compared byte for byte with the one-warp arm's from the same start state and controls.  Prints one JSON line with the card, its
power limit and SM clock, read in the same run.

Development tool, needs a GPU: python tools/cta_env_bench.py [--rounds 3] [--steps 5] [--warps 1,2,4,8,16]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="full_perpendicular")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warps", default="1,2,4,8,16")
    args = ap.parse_args()
    import torch

    import bench
    from robogym_b200 import build, engine

    build.build()
    cfg = bench.CONFIGS[args.config]
    blob = bench.load_blob(cfg["asset"])
    names = json.load(open(os.path.join(ROOT, "robogym_b200", "assets", cfg["asset"] + ".names.json")))
    model = engine.DeviceModel(blob, 0)
    n, caps = cfg["nenv"], cfg["caps"]
    outs = ("site_xpos", "act_force", "ncon", "warn")

    def make(w):
        os.environ["RG_WARPS_PER_ENV"] = str(w)
        sim = engine.BatchedSim(model, n, bench.NSUB, outputs=outs, contact_capacity=caps[0], row_capacity=caps[1], dofs_per_contact=caps[2])
        del os.environ["RG_WARPS_PER_ENV"]
        sim.set_balance(False)                 # every arm steps the environments in the same order from the same start
        return sim

    arms = [int(w) for w in args.warps.split(",")]
    sims = {w: make(w) for w in arms}
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1234)
    wl = bench.Workload(sims[arms[0]], model, names, torch.device("cuda"), gen)   # settled hand, reset cubes: the start state
    start = {k: getattr(sims[arms[0]], k).clone() for k in ("qpos", "qvel", "ctrl", "pid", "qacc_warmstart")}
    ctrls = []
    for _ in range(args.steps):
        ctrls.append(wl.ctrl_from_action(wl.sample_action()).clone())
    ms = {w: [] for w in arms}
    same = {w: True for w in arms}
    for _ in range(args.rounds):
        ref = None
        for w in arms:
            sim = sims[w]
            for k, v in start.items():
                getattr(sim, k).copy_(v)
            sim.step()                          # warm-up launch from the start state (the timed steps start over below)
            for k, v in start.items():
                getattr(sim, k).copy_(v)
            torch.cuda.synchronize()
            t = 0.0
            for c in ctrls:
                sim.ctrl.copy_(c)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                sim.step()
                e1.record()
                torch.cuda.synchronize()
                t += e0.elapsed_time(e1)
            ms[w].append(t / args.steps)
            got = [getattr(sim, k).cpu().numpy().tobytes() for k in ("qpos", "qvel", "pid", "qacc_warmstart", "site_xpos", "act_force", "ncon", "warn")]
            if ref is None:
                ref = got
            same[w] = same[w] and got == ref
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    res = {str(w): dict(ms_per_step=ms[w], env_steps_per_s=[n / x * 1e3 for x in ms[w]], median_env_steps_per_s=sorted(n / x * 1e3 for x in ms[w])[len(ms[w]) // 2],
                        bit_identical_to_first_arm=same[w], launch=sims[w].launch_info()) for w in arms}
    print(json.dumps(dict(config=args.config, nenv=n, rounds=args.rounds, steps=args.steps, card=smi, arms=res)))


if __name__ == "__main__":
    main()
