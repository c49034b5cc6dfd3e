"""Cycles per stage and env-step of one bench.py configuration, from the -DRG_PROFILE builds' clock64 counters (lane 0 of the
warp that owns the environment).  Level 1 splits the collision stage, level 2 the Newton solve.  The counters cost time of
their own: the shares are what counts, not the totals.

Development tool, needs a GPU: python tools/stage_profile.py [--config full_perpendicular] [--level 2] [--nenv 4096] [--steps 3]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

NAMES = ["kin", "massm", "bias", "tendon", "forces", "collide", "mkcon", "solve", "euler"]
SUB = {1: ["col:A-sphere", "col:B-obb", "col:C-narrow+write", "col:C-rounds", "-", "-", "col:loop"],
       2: ["sol:init", "sol:gradient", "sol:H-assembly", "sol:cholesky", "sol:tri-solves", "sol:linesearch", "sol:step+update"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="full_perpendicular")
    ap.add_argument("--level", type=int, default=2, choices=(1, 2))
    ap.add_argument("--nenv", type=int, default=0, help="0 = the configuration's batch")
    ap.add_argument("--steps", type=int, default=3, help="env-steps profiled after the workload's settling steps")
    args = ap.parse_args()
    from robogym_b200 import build

    os.environ["RG_LIB"] = build.build_profile(args.level)     # before the engine is imported: it loads RG_LIB
    import numpy as np
    import torch

    import bench
    from robogym_b200 import engine

    cfg = bench.CONFIGS[args.config]
    if cfg.get("workload"):
        raise SystemExit("stage_profile: dactyl configurations only")
    blob = bench.load_blob(cfg["asset"])
    names = json.load(open(os.path.join(ROOT, "robogym_b200", "assets", cfg["asset"] + ".names.json")))
    model = engine.DeviceModel(blob, 0)
    n = args.nenv or cfg["nenv"]
    c = cfg["caps"]
    sim = engine.BatchedSim(model, n, bench.NSUB, outputs=("site_xpos", "act_force", "ncon", "warn"), debug=True,
                            contact_capacity=c[0], row_capacity=c[1], dofs_per_contact=c[2])
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1234)
    wl = bench.Workload(sim, model, names, torch.device("cuda"), gen)
    acc = np.zeros(16)
    for _ in range(args.steps):
        wl.apply_action(wl.sample_action())
        sim.step()
        torch.cuda.synchronize()
        acc += sim.dbg.cpu().numpy()[:, -16:].mean(0)
        wl.auto_reset()
    acc /= args.steps
    tot = acc[:9].sum()
    rows = {nm: acc[i] for i, nm in enumerate(NAMES)}
    rows.update({nm: acc[9 + i] for i, nm in enumerate(SUB[args.level]) if nm != "-"})
    print(json.dumps(dict(config=args.config, level=args.level, nenv=n, launch=sim.launch_info(), device=torch.cuda.get_device_name(0),
                          ncon_mean=float(sim.ncon.float().mean().item()), total_cycles=float(tot),
                          cycles={k: round(float(v)) for k, v in rows.items()},
                          share_pct={k: round(100 * float(v) / max(tot, 1), 1) for k, v in rows.items()})))


if __name__ == "__main__":
    main()
