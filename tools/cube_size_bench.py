"""Throughput of dactyl/full_perpendicular with and without the cube-size randomisation (FullCubeRandomizer(cube_size_range=...)).

    python tools/cube_size_bench.py [--nenv 4096] [--steps 10] [--warmup 3] [--rounds 3]

Both arms run bench.py's full_perpendicular workload (4096 environments, capacities 96 / 288 / 32, relative random actions, cubes
that leave the palm are reset) with the randomisation stack of `bench.py --randomize` applied once and its per-step timestep and wind
draws; the second arm adds cube_size_range=(0.95, 1.05), i.e. per-environment body_pos, geom_rbound and mesh_scale rows and the device
set_const.  The arms alternate `--rounds` times in one process; each round times `--steps` env-steps with CUDA events around the step
launch only.  Prints one JSON line with the GPU's name and power limit beside the env-steps/s of every round."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.abspath(os.path.join(HERE, ".."))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def gpu_info():
    try:
        out = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], text=True).strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return dict(gpu=name, power_limit=limit)
    except (OSError, subprocess.CalledProcessError, IndexError, ValueError):
        return dict(gpu="unknown", power_limit="unknown")


def run_arm(nenv, steps, warmup, cube_size_range, seed=77):
    import torch

    import bench
    from robogym_b200 import engine
    from robogym_b200.locked_env import TorchRand
    from robogym_b200.randomization import FullCubeRandomizer

    cfg = bench.CONFIGS["full_perpendicular"]
    dev = torch.device("cuda", 0)
    blob = bench.load_blob(cfg["asset"])
    names = json.load(open(os.path.join(ROOT, "robogym_b200", "assets", cfg["asset"] + ".names.json")))
    model = engine.DeviceModel(blob, 0)
    caps = cfg["caps"]
    sim = engine.BatchedSim(model, nenv, bench.NSUB, outputs=("site_xpos", "act_force", "ncon", "warn"),
                            contact_capacity=caps[0], row_capacity=caps[1], dofs_per_contact=caps[2])
    gen = torch.Generator(device=dev)
    gen.manual_seed(1234)
    wl = bench.Workload(sim, model, names, dev, gen)
    R = FullCubeRandomizer(model.host, names, TorchRand(torch, dev, seed), torch, dev, torch.float32, cube_size_range=cube_size_range)
    R.apply(sim, R.sample(nenv))
    ts, wind = R.timestep_state(nenv), R.wind_state(nenv, sim.n_substeps * R.timestep0)
    timestep, xfrc = sim.enable_per_env_timestep(), sim.enable_xfrc()

    def one(timed):
        wl.apply_action(wl.sample_action())
        timestep.copy_(R.next_timestep(ts))
        R.next_wind(wind, xfrc)
        ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) if timed else None
        if ev:
            ev[0].record()
        wl.step_timed()
        if ev:
            ev[1].record()
        wl.auto_reset()
        return ev

    for _ in range(warmup):
        one(False)
    torch.cuda.synchronize()
    evs = [one(True) for _ in range(steps)]
    torch.cuda.synchronize()
    sec = sum(a.elapsed_time(b) for a, b in evs) / 1e3
    warn = int(sim.warn.max().item())
    info = sim.launch_info()
    return dict(env_steps_per_s=nenv * steps / sec, warn=warn, ctas=info["ctas"], warps_per_cta=info["warps_per_cta"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--nenv", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    from robogym_b200 import build

    build.build()
    res = {"without": [], "with": []}
    for _ in range(a.rounds):
        for key, rng in (("without", None), ("with", (0.95, 1.05))):
            res[key].append(run_arm(a.nenv, a.steps, a.warmup, rng))
    out = dict(config="full_perpendicular", nenv=a.nenv, steps=a.steps, **gpu_info(), rounds=res,
               median_without=statistics.median(r["env_steps_per_s"] for r in res["without"]),
               median_with=statistics.median(r["env_steps_per_s"] for r in res["with"]))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
