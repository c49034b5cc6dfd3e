"""What the robot's part of the rearrange reset costs on the device: initialize_sim_state + randomize_initial_position (one held
random action for 10 env-steps, one zero-action controller step, 100 zero-action env-steps) on a 2048-environment
rearrange_blocks5_tcp batch (ControlMode.TCP_ROLL_YAW, arm_reset_controller_error) for 1, 16, 128 and 2048 resetting
environments; and the unmasked controller env-step of the whole batch through the kernel (rg_arm_phase) and through the
float32 tensor path it replaces, alternated round by round in one run.

CUDA events around each call, after a warm-up of every shape.  The card's name, power limit and SM clock limit are read in the
same run.  Writes a JSON line to stdout (and to --out if given).

    python tools/robot_reset_bench.py [--rounds 3] [--steps 20] [--out robot_reset_bench.json]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NENV = 2048
CAPS = dict(contact_capacity=64, row_capacity=160, dofs_per_contact=16)   # bench.py's rearrange_blocks_tcp


def card():
    import torch

    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return dict(device=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out")
    args = ap.parse_args()

    import torch

    from robogym_b200 import build, engine
    from robogym_b200.rearrange_arm import BatchedTcpArmController

    build.build()
    dev = torch.device("cuda", 0)
    blobs = [open(os.path.join(ROOT, "robogym_b200", "assets", n + ".rgm"), "rb").read() for n in ("rearrange_blocks5_tcp", "rearrange_solver_arm")]
    main_sim = engine.BatchedSim(engine.DeviceModel(blobs[0], 0), NENV, 40, outputs=("site_xpos", "act_force", "ncon", "warn", "body_xpos", "body_xquat"), **CAPS)
    solver = engine.BatchedSim(engine.DeviceModel(blobs[1], 0), NENV, 40, outputs=("body_xpos", "body_xquat", "warn"))
    ctl = BatchedTcpArmController(main_sim, solver, max_position_change=0.1, reset_controller_error=True)
    ctl.initialize_sim_state()
    main_sim.forward()
    ctl.reset()
    g = torch.Generator(device=dev)
    g.manual_seed(0)
    acts = [torch.rand(NENV, 6, device=dev, generator=g) * 2 - 1 for _ in range(args.steps)]

    def timed(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    counts = (1, 16, 128, 2048)
    rng = np.random.RandomState(1)
    masks = {}
    for n in counts:
        m = np.zeros(NENV, dtype=np.uint8)
        m[rng.choice(NENV, n, replace=False)] = 1
        masks[n] = torch.as_tensor(m, device=dev)

    def reset(n, epoch):
        ctl.initialize_sim_state(masks[n])
        ctl.randomize_initial_position(masks[n], seed=3, epoch=epoch)

    def steps(path):
        for a in acts:
            if path == "kernel":
                ctl.step(a)
            else:
                ctl._step_torch(a, ctl.main_forwards)

    for n in counts:                      # warm-up of every shape
        reset(n, 0)
    steps("kernel"); steps("torch")
    res = {f"reset_ms_{n}": [] for n in counts}
    res.update(step_ms_kernel=[], step_ms_torch=[])
    for r in range(args.rounds):
        for n in counts:
            res[f"reset_ms_{n}"].append(timed(lambda: reset(n, r + 1)))
        for path in (("kernel", "torch") if r % 2 == 0 else ("torch", "kernel")):
            res[f"step_ms_{path}"].append(timed(lambda: steps(path)) / args.steps)
    out = dict(tool="robot_reset_bench", nenv=NENV, rounds=args.rounds, steps=args.steps, card=card(), warn=int(max(main_sim.warn.max().item(), solver.warn.max().item())),
               median={k: float(np.median(v)) for k, v in res.items()}, samples=res)
    line = json.dumps(out)
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
