"""What the settle costs on the device: stabilize_objects (100 env-steps of 40 substeps with the object damping at 1e-3) on a
2048-environment rearrange_blocks5_tcp batch for 1, 16, 128 and 2048 resetting environments, through the settle launch
(BatchedSim.settle) and through the per-environment-row composition it replaces (dof_damping bound per environment, a masked
step, the rows restored, a masked forward); and a normal env-step of the whole batch with and without dof_damping bound per
environment, which is what a batch pays on every step to carry those rows.

CUDA events around each call, after a warm-up of every shape; the arms alternate round by round.  The card's name, power limit
and SM clock limit are read in the same run.  Writes a JSON line to stdout (and to --out if given).

    python tools/settle_bench.py [--rounds 3] [--steps 20] [--out settle_bench.json]"""
import argparse
import gzip
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

NENV, NSUB, NSTEPS = 2048, 40, 100
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

    from helpers import golden_model
    from robogym_b200 import build, engine, rearrange_scene

    build.build()
    with gzip.open(os.path.join(ROOT, "tests", "golden", "reference_settle.json.gz"), "rt") as f:
        c = json.load(f)["cases"][0]
    blob, m, names = golden_model("rearrange_blocks5_tcp", c["model"])
    model = engine.DeviceModel(blob, 0)
    dev = torch.device("cuda", 0)
    sims = {k: engine.BatchedSim(model, NENV, NSUB, outputs=("site_xpos", "ncon", "warn"), **CAPS) for k in ("const", "rows")}
    bodies = [names["body"].index(f"object{k}") for k in range(5)]
    dofs = rearrange_scene.object_dofs(m, bodies)
    rows = np.repeat(np.asarray(m["dof_damping"], dtype=np.float64)[None], NENV, 0)
    sims["rows"].set_param("dof_damping", rows)

    # every environment starts from the recorded reset with its blocks 1-4 mm higher
    st = c["state0"]
    g = torch.Generator().manual_seed(0)
    start = {}
    for k, key in (("qpos", "qpos"), ("qvel", "qvel"), ("ctrl", "ctrl"), ("pid", "pid"), ("qacc_warmstart", "warm")):
        start[k] = torch.tensor(np.asarray(st[key], dtype=np.float32)).repeat(NENV, 1)
    for a in c["qposadr"]:
        start["qpos"][:, a + 2] += 1e-3 + 3e-3 * torch.rand(NENV, generator=g)
    start = {k: v.to(dev) for k, v in start.items()}
    for s in sims.values():
        s.mocap_pos.copy_(torch.tensor(np.asarray(st["mocap_pos"], dtype=np.float32).reshape(1, -1, 3)).expand_as(s.mocap_pos))
        s.mocap_quat.copy_(torch.tensor(np.asarray(st["mocap_quat"], dtype=np.float32).reshape(1, -1, 4)).expand_as(s.mocap_quat))

    def load(s):
        for k, v in start.items():
            getattr(s, k).copy_(v)

    perm = torch.randperm(NENV, generator=g)
    masks = {}
    for n in (1, 16, 128, 2048):
        mk = torch.zeros(NENV, dtype=torch.uint8)
        mk[perm[:n]] = 1
        masks[n] = mk.to(dev)
    low = {n: rows.copy() for n in masks}
    for n, mk in masks.items():
        low[n][np.ix_(mk.cpu().numpy().astype(bool), dofs)] = 1e-3

    def settle_const(n):
        sims["const"].settle(dofs, 1e-3, NSTEPS * NSUB, mask=masks[n])

    def settle_rows(n):
        s = sims["rows"]
        s.set_param("dof_damping", low[n])
        s.step(NSTEPS * NSUB, final_forward=0, mask=masks[n])
        s.set_param("dof_damping", rows)
        s.forward(mask=masks[n])

    def timed(fn, sim_key, *a):
        load(sims[sim_key])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn(*a)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def env_steps(key):
        s = sims[key]
        for _ in range(args.steps):
            s.step()

    # warm-up: every shape once
    for n in masks:
        timed(settle_const, "const", n)
        timed(settle_rows, "rows", n)
    timed(env_steps, "const", "const")
    timed(env_steps, "rows", "rows")

    res = {f"settle_const_{n}": [] for n in masks}
    res.update({f"settle_rows_{n}": [] for n in masks})
    res.update(step_unbound=[], step_rows=[])
    for r in range(args.rounds):
        for n in masks:
            arms = [("settle_const", settle_const, "const"), ("settle_rows", settle_rows, "rows")]
            for name, fn, key in (arms if r % 2 == 0 else arms[::-1]):
                res[f"{name}_{n}"].append(timed(fn, key, n))
        arms = [("step_unbound", "const"), ("step_rows", "rows")]
        for name, key in (arms if r % 2 == 0 else arms[::-1]):
            res[name].append(timed(env_steps, key, key) / args.steps)
    out = dict(card=card(), nenv=NENV, nsub=NSUB, settle_env_steps=NSTEPS, rounds=args.rounds,
               launch_const=sims["const"].launch_info(), launch_rows=sims["rows"].launch_info(),
               ms={k: dict(median=float(np.median(v)), min=float(np.min(v)), max=float(np.max(v))) for k, v in res.items()})
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
