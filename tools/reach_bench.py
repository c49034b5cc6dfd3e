"""Throughput of the batched dactyl/reach environment (robogym_b200.reach_env.BatchedReachEnv.step) with auto-reset, and what the goal
simulation costs (FingertipPosGoal.next_goal: one masked forward and two masked steps for the environments that draw a goal), twice:
`goal_launch_ms_per_step` is the time between CUDA events recorded around each of the goal simulation's three launch calls, i.e. the
launches alone; `goal_path_ms_per_step` is the time between events around the whole goal-draw path, which also holds the host
synchronisations that select the drawing environments and the tensor work around the launches.  Nominal and randomised environments are timed in alternated rounds with CUDA events after a warm-up; the card's
name, power limit and maximum SM clock are read in the same run.  Usage: python tools/reach_bench.py [nenv] [steps] [rounds]"""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from robogym_b200 import build  # noqa: E402
from robogym_b200.reach_env import make_cuda_env  # noqa: E402

build.build()
nenv = int(sys.argv[1]) if len(sys.argv) > 1 else 8192
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 100
rounds = int(sys.argv[3]) if len(sys.argv) > 3 else 4
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()

envs, goal_events = {}, {}


def timed(fn, events):
    def call(*args, **kw):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn(*args, **kw)
        b.record()
        events.append((a, b))
    return call


for label, kw in (("nominal", {}), ("randomize", dict(randomize=True))):
    env = make_cuda_env(nenv, seed=0, **kw)
    env.reset()
    goal_events[label] = dict(path=[], launch=[])
    env._draw_goals = timed(env._draw_goals, goal_events[label]["path"])
    env.goal_sim.step = timed(env.goal_sim.step, goal_events[label]["launch"])     # BatchedSim.forward(mask=...) launches through step()
    envs[label] = env
gen = torch.Generator(device="cuda")
gen.manual_seed(1)
for env in envs.values():                  # warm-up: every shape of the timed window, goal draws included
    for _ in range(20):
        env.step(torch.rand(nenv, 20, device=env.device, generator=gen) * 2 - 1)
torch.cuda.synchronize()

res = {label: dict(ms_per_step=[], path=[], launch=[], goals_per_step=[]) for label in envs}
for r in range(rounds):
    order = list(envs) if r % 2 == 0 else list(envs)[::-1]
    for label in order:
        env = envs[label]
        acts = [torch.rand(nenv, 20, device=env.device, generator=gen) * 2 - 1 for _ in range(steps)]
        for v in goal_events[label].values():
            v.clear()
        launches0 = env.goal_launches
        torch.cuda.synchronize()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for a in acts:
            env.step(a)
        t1.record()
        torch.cuda.synchronize()
        res[label]["ms_per_step"].append(t0.elapsed_time(t1) / steps)
        for key in ("path", "launch"):
            res[label][key].append(sum(a.elapsed_time(b) for a, b in goal_events[label][key]) / steps)
        res[label]["goals_per_step"].append((env.goal_launches - launches0) / 3 / steps)
out = dict(card=card, nenv=nenv, steps=steps, rounds=rounds)
for label, v in res.items():
    ms = statistics.median(v["ms_per_step"])
    lms, pms = statistics.median(v["launch"]), statistics.median(v["path"])
    out[label] = dict(env_steps_per_s=nenv / ms * 1e3, ms_per_step=ms, ms_per_step_rounds=[round(x, 3) for x in v["ms_per_step"]],
                      goal_launch_ms_per_step=lms, goal_launch_share=lms / ms, goal_path_ms_per_step=pms, goal_path_share=pms / ms,
                      goals_drawn_per_step=statistics.median(v["goals_per_step"]),
                      warn=[int(envs[label].sim.warn.max()), int(envs[label].goal_sim.warn.max())],
                      max_contacts=[int(envs[label].sim.ncon.max()), int(envs[label].goal_sim.ncon.max())])
print(json.dumps(out))
