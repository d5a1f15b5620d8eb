"""Cost of sweeping the general GAIL discriminator's choices (csrc/gail_general.cu) as replicas of one program, on a depth-2 tanh discriminator
(GAIL hopper, batch 256, tf32x3, CUDA graphs). Two measurements:

1. Step time: an 18-job grid (loss function BCE / Mixup / PUGAIL x reward function GAIL / AIRL / FAIRL x spectral norm on / off) of 56 replicas
   per job, 1008 replicas in all, as one Trainer(per_replica=...), against 1008 replicas at the defaults (BCE, AIRL, spectral norm). Both live
   in one process and alternate timed windows after a warm-up, so the comparison sees the same clocks; medians are reported. A group that mixes
   Mixup with BCE / PUGAIL runs the policy, expert and Mixup passes for every replica (each replica's dead passes are masked out), so the grid
   arm does three loss passes where the uniform arm does two.
2. Wall time of the same 18-job sweep at `--wall-replicas` replicas per job, end to end (construction, prefill, graph capture, every step):
   one program of 18 x R replicas against 18 programs of R replicas run one after another, as run_sweep ran them before.

Prints one JSON line with the card name, power limit and clocks.

  python scripts/gailx_choice_sweep_bench.py [--steps 50] [--rounds 5] [--wall-steps 400]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from scripts.gail_choice_sweep_bench import card  # noqa: E402

GENERAL = ['imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh']
JOBS = [(l, rf, sn) for l in ('BCE', 'Mixup', 'PUGAIL') for rf in ('GAIL', 'AIRL', 'FAIRL') for sn in (True, False)]
KEYS = ('imitation.loss_function', 'imitation.discriminator.reward_function', 'imitation.spectral_norm')


def _cfg(R, steps, start, B, extra=()):
  from il_b200.config import load_config
  return load_config(['algorithm=GAIL', 'env=hopper', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=5', f'replicas={R}',
                      'gemm_mode=tf32x3', f'memory.size={max(steps * 2, 4096)}', 'seed=0', *GENERAL, *extra])


def step_times(a):
  import numpy as np
  import torch
  from il_b200.train import Trainer
  R = len(JOBS) * a.per_job
  total = a.start + (a.rounds + 1) * a.steps + 10
  cfg = _cfg(R, total, a.start, a.batch_size)
  grid = {k: [j[i] for j in JOBS for _ in range(a.per_job)] for i, k in enumerate(KEYS)}
  arms = dict(uniform=Trainer(cfg, replicas=R, fast_init=True), grid=Trainer(cfg, replicas=R, fast_init=True, per_replica=grid))
  assert all(tr.discriminator.general for tr in arms.values())
  for tr in arms.values():  # prefill and warm-up (graph capture of both step kinds)
    for _ in range(a.start + 5): tr.train_step()
  torch.cuda.synchronize()
  times = {k: [] for k in arms}
  for _ in range(a.rounds):
    for k, tr in arms.items():
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      for _ in range(a.steps): tr.train_step()
      torch.cuda.synchronize()
      times[k].append((time.perf_counter() - t0) / a.steps)
  out = {}
  for k, ts in times.items():
    med = float(np.median(ts))
    out[k] = dict(step_ms_median=med * 1e3, step_ms_min=min(ts) * 1e3, step_ms_max=max(ts) * 1e3, env_steps_per_s=R / med)
  out['grid_over_uniform'] = out['grid']['step_ms_median'] / out['uniform']['step_ms_median']
  del arms
  torch.cuda.empty_cache()
  return R, out


def wall_times(a):
  import torch
  from il_b200.train import Trainer
  R = a.wall_replicas

  def run(cfg, **kw):
    tr = Trainer(cfg, replicas=cfg.replicas, **kw)
    for _ in range(cfg.steps): tr.train_step()
    torch.cuda.synchronize()

  t0 = time.perf_counter()
  run(_cfg(len(JOBS) * R, a.wall_steps, a.wall_start, a.batch_size), per_replica={k: [j[i] for j in JOBS for _ in range(R)] for i, k in enumerate(KEYS)})
  one = time.perf_counter() - t0
  t0 = time.perf_counter()
  for j in JOBS: run(_cfg(R, a.wall_steps, a.wall_start, a.batch_size, [f'{k}={str(v).lower() if isinstance(v, bool) else v}' for k, v in zip(KEYS, j)]))
  many = time.perf_counter() - t0
  return dict(replicas_per_job=R, steps=a.wall_steps, start=a.wall_start, one_program_s=one, programs_18_s=many, speedup=many / one)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--per-job', type=int, default=56, help='replicas per job of the 18-job grid (step-time arms)')
  p.add_argument('--batch-size', type=int, default=256)
  p.add_argument('--start', type=int, default=300)
  p.add_argument('--steps', type=int, default=50, help='timed steps per window')
  p.add_argument('--rounds', type=int, default=5, help='alternating windows per arm')
  p.add_argument('--wall-replicas', type=int, default=1, help='replicas per job of the wall-time sweep')
  p.add_argument('--wall-steps', type=int, default=400)
  p.add_argument('--wall-start', type=int, default=200)
  a = p.parse_args()
  import torch
  import il_b200  # noqa: F401
  assert torch.cuda.is_available(), 'this benchmark times the GPU program; it needs a CUDA device'
  R, steps = step_times(a)
  out = dict(workload=f'GAIL hopper, depth-2 tanh discriminator, batch {a.batch_size}, tf32x3, CUDA graphs; grid = 18 jobs (loss x reward function x spectral norm); '
                      f'step time at {R} replicas (fast_init) against {R} uniform replicas', **card(), step=steps, wall=wall_times(a))
  print(json.dumps(out))


if __name__ == '__main__':
  main()
