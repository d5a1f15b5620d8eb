"""Step time of the bench workload (GAIL hopper, batch 256, tf32x3, CUDA graphs, fast_init) with uniform discriminator choices against the same
program running a grid over them: 18 jobs (loss function BCE / Mixup / PUGAIL x reward function GAIL / AIRL / FAIRL x spectral norm on / off,
Mixup at alpha 0.4) of 56 replicas each, 1008 replicas in all, as one Trainer(per_replica=...). The uniform arm runs 1008 replicas at the
defaults. Both live in one process and alternate timed windows after a warm-up, so the comparison sees the same clocks. Mixup replicas run one
loss pass instead of two and replicas without spectral norm skip the power iterations, so the CTAs of the grid's launches finish unevenly; the
script reports the step times it measures and nothing else. Prints one JSON line with the card name, power limit and clocks.

  python scripts/gail_choice_sweep_bench.py [--steps 50] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.mem', '--format=csv,noheader'], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()[0]
    name, power, sm, mem = (x.strip() for x in out.split(','))
    return dict(card=name, power_limit=power, sm_clock=sm, mem_clock=mem)
  except Exception as e:  # the numbers are still printed; the card fields say why they are missing
    return dict(card=None, power_limit=None, card_error=str(e))


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--per-job', type=int, default=56, help='replicas per job of the 18-job grid')
  p.add_argument('--batch-size', type=int, default=256)
  p.add_argument('--start', type=int, default=300)
  p.add_argument('--steps', type=int, default=50, help='timed steps per window')
  p.add_argument('--rounds', type=int, default=5, help='alternating windows per arm')
  a = p.parse_args()
  import numpy as np
  import torch
  import il_b200  # noqa: F401
  from il_b200.config import load_config
  from il_b200.train import Trainer
  jobs = [(l, rf, sn) for l in ('BCE', 'Mixup', 'PUGAIL') for rf in ('GAIL', 'AIRL', 'FAIRL') for sn in (True, False)]
  R = len(jobs) * a.per_job
  total = a.start + (a.rounds + 1) * a.steps + 10
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={total}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5',
                     f'replicas={R}', 'gemm_mode=tf32x3', f'memory.size={max(total * 2, 4096)}', 'seed=0', 'imitation.mixup_alpha=0.4'])
  rep = lambda i: [j[i] for j in jobs for _ in range(a.per_job)]
  grid = {'imitation.loss_function': rep(0), 'imitation.discriminator.reward_function': rep(1), 'imitation.spectral_norm': rep(2)}
  arms = dict(uniform=Trainer(cfg, replicas=R, fast_init=True), grid=Trainer(cfg, replicas=R, fast_init=True, per_replica=grid))
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
  out = dict(workload=f'GAIL hopper, {R} replicas, batch {a.batch_size}, tf32x3, CUDA graphs, fast_init; grid = 18 jobs (loss x reward function x spectral norm, '
                      f'Mixup alpha 0.4) x {a.per_job} replicas; uniform = defaults', **card())
  for k, ts in times.items():
    med = float(np.median(ts))
    out[k] = dict(step_ms_median=med * 1e3, step_ms_min=min(ts) * 1e3, step_ms_max=max(ts) * 1e3, env_steps_per_s=R / med)
  print(json.dumps(out))


if __name__ == '__main__':
  main()
