"""Step time of the bench workload (GAIL hopper, 1024 replicas, batch 256, tf32x3, CUDA graphs) with uniform hyper-parameters against the same
program running a 1024-way per-replica grid (32 learning rates x 32 discounts, Trainer(per_replica=...)), both in one process, alternating
timed windows after a warm-up, so the comparison sees the same clocks. Prints one JSON line with the card name and power limit.

  python scripts/sweep_bench.py [--steps 50] [--rounds 5]
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
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    name, power = (x.strip() for x in out.split(','))
    return dict(card=name, power_limit=power)
  except Exception as e:  # the numbers are still printed; the card fields say why they are missing
    return dict(card=None, power_limit=None, card_error=str(e))


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--replicas', type=int, default=1024)
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
  R = a.replicas
  side = int(round(R ** 0.5))
  assert side * side == R, 'the grid is square: --replicas must be a square number'
  total = a.start + (a.rounds + 1) * a.steps + 10
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={total}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5',
                     f'replicas={R}', 'gemm_mode=tf32x3', f'memory.size={max(total * 2, 4096)}', 'seed=0'])
  lrs = np.geomspace(1e-4, 1e-3, side).tolist()
  discounts = np.linspace(0.9, 0.999, side).tolist()
  grid = {'training.learning_rate': [lr for lr in lrs for _ in discounts], 'reinforcement.discount': [d for _ in lrs for d in discounts]}
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
  out = dict(workload=f'GAIL hopper, {R} replicas, batch {a.batch_size}, tf32x3, CUDA graphs; grid = {side} learning rates x {side} discounts', **card())
  for k, ts in times.items():
    med = float(np.median(ts))
    out[k] = dict(step_ms_median=med * 1e3, step_ms_min=min(ts) * 1e3, step_ms_max=max(ts) * 1e3, env_steps_per_s=R / med)
  out['grid_over_uniform'] = out['grid']['step_ms_median'] / out['uniform']['step_ms_median']
  print(json.dumps(out))


if __name__ == '__main__':
  main()
