"""Step time of AdRIL and PWIL (hopper, batch 256, tf32x3, CUDA graphs, fast_init) with uniform values of their own search-space keys against the
same program running the reference's grid over them, at equal replica counts:
  * AdRIL: 14 jobs (imitation.balanced true / false x imitation.update_freq 0, 1250, 2500, 5000, 12500, 25000, 50000) of 72 replicas each,
    1008 replicas, against 1008 replicas at the defaults (balanced, update_freq 1250);
  * PWIL: 9 jobs (imitation.reward_scale 1 / 5 / 10 x imitation.reward_bandwidth_scale 1 / 5 / 10) of 112 replicas each, 1008 replicas,
    against 1008 replicas at the defaults (5, 5).
All four Trainers live in one process and alternate timed windows after a warm-up, so each comparison sees the same clocks. Prints one JSON
line with the card name, power limit and clocks.

  python scripts/adril_pwil_sweep_bench.py [--steps 50] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ADRIL_FREQS = (0, 1250, 2500, 5000, 12500, 25000, 50000)
PWIL_SCALES = (1.0, 5.0, 10.0)


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
  p.add_argument('--adril-per-job', type=int, default=72, help='replicas per job of the 14-job AdRIL grid')
  p.add_argument('--pwil-per-job', type=int, default=112, help='replicas per job of the 9-job PWIL grid')
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
  total = a.start + (a.rounds + 1) * a.steps + 10
  base = ['env=hopper', f'steps={total}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5', 'gemm_mode=tf32x3',
          f'memory.size={max(total * 2, 4096)}', 'seed=0']
  adril_jobs = [(b, f) for b in (True, False) for f in ADRIL_FREQS]
  pwil_jobs = [(s, w) for s in PWIL_SCALES for w in PWIL_SCALES]
  Ra, Rp = len(adril_jobs) * a.adril_per_job, len(pwil_jobs) * a.pwil_per_job
  rep = lambda jobs, i, n: [j[i] for j in jobs for _ in range(n)]
  cfg_a, cfg_p = load_config(['algorithm=AdRIL', f'replicas={Ra}'] + base), load_config(['algorithm=PWIL', f'replicas={Rp}'] + base)
  arms = dict(adril_uniform=Trainer(cfg_a, replicas=Ra, fast_init=True),
              adril_grid=Trainer(cfg_a, replicas=Ra, fast_init=True, per_replica={'imitation.balanced': rep(adril_jobs, 0, a.adril_per_job),
                                                                                 'imitation.update_freq': rep(adril_jobs, 1, a.adril_per_job)}),
              pwil_uniform=Trainer(cfg_p, replicas=Rp, fast_init=True),
              pwil_grid=Trainer(cfg_p, replicas=Rp, fast_init=True, per_replica={'imitation.reward_scale': rep(pwil_jobs, 0, a.pwil_per_job),
                                                                                'imitation.reward_bandwidth_scale': rep(pwil_jobs, 1, a.pwil_per_job)}))
  for k in ('adril_grid', 'pwil_grid'): assert len(arms[k].per_replica) == 2, k
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
  out = dict(workload=f'hopper, batch {a.batch_size}, tf32x3, CUDA graphs, fast_init; AdRIL: {Ra} replicas, grid = 14 jobs (balanced x update_freq) x '
                      f'{a.adril_per_job}, uniform = defaults; PWIL: {Rp} replicas, grid = 9 jobs (reward_scale x reward_bandwidth_scale) x {a.pwil_per_job}, '
                      f'uniform = defaults', **card())
  for k, ts in times.items():
    med = float(np.median(ts))
    R = Ra if k.startswith('adril') else Rp
    out[k] = dict(step_ms_median=med * 1e3, step_ms_min=min(ts) * 1e3, step_ms_max=max(ts) * 1e3, env_steps_per_s=R / med)
  for alg in ('adril', 'pwil'): out[f'{alg}_grid_over_uniform'] = out[f'{alg}_grid']['step_ms_median'] / out[f'{alg}_uniform']['step_ms_median']
  print(json.dumps(out))


if __name__ == '__main__':
  main()
