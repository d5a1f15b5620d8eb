"""Seed sweeps on the bench workload (GAIL hopper, batch 256, 256x2 actor / critic, tf32x3, CUDA graphs). Two measurements, one JSON line:

1. step time: 1024 replicas with per-replica seeds (the keyed RNG path, Trainer(per_replica={'seed': ...})) against 1024 uniform replicas, both
   in one process, alternating timed windows after a warm-up so both arms see the same clocks; medians with min / max over the windows.
2. wall time: a 10-seed sweep (`train.py -m seed=0,...,9`) as one program against the same 10 runs one after another (`train.py seed=s`), each
   with a short training run and one evaluation; both include the set-up a user pays (expert data, initialisation, graph capture).

The card's name, power limit and SM clock are read in the same run.

  python scripts/seed_sweep_bench.py [--steps 50] [--rounds 5] [--sweep-steps 600]
"""
import argparse
import contextlib
import json
import os
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = (x.strip() for x in out.split(','))
    return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
  except Exception as e:  # the numbers are still printed; the card fields say why they are missing
    return dict(card=None, power_limit=None, sm_clock=None, card_error=str(e))


def step_times(a):
  import numpy as np
  import torch
  from il_b200.config import load_config
  from il_b200.train import Trainer
  R = a.replicas
  total = a.start + (a.rounds + 1) * a.steps + 10
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={total}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5',
                     f'replicas={R}', 'gemm_mode=tf32x3', f'memory.size={max(total * 2, 4096)}', 'seed=0'])
  # per-replica seeds initialise every replica from its own stream (fast_init is refused); the uniform arm's weights do not change its step time
  arms = dict(uniform=Trainer(cfg, replicas=R, fast_init=True), per_replica_seeds=Trainer(cfg, replicas=R, per_replica={'seed': [1000 + 17 * r for r in range(R)]}))
  assert arms['per_replica_seeds'].seeds is not None and arms['uniform'].seeds is None
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
  out['per_replica_seeds_over_uniform'] = out['per_replica_seeds']['step_ms_median'] / out['uniform']['step_ms_median']
  del arms
  torch.cuda.empty_cache()
  return out


def sweep_wall(a):
  import torch
  from il_b200.train import main
  seeds = list(range(a.seeds))
  base = ['algorithm=GAIL', 'env=hopper', f'steps={a.sweep_steps}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5',
          'gemm_mode=tf32x3', f'evaluation.interval={a.sweep_steps}', 'evaluation.episodes=1', f'logging.interval={a.sweep_steps}']
  out = {}
  with tempfile.TemporaryDirectory() as tmp, open(os.devnull, 'w') as quiet, contextlib.redirect_stdout(quiet):  # the runs' own console lines
    main(base + ['seed=0', f'output_dir={tmp}/warm'])  # module loads and first-call costs, paid by neither arm
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    main(['-m'] + base + ['seed=' + ','.join(map(str, seeds)), f'output_dir={tmp}/sweep'])
    torch.cuda.synchronize()
    out['one_program_s'] = time.perf_counter() - t0
    t0 = time.perf_counter()
    for s in seeds: main(base + [f'seed={s}', f'output_dir={tmp}/single{s}'])
    torch.cuda.synchronize()
    out['sequential_programs_s'] = time.perf_counter() - t0
  out['speed_up'] = out['sequential_programs_s'] / out['one_program_s']
  return dict(workload=f'{a.seeds}-seed sweep, {a.sweep_steps} steps (start {a.start}), one evaluation episode', **out)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--replicas', type=int, default=1024)
  p.add_argument('--batch-size', type=int, default=256)
  p.add_argument('--start', type=int, default=300)
  p.add_argument('--steps', type=int, default=50, help='timed steps per window')
  p.add_argument('--rounds', type=int, default=5, help='alternating windows per arm')
  p.add_argument('--seeds', type=int, default=10)
  p.add_argument('--sweep-steps', type=int, default=600, help='training steps of each run of the wall-time comparison')
  a = p.parse_args()
  import il_b200  # noqa: F401
  out = dict(workload=f'GAIL hopper, batch {a.batch_size}, tf32x3, CUDA graphs', **card())
  out['step_time'] = dict(replicas=a.replicas, **step_times(a))
  out['sweep_wall_time'] = sweep_wall(a)
  out.update({k + '_after': v for k, v in card().items() if k.startswith('sm_clock')})
  print(json.dumps(out))


if __name__ == '__main__':
  main()
