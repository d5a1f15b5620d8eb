"""RED and DRIL sweeps over the dropout rates and the activation, run as per-replica values of one program (hopper, batch 256, tf32x3, CUDA graphs):
1. step time: for each algorithm, the 8-job grid (imitation.discriminator.input_dropout 0.1 / 0.3 x dropout 0.2 / 0.5 x activation relu / tanh)
   of 126 replicas per job, 1008 replicas, against 1008 uniform replicas at the grid's first job (fast_init, discriminator pre-trained for a few
   iterations so the threshold / bandwidth exist). All four Trainers live in one process and alternate timed windows after a warm-up, so each
   comparison sees the same clocks; medians with min / max over the windows.
2. wall time: the same 8-job grid as a multirun (`train.py -m ...`, one program of 8 replicas) against its 8 jobs as separate programs one after
   another, discriminator pre-training included, for each algorithm.
Prints one JSON line with the card name, power limit and clocks.

  python scripts/red_dril_sweep_bench.py [--steps 50] [--rounds 5] [--pretrain 1000] [--sweep-steps 600]
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

KEYS = ('imitation.discriminator.input_dropout', 'imitation.discriminator.dropout', 'imitation.discriminator.activation')
GRID = [(i, d, a) for i in (0.1, 0.3) for d in (0.2, 0.5) for a in ('relu', 'tanh')]  # Hydra order: the last key varies fastest
SWEEP = [f'{k}={v}' for k, v in zip(KEYS, ('0.1,0.3', '0.2,0.5', 'relu,tanh'))]  # the same 8 jobs as a multirun command line


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
  R = len(GRID) * a.per_job
  total = a.start + (a.rounds + 1) * a.steps + 10
  base = ['env=hopper', f'steps={total}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5', f'replicas={R}',
          'gemm_mode=tf32x3', f'memory.size={max(total * 2, 4096)}', 'seed=0'] + [f'{k}={v}' for k, v in zip(KEYS, GRID[0])]
  arms = {}
  for alg in ('DRIL', 'RED'):
    cfg = load_config([f'algorithm={alg}'] + base)
    arms[f'{alg.lower()}_uniform'] = Trainer(cfg, replicas=R, fast_init=True)
    arms[f'{alg.lower()}_grid'] = Trainer(cfg, replicas=R, fast_init=True, per_replica={k: [job[i] for job in GRID for _ in range(a.per_job)] for i, k in enumerate(KEYS)})
    assert len(arms[f'{alg.lower()}_grid'].per_replica) == 3 and not arms[f'{alg.lower()}_uniform'].per_replica
  for tr in arms.values():  # pre-training (threshold / bandwidth), prefill and warm-up (graph capture of both step kinds)
    tr.pretrain_discriminator(iterations=4)
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
  out = dict(replicas=R, per_job=a.per_job)
  for k, ts in times.items():
    med = float(np.median(ts))
    out[k] = dict(step_ms_median=med * 1e3, step_ms_min=min(ts) * 1e3, step_ms_max=max(ts) * 1e3, env_steps_per_s=R / med)
  for alg in ('dril', 'red'): out[f'{alg}_grid_over_uniform'] = out[f'{alg}_grid']['step_ms_median'] / out[f'{alg}_uniform']['step_ms_median']
  del arms
  torch.cuda.empty_cache()
  return out


def sweep_wall(a):
  import torch
  from il_b200.train import main
  out = {}
  with tempfile.TemporaryDirectory() as tmp, open(os.devnull, 'w') as quiet, contextlib.redirect_stdout(quiet):  # the runs' own console lines
    for alg in ('DRIL', 'RED'):
      base = [f'algorithm={alg}', 'env=hopper', f'steps={a.sweep_steps}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5',
              'gemm_mode=tf32x3', f'evaluation.interval={a.sweep_steps}', 'evaluation.episodes=1', f'logging.interval={a.sweep_steps}',
              f'imitation.pretraining.iterations={a.pretrain}']
      jobs = [[f'{k}={v}' for k, v in zip(KEYS, job)] for job in GRID]
      main(base + jobs[0] + ['steps=20', 'imitation.pretraining.iterations=2', f'output_dir={tmp}/warm'])  # module loads and first-call costs, paid by neither arm
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      main(['-m'] + base + SWEEP + [f'output_dir={tmp}/sweep'])
      torch.cuda.synchronize()
      one = time.perf_counter() - t0
      t0 = time.perf_counter()
      for n, job in enumerate(jobs): main(base + job + [f'output_dir={tmp}/single{n}'])
      torch.cuda.synchronize()
      seq = time.perf_counter() - t0
      out[alg.lower()] = dict(one_program_s=one, sequential_programs_s=seq, speed_up=seq / one)
  return dict(workload=f'8-job sweep (input_dropout 0.1,0.3 x dropout 0.2,0.5 x activation relu,tanh), {a.pretrain} pre-training iterations, {a.sweep_steps} steps '
                       f'(start {a.start}), one evaluation episode', **out)


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--per-job', type=int, default=126, help='replicas per job of the 8-job grid in the step-time comparison')
  p.add_argument('--batch-size', type=int, default=256)
  p.add_argument('--start', type=int, default=300)
  p.add_argument('--steps', type=int, default=50, help='timed steps per window')
  p.add_argument('--rounds', type=int, default=5, help='alternating windows per arm')
  p.add_argument('--pretrain', type=int, default=1000, help='discriminator pre-training iterations of each run of the wall-time comparison')
  p.add_argument('--sweep-steps', type=int, default=600, help='training steps of each run of the wall-time comparison')
  a = p.parse_args()
  import il_b200  # noqa: F401
  out = dict(workload=f'hopper, batch {a.batch_size}, tf32x3, CUDA graphs; discriminator hidden 64 (DRIL) / 32 (RED), depth 1', **card())
  out['step_time'] = step_times(a)
  out['sweep_wall_time'] = sweep_wall(a)
  out.update({k + '_after': v for k, v in card().items() if k.startswith('sm_clock')})
  print(json.dumps(out))


if __name__ == '__main__':
  main()
