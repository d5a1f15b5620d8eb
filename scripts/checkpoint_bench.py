"""Checkpoint size, save time and load time (checkpoint.interval, il_b200/checkpoint.py) for two workloads, and the interval at which saving
costs under 1 % of the training time:

* bench: bench.py's flagship workload, GAIL on hopper with 1024 replicas and memory.size 4096;
* sweep: a 10-seed sweep (per-replica seeds) of GAIL on hopper with memory.size 1 000 000, as after 1 M steps.

Each replay ring is marked full before the timing, so a checkpoint holds every row as it does once a run has taken memory.size steps (what a
checkpoint costs does not depend on the values in the rows). Save: Trainer.checkpoint_state() and checkpoint.save() to a temporary directory,
fsync included. Load: checkpoint.load() (sha256 check included) and load_checkpoint_state() into a freshly constructed Trainer (its
construction not timed). Step time: the mean of `--steps` training steps (rollout + update, CUDA graphs) after `--warmup`, ended by a device
synchronise. Prints one JSON line per workload with the card's name, power limit and maximum SM clock.

  python scripts/checkpoint_bench.py [--workloads bench,sweep] [--repeats 3] [--steps 200] [--warmup 50]
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import il_b200  # noqa: E402
from il_b200 import checkpoint  # noqa: E402
from il_b200.config import load_config  # noqa: E402
from il_b200.train import Trainer  # noqa: E402

WORKLOADS = {
    'bench': (['algorithm=GAIL', 'env=hopper', 'replicas=1024', 'memory.size=4096', 'steps=1000000', 'training.start=1'], None),
    'sweep': (['algorithm=GAIL', 'env=hopper', 'replicas=10', 'memory.size=1000000', 'steps=1000000', 'training.start=1'], {'seed': list(range(10))}),
}


def card() -> dict:
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True)
  name, power, clock = ([x.strip() for x in q.stdout.splitlines()[0].split(',')] + ['?', '?', '?'])[:3] if q.returncode == 0 and q.stdout.strip() else (torch.cuda.get_device_name(), '?', '?')
  return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def measure(name: str, repeats: int, steps: int, warmup: int) -> dict:
  args, per_replica = WORKLOADS[name]
  cfg = load_config(args)
  tr = Trainer(cfg, per_replica=per_replica)
  for _ in range(warmup): tr.train_step()
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(steps): tr.train_step()
  torch.cuda.synchronize()
  step_s = (time.perf_counter() - t0) / steps
  tr.memory._full.fill_(1)  # every row counts, as once memory.size steps have been taken
  work = tempfile.mkdtemp(prefix='il_ckpt_')
  saves, loads, size = [], [], 0
  try:
    fresh = Trainer(load_config(args), per_replica=per_replica)
    for i in range(repeats):
      d = os.path.join(work, f'r{i}')
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      path = checkpoint.save(d, tr.step, tr.checkpoint_state(), dict(config=cfg, overrides=args, replicas=tr.R))
      saves.append(time.perf_counter() - t0)
      size = sum(os.path.getsize(os.path.join(path, f)) for f in os.listdir(path))
      t0 = time.perf_counter()
      _, state = checkpoint.load(d)
      fresh.step, fresh.graphs = 0, {}
      fresh.load_checkpoint_state(state)
      torch.cuda.synchronize()
      loads.append(time.perf_counter() - t0)
      del state
      shutil.rmtree(d)
  finally:
    shutil.rmtree(work, ignore_errors=True)
  save_s, load_s = statistics.median(saves), statistics.median(loads)
  return dict(workload=name, replicas=tr.R, memory_size=int(cfg.memory.size), checkpoint_bytes=size, save_s=save_s, load_s=load_s, saves_s=saves, loads_s=loads,
              step_s=step_s, interval_for_1pct=int(-(-100 * save_s // step_s)), **card())


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--workloads', default='bench,sweep')
  p.add_argument('--repeats', type=int, default=3)
  p.add_argument('--steps', type=int, default=200)
  p.add_argument('--warmup', type=int, default=50)
  a = p.parse_args()
  if not torch.cuda.is_available(): raise SystemExit('checkpoint_bench needs a CUDA device')
  for w in a.workloads.split(','):
    print(json.dumps(measure(w, a.repeats, a.steps, a.warmup)), flush=True)
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
