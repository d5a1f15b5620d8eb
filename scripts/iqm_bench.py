"""Times the seed-sweep statistics (il_b200.results) on the device and their float64 numpy restatement (oracle/iqm.py) on the host cores,
at the reference's protocol (10 runs x 4 envs x 100 evaluation points, 50 000 bootstrap reps) and at 1024 runs x 4 envs x 100 points,
50 000 reps. Prints one JSON line with the card's name, power limit and clocks read in the same run.

Device: CUDA events around the two launches alone (il_bootstrap_iqm: sort set-up + resample IQMs into the [reps, T] distribution;
il_percentile_interval: the [2, T] interval, left on the device), with scores, workspace and outputs already resident; median of --repeats
timed calls after a warm-up call. End to end: host wall time of results.get_interval_estimates (upload, point estimate, bootstrap,
interval, copies back), ending in a device synchronise. Host: the numpy restatement over host-drawn indices at --host-reps reps (a count it
finishes in seconds), with its per-rep time scaled to 50 000 reps and labelled as such. The card's clocks are read right after each
size's device loops.

  python scripts/iqm_bench.py [--reps 50000] [--repeats 5] [--host-reps 200]
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
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()[0]
    name, power, sm, sm_max = (x.strip() for x in out.split(','))
    return dict(card=name, power_limit=power, sm_clock=sm, sm_clock_max=sm_max)
  except Exception as e:  # the numbers are still printed; the card fields say why they are missing
    return dict(card=f'unknown ({e})')


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--reps', type=int, default=50000)
  p.add_argument('--points', type=int, default=100)
  p.add_argument('--repeats', type=int, default=5)
  p.add_argument('--host-reps', type=int, default=200)
  a = p.parse_args()
  import numpy as np
  import torch
  from il_b200 import _lib, results
  from oracle import iqm
  if not torch.cuda.is_available(): raise SystemExit('iqm_bench needs a CUDA device')
  lib, h, st = _lib.lib(), _lib.handle(), _lib.stream()
  line = dict(reps=a.reps, points=a.points, sizes={})
  for runs, envs in ((10, 4), (1024, 4)):
    rng = np.random.default_rng(runs)
    scores = rng.random((runs, envs, a.points))
    T = a.points
    dx = torch.from_numpy(np.ascontiguousarray(scores.transpose(2, 1, 0))).cuda()  # [T, envs, runs], as results.bootstrap_iqm uploads it
    nb = lib.il_bootstrap_iqm_workspace_bytes(T, envs, runs)
    ws = torch.empty(nb, dtype=torch.uint8, device='cuda')
    dist = torch.empty(a.reps, T, dtype=torch.float64, device='cuda')
    ci = torch.empty(2, T, dtype=torch.float64, device='cuda')
    q_lo, q_hi = results.interval_percentiles(0.95)

    def launch(seed):
      _lib.check(lib.il_bootstrap_iqm(h, dx.data_ptr(), T, envs, runs, a.reps, seed, None, dist.data_ptr(), ws.data_ptr(), nb, st))

    def interval():
      _lib.check(lib.il_percentile_interval(h, dist.data_ptr(), a.reps, T, q_lo, q_hi, ci.data_ptr(), st))
    launch(1)  # warm-up: module load, first launches
    interval()
    torch.cuda.synchronize()
    boot_ms, ci_ms = [], []
    for i in range(a.repeats):
      e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
      e0.record()
      launch(2 + i)
      e1.record()
      interval()
      e2.record()
      torch.cuda.synchronize()
      boot_ms.append(e0.elapsed_time(e1))
      ci_ms.append(e1.elapsed_time(e2))
    wall = []
    for i in range(a.repeats):
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      _, cis = results.get_interval_estimates({'x': scores}, reps=a.reps, seed=10 + i)
      torch.cuda.synchronize()
      wall.append((time.perf_counter() - t0) * 1e3)
    clk = card()  # right after the device work of this size, before the host timing
    hr = a.host_reps if runs * envs <= 256 else max(1, a.host_reps // 10)
    idx = iqm.stratified_indices(rng, hr, a.points, envs, runs)
    t0 = time.perf_counter()
    iqm.percentile_interval(iqm.bootstrap_iqm(scores, idx))
    host_s = time.perf_counter() - t0
    line['sizes'][f'{runs}x{envs}'] = dict(device_bootstrap_ms=float(np.median(boot_ms)), device_interval_ms=float(np.median(ci_ms)),
                                           device_total_ms_min_max=[min(b + c for b, c in zip(boot_ms, ci_ms)), max(b + c for b, c in zip(boot_ms, ci_ms))],
                                           get_interval_estimates_wall_ms=float(np.median(wall)), host_numpy_reps=hr, host_numpy_s=host_s,
                                           host_numpy_s_scaled_to_reps=host_s / hr * a.reps, host_cores=os.cpu_count(),
                                           finite=bool(torch.isfinite(ci).all()) and bool(np.isfinite(cis['x']).all()), sm_clock_after=clk.get('sm_clock'))
  line = dict(clk, **line)
  print(json.dumps(line), flush=True)


if __name__ == '__main__':
  main()
