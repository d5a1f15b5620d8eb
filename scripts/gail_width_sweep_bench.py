"""Step time of the bench workload (GAIL hopper, batch 256, tf32x3, CUDA graphs, fast_init) with per-replica discriminator widths against uniform
widths, all arms at the same replica count (54 x 19 = 1026 by default):
  uniform64   every replica at hidden size 64 (the defaults);
  uniform128  every replica at 128;
  widths      32 / 64 / 128 in three equal blocks (three width classes, one launch each);
  widths_x_choices  the 3 widths crossed with the 18-job choice grid of gail_choice_sweep_bench.py (loss function x reward function x spectral
              norm, Mixup at alpha 0.4): 54 jobs of `--per-job` replicas.
All arms live in one process and alternate timed windows after a warm-up, so the comparison sees the same clocks. Then the il_gail_update call
alone is timed per arm with CUDA events in eager mode (alternating rounds as well). Each width class is its own launch, so a mixed-width update
adds the tail waves of every class; the script reports the times it measures and nothing else. Prints one JSON line with the card name, power
limit and clocks.

  python scripts/gail_width_sweep_bench.py [--steps 50] [--rounds 5]
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
  p.add_argument('--per-job', type=int, default=19, help='replicas per job of the 54-job widths x choices grid (every arm runs 54 x per-job replicas)')
  p.add_argument('--batch-size', type=int, default=256)
  p.add_argument('--start', type=int, default=300)
  p.add_argument('--steps', type=int, default=50, help='timed steps per window')
  p.add_argument('--rounds', type=int, default=5, help='alternating windows per arm')
  p.add_argument('--update-calls', type=int, default=50, help='eager il_gail_update calls per timed round')
  a = p.parse_args()
  import numpy as np
  import torch
  import il_b200  # noqa: F401
  from il_b200.config import load_config
  from il_b200.train import Trainer
  from il_b200.training import adversarial_imitation_update
  widths = (32, 64, 128)
  choices = [(l, rf, sn) for l in ('BCE', 'Mixup', 'PUGAIL') for rf in ('GAIL', 'AIRL', 'FAIRL') for sn in (True, False)]
  jobs = [(H, ) + c for H in widths for c in choices]
  R = len(jobs) * a.per_job
  total = a.start + (a.rounds + 1) * a.steps + 10
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={total}', f'training.start={a.start}', f'training.batch_size={a.batch_size}', 'imitation.trajectories=5',
                     f'replicas={R}', 'gemm_mode=tf32x3', f'memory.size={max(total * 2, 4096)}', 'seed=0', 'imitation.mixup_alpha=0.4'])
  W = 'imitation.discriminator.hidden_size'
  rep = lambda i: [j[i] for j in jobs for _ in range(a.per_job)]
  grid = {W: rep(0), 'imitation.loss_function': rep(1), 'imitation.discriminator.reward_function': rep(2), 'imitation.spectral_norm': rep(3)}
  blocks = [widths[r * len(widths) // R] for r in range(R)]
  arms = dict(uniform64=Trainer(cfg, replicas=R, fast_init=True), uniform128=Trainer(cfg, replicas=R, fast_init=True, per_replica={W: [128] * R}),
              widths=Trainer(cfg, replicas=R, fast_init=True, per_replica={W: blocks}), widths_x_choices=Trainer(cfg, replicas=R, fast_init=True, per_replica=grid))
  assert arms['uniform128'].discriminator.mlp.dims[1] == 128 and arms['widths'].discriminator.hidden_size_r == blocks
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

  def update_call(tr):
    adversarial_imitation_update(tr.actor, tr.discriminator, tr.batch, tr.expert_batch, tr.discriminator_optimiser, tr.imitation_cfg, eps_gp=tr.eps_gp,
                                 eps_mix=tr.eps_mix if tr._mixup_on else None, out_losses=tr.gail_losses)

  upd = {k: [] for k in arms}
  for tr in arms.values():
    tr.discriminator.train()
    for _ in range(3): update_call(tr)
  for _ in range(a.rounds):
    for k, tr in arms.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      torch.cuda.synchronize()
      e0.record()
      for _ in range(a.update_calls): update_call(tr)
      e1.record()
      torch.cuda.synchronize()
      upd[k].append(e0.elapsed_time(e1) / a.update_calls)
  out = dict(workload=f'GAIL hopper, {R} replicas, batch {a.batch_size}, tf32x3, CUDA graphs, fast_init; widths = 32 / 64 / 128 in equal blocks; widths_x_choices = '
                      f'3 widths x 18 choice jobs (loss x reward function x spectral norm, Mixup alpha 0.4) x {a.per_job} replicas; uniform64 = defaults', **card())
  for k, ts in times.items():
    med = float(np.median(ts))
    out[k] = dict(step_ms_median=med * 1e3, step_ms_min=min(ts) * 1e3, step_ms_max=max(ts) * 1e3, env_steps_per_s=R / med,
                  gail_update_eager_ms_median=float(np.median(upd[k])), gail_update_eager_ms_min=min(upd[k]), gail_update_eager_ms_max=max(upd[k]))
  print(json.dumps(out))


if __name__ == '__main__':
  main()
