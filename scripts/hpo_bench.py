"""Times the search's two CUDA launches (il_gp_posterior, il_gp_select) against a torch float64 statement of the same maths, and one search
round as grouped programs against the same trial-envs as single programs. Prints one JSON line per measurement.

`python scripts/hpo_bench.py [--sizes 30,256,1024,4096] [--M 65536] [--qs 1,64,256] [--trials 64] [--steps 60]`

Kernel times are CUDA events around the il_gp_posterior / il_gp_select launches alone (inputs, the transposed candidates, workspace and outputs
resident; var and V restored before each timed selection, outside the events), the median of 5 after a warm-up launch. The torch statement
is timed the same way around its own ops. Rates are computed from shapes:
  posterior FLOPs = M (n^2 + n (3 d + 12))   (forward substitution n^2 M, the kernel rows and the mean)
  selection bytes = sum over picks j of 8 M (n + j + d + 4)   (V rows read, the new V row, var read and written, mu, the candidate)
and compared with the H100 SXM data-sheet FP64 (34 TFLOP/s without tensor cores) and HBM3 (3.35 TB/s) figures.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import il_b200  # noqa: E402,F401
from il_b200 import _lib, hpo  # noqa: E402

DATASHEET_FP64, DATASHEET_HBM = 34e12, 3.35e12


def card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
  return q.splitlines()[0] if q else torch.cuda.get_device_name()


def timed(fn, prep=lambda: None, reps=5):
  prep()
  fn()
  ts = []
  for _ in range(reps):
    prep()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b) * 1e-3)
  return statistics.median(ts)


def torch_posterior(fit, C):
  ls = fit.lengthscales.to(C.device)
  r = torch.cdist(C / ls, fit.X / ls, compute_mode='donot_use_mm_for_euclid_dist')
  Ks = fit.outputscale * (1 + 5**0.5 * r + 5.0 / 3.0 * r * r) * torch.exp(-5**0.5 * r)
  V = torch.linalg.solve_triangular(fit.L, Ks.T, upper=False)
  return Ks @ fit.alpha, fit.outputscale - (V * V).sum(0), V


def torch_select(fit, C, mu, var, V, q, fstar):
  ls = fit.lengthscales.to(C.device)
  var, rows, picked, picks = var.clone(), [V], torch.zeros(len(C), dtype=torch.bool, device=C.device), []
  normal = torch.distributions.Normal(torch.zeros((), dtype=torch.float64, device=C.device), torch.ones((), dtype=torch.float64, device=C.device), validate_args=False)
  for _ in range(q):
    s = var.clamp_min(0).sqrt()
    z = (mu - fstar) / s
    ei = torch.where(s > 0, (mu - fstar) * normal.cdf(z) + s * normal.log_prob(z).exp(), (mu - fstar).clamp_min(0)).masked_fill(picked, -float('inf'))
    w = int(torch.argmax(ei))
    picks.append(w)
    picked[w] = True
    Vc = torch.cat(rows)
    r = torch.cdist(C / ls, C[w:w + 1] / ls, compute_mode='donot_use_mm_for_euclid_dist')[:, 0]
    c = fit.outputscale * (1 + 5**0.5 * r + 5.0 / 3.0 * r * r) * torch.exp(-5**0.5 * r) - Vc.T @ Vc[:, w]
    den = var[w] + fit.noise
    var = var - c * c / den
    rows.append((c / den.sqrt())[None])
    fstar = max(fstar, float(mu[w]))
  return picks, var


def kernels(args, d):
  rng = np.random.default_rng(0)
  for n in args.sizes:
    X, y = rng.random((n, d)), rng.standard_normal(n)
    ls = torch.full((d, ), 0.5 * d**0.5, dtype=torch.float64)
    Xc = torch.tensor(X, device='cuda')
    K = hpo.matern52(Xc, Xc, ls.cuda(), 1.0) + 0.01 * torch.eye(n, dtype=torch.float64, device='cuda')
    L = torch.linalg.cholesky(K)
    yc = torch.tensor(y, device='cuda')
    fit = hpo.GpFit(Xc, yc, 0.0, 1.0, ls, 1.0, 0.01, L, torch.cholesky_solve(yc[:, None], L)[:, 0], 0.0)
    C = torch.rand(args.M, d, dtype=torch.float64, device='cuda')
    fstar = float(((K - 0.01 * torch.eye(n, device='cuda', dtype=torch.float64)) @ fit.alpha).max())  # the largest posterior mean over X
    qmax = max(args.qs)
    mu, var, V = hpo.gp_posterior(fit, C, extra_rows=qmax)
    lib, h, st = _lib.lib(), _lib.handle(), _lib.stream()
    # row-major copies, as hpo.gp_posterior passes them (torch.linalg.cholesky may return a column-major factor)
    Ct, Lc, ac, ls_h = C.t().contiguous(), L.contiguous(), fit.alpha.contiguous(), hpo._host_doubles(fit.lengthscales)
    post = lambda: _lib.check(lib.il_gp_posterior(h, Xc.data_ptr(), ac.data_ptr(), Lc.data_ptr(), n, d, Ct.data_ptr(), args.M, ls_h, 1.0, 0.01, mu.data_ptr(),
                                                  var.data_ptr(), V.data_ptr(), st))
    t_post = timed(post)
    post()
    t_post_torch = timed(lambda: torch_posterior(fit, C))
    mu_t, var_t, _ = torch_posterior(fit, C)
    flops = args.M * (n * n + n * (3 * d + 12))
    print(json.dumps(dict(what='il_gp_posterior', card=card(), n=n, d=d, M=args.M, seconds=t_post, torch_seconds=t_post_torch, gflops=flops / t_post / 1e9,
                          share_of_datasheet_fp64=flops / t_post / DATASHEET_FP64, max_diff_mu=float((mu - mu_t).abs().max()), max_diff_var=float((var - var_t).abs().max()))),
          flush=True)
    for q in args.qs:
      ws_bytes = lib.il_gp_select_workspace_bytes(n, d, args.M, q)
      ws, group = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda'), torch.zeros(args.M, dtype=torch.int32, device='cuda')
      picks_d, ei_d = torch.empty(q, dtype=torch.int32, device='cuda'), torch.empty(q, dtype=torch.float64, device='cuda')
      var_s, V_s = var.clone(), V[:n + q].clone()

      def prep():
        var_s.copy_(var)
        V_s.copy_(V[:n + q])
        torch.cuda.synchronize()

      def run():
        _lib.check(lib.il_gp_select(h, n, d, Ct.data_ptr(), args.M, ls_h, 1.0, 0.01, mu.data_ptr(), var_s.data_ptr(), V_s.data_ptr(), group.data_ptr(), 0, fstar, q,
                                    picks_d.data_ptr(), ei_d.data_ptr(), ws.data_ptr(), ws_bytes, st))
      t_sel = timed(run, prep)
      picks = picks_d.cpu().tolist()
      tq = min(q, args.torch_q)
      torch_select(fit, C, mu, var, V[:n], 1, fstar)  # warm-up
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      picks_t, var_after_t = torch_select(fit, C, mu, var, V[:n], tq, fstar)
      torch.cuda.synchronize()
      t_torch = (time.perf_counter() - t0) * q / tq
      nbytes = sum(8 * args.M * (n + j + d + 4) for j in range(q))
      print(json.dumps(dict(what='il_gp_select', card=card(), n=n, d=d, M=args.M, q=q, seconds=t_sel, torch_seconds=t_torch, torch_scaled_from_q=tq, gbytes_per_s=nbytes / t_sel / 1e9,
                            share_of_datasheet_hbm=nbytes / t_sel / DATASHEET_HBM, picks_equal_torch=picks[:tq] == picks_t)), flush=True)


def end_to_end(args):
  """One round of `--trials` SAC trials over the four envs: as grouped programs (hpo.run_trials) and as one program per trial-env."""
  from il_b200.environments import ENVS
  from il_b200.train import train
  from il_b200.config import load_config
  base = ['algorithm=SAC', f'steps={args.steps}', 'evaluation.interval=30', 'evaluation.episodes=1', 'logging.interval=20', 'memory.size=100', 'training.start=20',
          'training.batch_size=32']
  space = hpo.Space.of('SAC', base)
  xs, _ = hpo.sobol_round(space, args.trials, 0)
  trials = [dict(trial=i, overrides=hpo.Space.overrides(space.decode(x)), scores={}) for i, x in enumerate(xs)]
  with tempfile.TemporaryDirectory() as tmp:
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    programs = hpo.run_trials(base, trials, tmp, 0, 1)
    torch.cuda.synchronize()
    grouped = time.perf_counter() - t0
    t0 = time.perf_counter()
    for env in ENVS:
      for j in hpo.trial_jobs(base, trials, env, 0, 1):
        d = os.path.join(tmp, 'single', str(j.num), env)
        os.makedirs(d)
        train(load_config(j.overrides), file_prefix=d + os.sep)
    torch.cuda.synchronize()
    single = time.perf_counter() - t0
  print(json.dumps(dict(what='search round', card=card(), trials=args.trials, envs=len(ENVS), steps=args.steps, programs_per_env=programs, grouped_seconds=grouped,
                        single_programs_seconds=single, speedup=single / grouped)), flush=True)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--sizes', default='30,256,1024,4096')
  ap.add_argument('--M', type=int, default=65536)
  ap.add_argument('--qs', default='1,64,256')
  ap.add_argument('--torch-q', type=int, default=16, help='picks of the torch selection loop that are timed (its time is scaled to q)')
  ap.add_argument('--trials', type=int, default=64)
  ap.add_argument('--steps', type=int, default=60)
  ap.add_argument('--skip-e2e', action='store_true')
  args = ap.parse_args()
  args.sizes, args.qs = [int(x) for x in args.sizes.split(',')], [int(x) for x in args.qs.split(',')]
  if not torch.cuda.is_available(): raise SystemExit('hpo_bench needs a CUDA device')
  kernels(args, hpo.Space.of('GAIL', ['algorithm=GAIL']).d)
  if not args.skip_e2e: end_to_end(args)


if __name__ == '__main__':
  main()
