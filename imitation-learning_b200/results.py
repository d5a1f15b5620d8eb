"""Seed-sweep results as the reference reports them (scripts/print_plot_seed_sweep_results.py, its printing half): the IQM of the
normalised test return over runs x envs at every evaluation point, with a 95 % stratified-bootstrap percentile interval.

The reference computes these with scipy's trim_mean and rliable's `aggregate_iqm` / `get_interval_estimates`; here every statistic runs
as fp64 CUDA (il_iqm, il_bootstrap_iqm, il_percentile_interval), and only the [2, T] interval and the [T] point estimate return to the
host. Score matrices follow rliable's layout: [runs, envs, T].
"""
from __future__ import annotations

import glob
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from . import _lib


def _device(x) -> torch.Tensor:
  return torch.as_tensor(np.ascontiguousarray(x, dtype=np.float64)).to('cuda', non_blocking=False)


def _finite(x, what: str) -> np.ndarray:
  """x as float64, refused when any value is NaN or infinite: a diverged run is not a score the IQM can summarise."""
  x = np.asarray(x, dtype=np.float64)
  if not np.isfinite(x).all(): raise ValueError(f'{what}: {int((~np.isfinite(x)).sum())} non-finite score(s); the statistics need finite values')
  return x


def trim_mean(x) -> np.ndarray:
  """scipy.stats.trim_mean(x, 0.25, axis=-1): the mean of the order statistics [floor(n / 4), n - floor(n / 4)) of the last axis."""
  x = _finite(x, 'trim_mean')
  n = x.shape[-1]
  if n < 1 or x.size == 0: raise ValueError(f'trim_mean needs at least one value per group (shape {x.shape})')
  if n > _lib.IQM_MAX_N: raise ValueError(f'trim_mean: {n} values per group exceed the supported {_lib.IQM_MAX_N}')
  G = x.size // n
  dx = _device(x.reshape(G, n))
  out = torch.empty(G, dtype=torch.float64, device='cuda')
  _lib.check(_lib.lib().il_iqm(_lib.handle(), dx.data_ptr(), G, n, out.data_ptr(), _lib.stream()))
  return out.cpu().numpy().reshape(x.shape[:-1])


def aggregate_iqm(scores) -> np.ndarray:
  """rliable's metrics.aggregate_iqm: the IQM over runs x envs. scores [runs, envs] gives a scalar, [runs, envs, T] one value per t."""
  s = _finite(scores, 'aggregate_iqm')
  if s.ndim not in (2, 3): raise ValueError(f'aggregate_iqm expects [runs, envs] or [runs, envs, T] scores, got shape {s.shape}')
  if s.ndim == 2: return trim_mean(s.reshape(-1))[()]
  return trim_mean(s.reshape(-1, s.shape[2]).T)


def bootstrap_iqm(scores, reps: int, seed: int = 0, indices: Optional[torch.Tensor] = None) -> torch.Tensor:
  """The stratified-bootstrap distribution of the IQM, [reps, T] on the device, for scores [runs, envs, T]: each rep resamples runs with
  replacement within each env, independently per evaluation point. `indices` ([reps, T, envs, runs] int32 CUDA, values in [0, runs))
  replaces the device draws, which are a function of (seed, rep, t, env) alone.

  rliable's StratifiedBootstrap draws, as we recall it, one index array shaped like the score array's [runs, envs] per rep, which would
  share a resample across all t; rliable is not a dependency of this project, so that recollection is unchecked. The interval at each t is a marginal of the rep
  distribution at that t, which has the same law under either scheme; only the correlation between points of the curve differs."""
  s = _finite(scores, 'bootstrap_iqm')
  if s.ndim != 3: raise ValueError(f'bootstrap_iqm expects [runs, envs, T] scores, got shape {s.shape}')
  runs, envs, T = s.shape
  ws_bytes = _lib.lib().il_bootstrap_iqm_workspace_bytes(T, envs, runs)
  if ws_bytes < 0: raise ValueError(f'bootstrap_iqm: runs x envs = {runs * envs} must be in [1, {_lib.BOOTSTRAP_MAX_N}] with T >= 1 (shape {s.shape})')
  if indices is not None:
    if indices.dtype != torch.int32 or not indices.is_cuda or tuple(indices.shape) != (reps, T, envs, runs): raise ValueError('indices must be [reps, T, envs, runs] int32 on CUDA')
    indices = indices.contiguous()
  dx = _device(s.transpose(2, 1, 0))  # [T, envs, runs]
  out = torch.empty(reps, T, dtype=torch.float64, device='cuda')
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
  _lib.check(_lib.lib().il_bootstrap_iqm(_lib.handle(), dx.data_ptr(), T, envs, runs, int(reps), int(seed) & (2**64 - 1), _lib.ptr(indices), out.data_ptr(), ws.data_ptr(), ws_bytes,
                                          _lib.stream()))
  return out


def interval_percentiles(confidence: float) -> Tuple[float, float]:
  """The two percentiles of a two-sided percentile interval at `confidence` (2.5 and 97.5 at 0.95)."""
  if not 0.0 < confidence < 1.0: raise ValueError(f'confidence must be in (0, 1), got {confidence}')
  alpha = (1.0 - confidence) / 2.0
  return 100.0 * alpha, 100.0 * (1.0 - alpha)


def percentile_interval(dist: torch.Tensor, confidence: float = 0.95) -> np.ndarray:
  """[2, T]: numpy.percentile(dist, interval_percentiles(confidence), axis=0) (linear interpolation) of a device distribution [reps, T].
  rliable takes arch's 'percentile' interval; that arch uses exactly numpy's linear rule is our reading of it, unchecked (arch is not a dependency)."""
  if dist.dim() != 2 or dist.dtype != torch.float64 or not dist.is_cuda: raise ValueError('dist must be a [reps, T] float64 CUDA tensor')
  q_lo, q_hi = interval_percentiles(confidence)
  dist = dist.contiguous()
  out = torch.empty(2, dist.shape[1], dtype=torch.float64, device='cuda')
  _lib.check(_lib.lib().il_percentile_interval(_lib.handle(), dist.data_ptr(), dist.shape[0], dist.shape[1], q_lo, q_hi, out.data_ptr(), _lib.stream()))
  return out.cpu().numpy()


def get_interval_estimates(score_dict: Dict[str, np.ndarray], reps: int = 50000, confidence: float = 0.95, seed: int = 0) -> Tuple[Dict[str, np.ndarray], Dict[str, np.ndarray]]:
  """rliable's library.get_interval_estimates(score_dict, iqm, reps) with the stratified bootstrap: per key, the point estimate [T] and the
  percentile interval [2, T] of scores [runs, envs, T]. Every key is bootstrapped with the same `seed`, so a key's result does not depend
  on the others in the dict."""
  if reps < 1: raise ValueError(f'reps must be positive, got {reps}')
  points, intervals = {}, {}
  for k, scores in score_dict.items():
    points[k] = aggregate_iqm(scores)
    intervals[k] = percentile_interval(bootstrap_iqm(scores, reps, seed), confidence)
  return points, intervals


# ---- sweep outputs ---------------------------------------------------------------------------------------------------------------
def resolve_sweep_dir(pattern: str, algorithm: str, env: str, trajectories: str) -> str:
  """The one directory that `pattern` (with {algorithm}, {env}, {trajectories} fields and optionally glob wildcards) names."""
  path = pattern.format(algorithm=algorithm, env=env, trajectories=trajectories)
  found = sorted(p for p in glob.glob(path) if os.path.isdir(p))
  if len(found) != 1: raise ValueError(f'{path!r} must match exactly one directory, matched {len(found)}' + (f': {found}' if found else ''))
  return found[0]


def _job_dirs(sweep_dir: str) -> List[str]:
  """The job directories <n>/ holding metrics.pth, in job order. Jobs pool into one cell only when they differ in `seed` alone: a multirun
  that also swept another key writes all its jobs under one directory, and their overrides.yaml files (train.py -m) tell them apart."""
  import yaml
  jobs = sorted((int(d), os.path.join(sweep_dir, d)) for d in os.listdir(sweep_dir) if d.isdigit() and os.path.isfile(os.path.join(sweep_dir, d, 'metrics.pth')))
  if not jobs: raise ValueError(f'{sweep_dir}: no job directories <n>/metrics.pth')
  first = None
  for _, d in jobs:
    f = os.path.join(d, 'overrides.yaml')
    if not os.path.isfile(f): continue
    with open(f) as fh: rest = sorted(o for o in (yaml.safe_load(fh) or []) if not str(o).lstrip('+~').startswith('seed='))
    if first is None: first = (d, rest)
    elif rest != first[1]: raise ValueError(f'{d}: overrides {rest} differ from {first[1]} of {first[0]} in more than the seed; a cell pools seeds of one configuration only')
  return [p for _, p in jobs]


def load_sweep_returns(sweep_dir: str, unnormalise: bool = False) -> Tuple[List[int], np.ndarray]:
  """(test_steps, returns [runs, T, episodes]) of one sweep directory (<dir>/<job>/metrics.pth). A job of a replicas=1 run stores one list
  of episodes per evaluation, a job of R > 1 replicas [R][episodes]; each replica is one run, ordered job-major, then replica-minor."""
  key = 'test_returns' if unnormalise else 'test_returns_normalized'
  steps, runs = None, []
  for d in _job_dirs(sweep_dir):
    m = torch.load(os.path.join(d, 'metrics.pth'), weights_only=False)
    if not m['test_steps']: raise ValueError(f'{d}: no evaluation points')
    if steps is None: steps = list(m['test_steps'])
    elif list(m['test_steps']) != steps: raise ValueError(f'{d}: test_steps {list(m["test_steps"])} differ from {steps}')
    r = np.asarray(m[key], dtype=np.float64)
    if r.ndim == 2: r = r[:, None, :]  # [T, episodes]: a single replica
    if r.ndim != 3 or r.shape[0] != len(steps): raise ValueError(f'{d}: {key} has shape {r.shape}, expected [T, episodes] or [T, R, episodes] with T = {len(steps)}')
    runs.extend(r.transpose(1, 0, 2))
  returns = np.stack(runs)
  if not np.isfinite(returns).all(): raise ValueError(f'{sweep_dir}: non-finite {key}')
  return steps, returns


def load_returns(sweep_dirs: Sequence[str], seeds: Optional[int] = None, unnormalise: bool = False) -> Tuple[List[int], List[np.ndarray]]:
  """(test_steps, one [runs, T, episodes] array per env) from one sweep directory per env: the first `seeds` runs of every env, or all
  runs, equal in number across envs, when `seeds` is None. Refuses unequal test_steps across envs and fewer runs than requested."""
  steps, per_env = None, []
  for d in sweep_dirs:
    s, r = load_sweep_returns(d, unnormalise)
    if steps is None: steps = s
    elif s != steps: raise ValueError(f'{d}: test_steps {s} differ from {steps} of {sweep_dirs[0]}')
    if seeds is not None:
      if r.shape[0] < seeds: raise ValueError(f'{d}: {r.shape[0]} runs, fewer than the {seeds} requested')
      r = r[:seeds]
    elif per_env and r.shape[0] != per_env[0].shape[0]: raise ValueError(f'{d}: {r.shape[0]} runs, but {sweep_dirs[0]} has {per_env[0].shape[0]}')
    per_env.append(r)
  return steps, per_env


def load_score_matrix(sweep_dirs: Sequence[str], seeds: Optional[int] = None, unnormalise: bool = False) -> Tuple[List[int], np.ndarray]:
  """(test_steps, scores [runs, envs, T]): load_returns, then each run's IQM over its evaluation episodes (print_plot_seed_sweep_results.py:43-44)."""
  steps, per_env = load_returns(sweep_dirs, seeds, unnormalise)
  return steps, np.stack([trim_mean(r) for r in per_env], axis=1)
