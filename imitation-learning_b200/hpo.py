"""Hyper-parameter search over all four environments (the reference's `train_all.py -m`, its Ax sweeper replaced by a batched
Bayesian optimiser that this project states and tests itself).

A trial is one configuration trained on every env in ENVS with one seed; its objective is the minimum over envs of train()'s score
(the mean normalised test return). Rounds are synchronous:

* Round 0: `hpo.initial` scrambled Sobol points (torch.quasirandom.SobolEngine, seed `hpo.seed`), snapped to feasible values;
  with `hpo.max_groups` G > 0, points outside the first G groups met are passed over.
* Every later round proposes `hpo.batch` trials:
  1. fit_gp: a zero-mean GP on the standardised finite objectives, Matérn-5/2 ARD kernel with output scale and Gaussian noise, its
     log-parameters fitted by L-BFGS on the log marginal likelihood within GP_BOUNDS from GP_STARTS (best kept; never below a start);
  2. candidates: `hpo.candidates` feasible points (the rule is on the function);
  3. il_gp_posterior (csrc/gp.cu): mean, latent variance and V = L^-1 K*^T of every candidate;
  4. il_gp_select (csrc/gp.cu): greedy expected-improvement picks with the kriging believer, at most `hpo.max_groups` programs per env.
* The search stops after `hpo.max_trials` trials, or after `hpo.patience` rounds without a better best objective.

Trials of a round run env by env; each env's trials go through config.sweep_groups, so trials that agree on every grouping key are one
program (train._train, one replica block per trial).
"""
from __future__ import annotations

import copy
import itertools
import json
import math
import os
import time
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
import yaml

from . import _lib, checkpoint
from .config import (BOTH, CONF_DIR, IGNORED, MULTIRUN_FLAGS, PER_REPLICA_KEYS, SWEEP, Config, SweepError, SweepJob, _parse, _reject_sweep, load_config,
                     replica_values, seed_per_replica, set_key, sweep_groups)

SPACE_DIR = os.path.join(CONF_DIR, 'hyperparameter_search_space')
# GP hyper-parameter bounds, on the standardised objective and inputs in [0, 1]^d: lengthscales, output scale, noise variance
GP_BOUNDS = {'lengthscale': (1e-2, 1e2), 'outputscale': (1e-2, 1e2), 'noise': (1e-6, 1.0)}
# L-BFGS starts: (lengthscale of every dimension, output scale, noise variance)
GP_STARTS = ((0.3, 1.0, 1e-2), (1.0, 1.0, 1e-3), (3.0, 1.0, 1e-1))
JITTER = (0.0, 1e-10, 1e-8, 1e-6, 1e-4)  # added to the noise (times the output scale) when a Cholesky factorisation fails, in this order
TOP_K, STEP, RESAMPLE = 5, 0.1, 0.2  # candidates: parents among the top-k trials, Gaussian step on range dims, categorical resample probability


# ---- search spaces -------------------------------------------------------------------------------------------------------------
def load_space_spec(algorithm: str, space_dir: str = SPACE_DIR) -> Dict[str, Dict[str, Any]]:
  """{key: {type, bounds | values, value_type}} of conf/hyperparameter_search_space/<algorithm>.yaml, with its `defaults` composed the way
  Hydra composes a defaults list without _self_: the listed spaces' params first, then the file's own."""
  path = os.path.join(space_dir, f'{algorithm}.yaml')
  if not os.path.exists(path): raise FileNotFoundError(f'no search space for algorithm={algorithm!r} under {space_dir}')
  with open(path) as f: d = yaml.safe_load(f) or {}
  params = {}
  for base in d.get('defaults', []): params.update(load_space_spec(base, space_dir))
  params.update(d.get('params', {}))
  return params


@dataclass
class Param:
  key: str
  type: str                 # range | choice
  value_type: str           # int | float | str | bool
  bounds: Tuple[float, float] = (0.0, 1.0)
  values: Tuple[Any, ...] = ()
  col: int = 0              # first column of x
  structural: bool = False  # only whether the value is > 0 separates programs

  @property
  def kind(self) -> str:
    """range: x = (v - lo) / (hi - lo); ordered (numeric choice): x = index / (k - 1); onehot (str / bool choice): one column per value."""
    if self.type == 'range': return 'range'
    return 'onehot' if self.value_type in ('str', 'bool') else 'ordered'

  @property
  def width(self) -> int:
    return len(self.values) if self.kind == 'onehot' else 1

  @property
  def levels(self) -> int:
    """Distinct program-relevant values: choice levels, integer range values, or 2 (zero / positive) for a structural rate."""
    if self.structural: return 2
    if self.type == 'choice': return len(self.values)
    if self.value_type == 'int': return int(self.bounds[1]) - int(self.bounds[0]) + 1
    raise SweepError(f'{self.key}: a float range that separates programs cannot be given a group id')


def _typed(v, value_type):
  return {'int': int, 'float': float, 'str': str, 'bool': bool}[value_type](v)


class Space:
  """The encoded search space of one configuration: x in [0, 1]^d, one block of columns per searched key."""

  def __init__(self, params: List[Param], group_keys: Sequence[str] = ()):
    col = 0
    for p in params:
      p.col = col
      col += p.width
    self.params, self.d = params, col
    self.group_params = [p for p in params if p.key in group_keys]

  @classmethod
  def of(cls, algorithm: str, overrides: Sequence[str], space_dir: str = SPACE_DIR) -> 'Space':
    """The space of `algorithm` under the fixed `overrides`: keys the command line fixes leave the search, keys the configuration ignores
    (config.PER_REPLICA_KEYS role IGNORED) are dropped, and the keys that may separate programs are found by group_keys."""
    spec = load_space_spec(algorithm, space_dir)
    fixed = {o.partition('=')[0].lstrip('+') for o in overrides}
    base = load_config(list(overrides))
    params = []
    for k, s in spec.items():
      if k in fixed: continue
      e = PER_REPLICA_KEYS.get(k)
      if e is not None and e.role(base) == IGNORED: continue
      p = Param(k, s['type'], s['value_type'], structural=bool(e and e.structural))
      if s['type'] == 'range': p.bounds = tuple(_typed(b, 'float') for b in s['bounds'])
      else: p.values = tuple(_typed(v, s['value_type']) for v in s['values'])
      params.append(p)
    space = cls(params)
    space.group_params = [p for p in params if p.key in group_keys(space, base)]
    return space

  # -- encoding
  def level_index(self, p: Param, x: torch.Tensor) -> torch.Tensor:
    """The level of p in each row of x [.., d] (int64): choice index, integer offset from the lower bound, or (value > 0) for a structural rate."""
    c = x[..., p.col:p.col + p.width]
    if p.kind == 'onehot': return c.argmax(-1)
    c = c[..., 0].clamp(0.0, 1.0)
    if p.kind == 'ordered': return torch.round(c * (len(p.values) - 1)).long()
    lo, hi = p.bounds
    v = lo + c * (hi - lo)
    if p.structural: return (v > 0).long()
    return (torch.round(v) - round(lo)).long()

  def snap(self, x: torch.Tensor) -> torch.Tensor:
    """The nearest feasible encoding: ranges clipped to [0, 1] (integer ranges rounded to an integer value), ordered choices rounded to a
    level, one-hot blocks set to the one-hot of their largest column (the first on a tie)."""
    x = x.clone()
    for p in self.params:
      c = x[..., p.col:p.col + p.width]
      if p.kind == 'onehot':
        x[..., p.col:p.col + p.width] = torch.nn.functional.one_hot(c.argmax(-1), p.width).to(x.dtype)
      elif p.kind == 'ordered':
        k = len(p.values)
        x[..., p.col] = self.level_index(p, x).to(x.dtype) / (k - 1) if k > 1 else 0.0
      else:
        c = c[..., 0].clamp(0.0, 1.0)
        if p.value_type == 'int':
          lo, hi = p.bounds
          c = (torch.round(lo + c * (hi - lo)) - lo) / (hi - lo)
        x[..., p.col] = c
    return x

  def decode(self, x) -> Dict[str, Any]:
    """{key: value} of one encoded row, each value in its value_type."""
    x = torch.as_tensor(x, dtype=torch.float64).cpu()
    out = {}
    for p in self.params:
      if p.type == 'choice': out[p.key] = p.values[int(self.level_index(p, x))]
      elif p.value_type == 'int': out[p.key] = int(round(p.bounds[0] + float(x[p.col].clamp(0, 1)) * (p.bounds[1] - p.bounds[0])))
      else: out[p.key] = float(p.bounds[0] + float(x[p.col].clamp(0, 1)) * (p.bounds[1] - p.bounds[0]))
    return out

  def encode(self, values: Dict[str, Any]) -> torch.Tensor:
    x = torch.zeros(self.d, dtype=torch.float64)
    for p in self.params:
      v = values[p.key]
      if p.kind == 'onehot': x[p.col + p.values.index(v)] = 1.0
      elif p.kind == 'ordered': x[p.col] = p.values.index(v) / (len(p.values) - 1) if len(p.values) > 1 else 0.0
      else: x[p.col] = (float(v) - p.bounds[0]) / (p.bounds[1] - p.bounds[0])
    return x

  @staticmethod
  def overrides(values: Dict[str, Any]) -> List[str]:
    """key=value strings that load_config reads back exactly: floats by repr, bools as true / false."""
    fmt = lambda v: ('true' if v else 'false') if isinstance(v, bool) else repr(v) if isinstance(v, float) else str(v)
    return [f'{k}={fmt(v)}' for k, v in values.items()]

  def group_ids(self, x: torch.Tensor) -> torch.Tensor:
    """int32 group id of each row of x [.., d]: the mixed-radix index of its levels of group_params. Equal ids never run as different programs."""
    gid = torch.zeros(x.shape[:-1], dtype=torch.int64, device=x.device)
    for p in self.group_params: gid = gid * p.levels + self.level_index(p, x)
    return gid.to(torch.int32)


def group_keys(space: Space, base: Config) -> List[str]:
  """The searched keys that separate programs in some configuration the space can reach: a key whose PER_REPLICA_KEYS role is neither
  per replica nor ignored, or whose > 0 is structural, in any configuration of the product of the choice values, with structural rates at
  either bound and other ranges at their lower bound (a key's role depends on choices and on whether a rate is zero, nothing else)."""
  params = space.params
  values = [p.values if p.type == 'choice' else tuple(_typed(b, p.value_type) for b in (p.bounds if p.structural else p.bounds[:1])) for p in params]
  keys, cfg = set(), Config(copy.deepcopy(base))
  for combo in itertools.product(*values):
    for p, v in zip(params, combo): set_key(cfg, p.key, v)
    for p in params:
      e = PER_REPLICA_KEYS.get(p.key)
      role = e.role(cfg) if e else None
      if role not in (BOTH, SWEEP, IGNORED) or (e.structural and role != IGNORED): keys.add(p.key)
    if len(keys) == len(params): break
  n = 1
  for p in params:
    if p.key in keys: n *= p.levels
  if n > 2**31 - 1: raise SweepError(f'{n} possible programs per env exceed the int32 group id')
  return [p.key for p in params if p.key in keys]


def sobol_round(space: Space, n: int, seed: int, skip: int = 0, max_groups: int = 0) -> Tuple[torch.Tensor, int]:
  """(n points [n, d] float64, points consumed): the scrambled Sobol sequence (seeded) after its first `skip` points, snapped. With
  max_groups G > 0, a point whose group id is not among the first G groups met is passed over (up to 100 n points in all)."""
  eng = torch.quasirandom.SobolEngine(space.d, scramble=True, seed=seed)
  if skip: eng.fast_forward(skip)
  if max_groups <= 0: return space.snap(eng.draw(n, dtype=torch.float64)), n
  kept, groups, used = [], [], 0
  while len(kept) < n and used < 100 * n:
    x = space.snap(eng.draw(1, dtype=torch.float64))
    used += 1
    g = int(space.group_ids(x)[0])
    if g not in groups and len(groups) >= max_groups: continue
    if g not in groups: groups.append(g)
    kept.append(x)
  return torch.cat(kept), used


# ---- GP fit (host plumbing, torch float64) ------------------------------------------------------------------------------------
def matern52(A: torch.Tensor, B: torch.Tensor, ls: torch.Tensor, s2) -> torch.Tensor:
  r2 = (((A[:, None, :] - B[None, :, :]) / ls)**2).sum(-1)
  r = torch.sqrt(r2.clamp_min(1e-300))
  return s2 * (1.0 + math.sqrt(5.0) * r + (5.0 / 3.0) * r2) * torch.exp(-math.sqrt(5.0) * r)


def cholesky_jitter(K: torch.Tensor, s2) -> Tuple[torch.Tensor, float]:
  """(L, jitter): the Cholesky factor of K + jitter I with the first JITTER step (times s2) that factorises."""
  eye, s2 = torch.eye(K.shape[0], dtype=K.dtype, device=K.device), float(torch.as_tensor(s2).detach())
  for j in JITTER:
    L, info = torch.linalg.cholesky_ex(K + (j * s2) * eye)
    if int(info) == 0: return L, j * s2
  raise np.linalg.LinAlgError(f'Cholesky failed with jitter up to {JITTER[-1]} x the output scale')


def _unpack(u: torch.Tensor, d: int):
  out = []
  for i, (name, n) in enumerate((('lengthscale', d), ('outputscale', 1), ('noise', 1))):
    lo, hi = (math.log(b) for b in GP_BOUNDS[name])
    seg = u[sum((d, 1, 1)[:i]):sum((d, 1, 1)[:i + 1])]
    out.append(torch.exp(lo + (hi - lo) * torch.sigmoid(seg)))
  return out[0], out[1][0], out[2][0]


def _pack(ls: float, s2: float, noise: float, d: int, device) -> torch.Tensor:
  def logit(v, name):
    lo, hi = (math.log(b) for b in GP_BOUNDS[name])
    t = (math.log(v) - lo) / (hi - lo)
    return math.log(t / (1 - t))
  return torch.tensor([logit(ls, 'lengthscale')] * d + [logit(s2, 'outputscale'), logit(noise, 'noise')], dtype=torch.float64, device=device)


def log_marginal_likelihood(X, y, ls, s2, noise) -> torch.Tensor:
  K = matern52(X, X, ls, s2) + noise * torch.eye(X.shape[0], dtype=X.dtype, device=X.device)
  L, _ = cholesky_jitter(K, s2)
  a = torch.cholesky_solve(y[:, None], L)[:, 0]
  return -0.5 * (y @ a) - torch.log(torch.diagonal(L)).sum() - 0.5 * X.shape[0] * math.log(2 * math.pi)


@dataclass
class GpFit:
  X: torch.Tensor            # [n, d]
  y: torch.Tensor            # [n] standardised
  y_mean: float
  y_std: float
  lengthscales: torch.Tensor
  outputscale: float
  noise: float               # fitted noise plus the Cholesky jitter: the noise the factor L holds
  L: torch.Tensor            # Cholesky factor of K + noise I
  alpha: torch.Tensor        # (K + noise I)^-1 y
  lml: float
  start_lml: List[float] = field(default_factory=list)

  def summary(self) -> Dict[str, Any]:
    return dict(lengthscales=self.lengthscales.tolist(), outputscale=self.outputscale, noise=self.noise, lml=self.lml, y_mean=self.y_mean, y_std=self.y_std)


def fit_gp(X: torch.Tensor, y: torch.Tensor, max_iter: int = 100) -> GpFit:
  """Fits the GP to finite objectives y [n] at X [n, d] (float64, any device): y is standardised (mean 0, population std 1; std 1 when
  it is 0), then the log marginal likelihood is maximised by L-BFGS (strong Wolfe) over u, with each log-parameter
  log p = log lo + (log hi - log lo) sigmoid(u) inside GP_BOUNDS, from each of GP_STARTS. The best of every start and every end point is kept."""
  X, y = X.to(torch.float64), y.to(torch.float64)
  if not torch.isfinite(y).all() or not torch.isfinite(X).all(): raise ValueError('fit_gp: non-finite inputs')
  n, d = X.shape
  y_mean = float(y.mean())
  y_std = float(y.std(unbiased=False)) if n > 1 else 1.0
  if not y_std > 0: y_std = 1.0
  ys = (y - y_mean) / y_std
  best, starts = None, []
  for ls0, s20, noise0 in GP_STARTS:
    u0 = _pack(ls0, s20, noise0, d, X.device)
    with torch.no_grad(): l0 = float(log_marginal_likelihood(X, ys, *_unpack(u0, d)))
    starts.append(l0)
    cands = [(l0, u0)]
    u = u0.clone().requires_grad_(True)
    opt = torch.optim.LBFGS([u], lr=1.0, max_iter=max_iter, line_search_fn='strong_wolfe')

    def closure():
      opt.zero_grad()
      loss = -log_marginal_likelihood(X, ys, *_unpack(u, d)) / n
      loss.backward()
      return loss
    try:
      opt.step(closure)
      with torch.no_grad(): l1 = float(log_marginal_likelihood(X, ys, *_unpack(u.detach(), d)))
      if math.isfinite(l1): cands.append((l1, u.detach().clone()))
    except np.linalg.LinAlgError:
      pass
    for c in cands:
      if best is None or c[0] > best[0]: best = c
  ls, s2, noise = (t.detach() for t in _unpack(best[1], d))
  s2, noise = float(s2), float(noise)
  K = matern52(X, X, ls, s2) + noise * torch.eye(n, dtype=X.dtype, device=X.device)
  L, jitter = cholesky_jitter(K, s2)
  alpha = torch.cholesky_solve(ys[:, None], L)[:, 0]
  return GpFit(X, ys, y_mean, y_std, ls, s2, noise + jitter, L, alpha, best[0], starts)


# ---- candidates (host plumbing, torch on the device) -----------------------------------------------------------------------------
def candidates(space: Space, X: torch.Tensor, y: torch.Tensor, M: int, seed: int) -> torch.Tensor:
  """M feasible candidates [M, d] on X's device, from torch.Generator(device).manual_seed(seed), drawn in this order:
    1. U = rand(M - M // 2, d): the uniform half, snap(U);
    2. parent = randint(0, k, (M // 2,)) with k = min(TOP_K, n): indices into the top-k trials by y (descending, the lower trial index on ties);
    3. step = randn(M // 2, d): range columns of the parent move by STEP * step, then are clipped;
    4. flip = rand(M // 2, P) < RESAMPLE and level = floor(rand(M // 2, P) * levels), P = the number of params: a choice param with flip set
       takes that level (its ordered value, or its one-hot);
  then the perturbed half is snapped. Rows: the uniform half, then the perturbed half."""
  dev = X.device
  g = torch.Generator(device=dev).manual_seed(int(seed))
  mu_, mp = M - M // 2, M // 2
  U = torch.rand(mu_, space.d, generator=g, dtype=torch.float64, device=dev)
  k = min(TOP_K, X.shape[0])
  order = sorted(range(X.shape[0]), key=lambda i: (-float(y[i]), i))[:k]
  top = X[torch.tensor(order, device=dev)]
  parent = torch.randint(0, k, (mp, ), generator=g, device=dev)
  step = torch.randn(mp, space.d, generator=g, dtype=torch.float64, device=dev)
  P = len(space.params)
  flip = torch.rand(mp, P, generator=g, dtype=torch.float64, device=dev) < RESAMPLE
  lev_u = torch.rand(mp, P, generator=g, dtype=torch.float64, device=dev)
  Z = top[parent].clone()
  for i, p in enumerate(space.params):
    if p.type == 'range':
      Z[:, p.col] = (Z[:, p.col] + STEP * step[:, p.col]).clamp(0.0, 1.0)
      continue
    kk = len(p.values)
    lev = torch.clamp(torch.floor(lev_u[:, i] * kk).long(), max=kk - 1)
    f = flip[:, i]
    if p.kind == 'onehot':
      Z[:, p.col:p.col + kk] = torch.where(f[:, None], torch.nn.functional.one_hot(lev, kk).to(Z.dtype), Z[:, p.col:p.col + kk])
    else:
      Z[:, p.col] = torch.where(f, lev.to(Z.dtype) / max(kk - 1, 1), Z[:, p.col])
  return torch.cat([space.snap(U), space.snap(Z)])


# ---- CUDA posterior and selection -----------------------------------------------------------------------------------------------
def _finite_cuda(t: torch.Tensor, what: str) -> torch.Tensor:
  if not t.is_cuda or t.dtype != torch.float64: raise ValueError(f'{what} must be a float64 CUDA tensor')
  if not torch.isfinite(t).all(): raise ValueError(f'{what}: non-finite values')
  return t.contiguous()


def gp_posterior(fit: GpFit, C: torch.Tensor, extra_rows: int = 0) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
  """(mu [M], var [M], V [n + extra_rows, M]) of candidates C [M, d] under `fit` (il_gp_posterior); rows n.. of V are left for il_gp_select."""
  X, alpha, L = (_finite_cuda(t, w) for t, w in ((fit.X, 'X'), (fit.alpha, 'alpha'), (fit.L, 'L')))
  Ct = _finite_cuda(C, 'candidates').t().contiguous()
  n, d = X.shape
  M = C.shape[0]
  mu, var = (torch.empty(M, dtype=torch.float64, device='cuda') for _ in range(2))
  V = torch.empty(n + extra_rows, M, dtype=torch.float64, device='cuda')
  ls = _host_doubles(fit.lengthscales)
  _lib.check(_lib.lib().il_gp_posterior(_lib.handle(), X.data_ptr(), alpha.data_ptr(), L.data_ptr(), n, d, Ct.data_ptr(), M, ls, fit.outputscale, fit.noise, mu.data_ptr(),
                                        var.data_ptr(), V.data_ptr(), _lib.stream()))
  return mu, var, V


def _host_doubles(t: torch.Tensor):
  import ctypes
  vals = [float(v) for v in t.reshape(-1).tolist()]
  return (ctypes.c_double * len(vals))(*vals)


def gp_select(fit: GpFit, C: torch.Tensor, mu: torch.Tensor, var: torch.Tensor, V: torch.Tensor, group: torch.Tensor, q: int, max_groups: int,
              f_star: float) -> Tuple[List[int], List[float]]:
  """(picks, ei) of il_gp_select: q greedy EI picks (indices into C; -1 once none is admissible). var and rows [n, n + q) of V are updated in place."""
  n, d = fit.X.shape
  M = C.shape[0]
  if V.shape != (n + q, M) or not V.is_contiguous(): raise ValueError(f'V must be a contiguous [{n + q}, {M}] tensor')
  if group.dtype != torch.int32 or not group.is_cuda or group.shape != (M, ): raise ValueError('group must be [M] int32 on CUDA')
  Ct = _finite_cuda(C, 'candidates').t().contiguous()
  ws_bytes = _lib.lib().il_gp_select_workspace_bytes(n, d, M, q)
  if ws_bytes < 0: raise ValueError(f'il_gp_select refuses n={n}, d={d}, M={M}, q={q}')
  ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
  picks = torch.empty(q, dtype=torch.int32, device='cuda')
  ei = torch.empty(q, dtype=torch.float64, device='cuda')
  _lib.check(_lib.lib().il_gp_select(_lib.handle(), n, d, Ct.data_ptr(), M, _host_doubles(fit.lengthscales), fit.outputscale, fit.noise, mu.data_ptr(), var.data_ptr(),
                                     V.data_ptr(), group.contiguous().data_ptr(), int(max_groups), float(f_star), q, picks.data_ptr(), ei.data_ptr(), ws.data_ptr(), ws_bytes,
                                     _lib.stream()))
  return picks.cpu().tolist(), ei.cpu().tolist()


def propose(space: Space, X: torch.Tensor, y: torch.Tensor, q: int, M: int, max_groups: int, seed: int) -> Tuple[torch.Tensor, Dict[str, Any]]:
  """One GP round: q encoded trials [<= q, d] (fewer when the admissible candidates run out) and the round's record (fit, f*, EI, groups)."""
  X, y = X.to('cuda', torch.float64), y.to('cuda', torch.float64)
  fit = fit_gp(X, y)
  C = candidates(space, X, y, M, seed)
  group = space.group_ids(C)
  mu, var, V = gp_posterior(fit, C, extra_rows=q)
  f_star = float((matern52(fit.X, fit.X, fit.lengthscales, fit.outputscale) @ fit.alpha).max())
  picks, ei = gp_select(fit, C, mu, var, V, group, q, max_groups, f_star)
  keep = [i for i, p in enumerate(picks) if p >= 0]
  idx = torch.tensor([picks[i] for i in keep], dtype=torch.long, device='cuda')
  info = dict(gp=fit.summary(), f_star=f_star, picks=[dict(candidate=picks[i], ei=ei[i], group=int(group[picks[i]])) for i in keep])
  return C[idx].cpu(), info


# ---- rounds ------------------------------------------------------------------------------------------------------------------------
HPO_KEYS = ('max_trials', 'patience', 'minimize', 'batch', 'initial', 'candidates', 'max_groups', 'seed')


def load_hpo(overrides: Sequence[str], conf_dir: str = CONF_DIR) -> Dict[str, Any]:
  """conf/train_all_config.yaml's hpo block with `hpo.<key>=value` overrides applied."""
  with open(os.path.join(conf_dir, 'train_all_config.yaml')) as f: hpo = dict((yaml.safe_load(f) or {})['hpo'])
  for o in overrides:
    k, _, v = o.partition('=')
    key = k.lstrip('+')[len('hpo.'):]
    if key not in HPO_KEYS: raise SweepError(f'{o}: unknown search setting (hpo keys: {", ".join(HPO_KEYS)})')
    hpo[key] = _parse(v)
  for k in HPO_KEYS:
    if k == 'minimize': continue
    if not isinstance(hpo[k], int) or isinstance(hpo[k], bool) or hpo[k] < (0 if k in ('max_groups', 'patience', 'seed') else 1):
      raise SweepError(f'hpo.{k}={hpo[k]!r} must be an integer >= {0 if k in ("max_groups", "patience", "seed") else 1}')
  if not isinstance(hpo['minimize'], bool): raise SweepError(f'hpo.minimize={hpo["minimize"]!r} must be true or false')
  if hpo['max_trials'] > _lib.GP_MAX_N: raise SweepError(f'hpo.max_trials={hpo["max_trials"]} exceeds the {_lib.GP_MAX_N} observed trials one GP fit takes')
  if hpo['batch'] > _lib.GP_MAX_Q or hpo['candidates'] > _lib.GP_MAX_M or hpo['batch'] > hpo['candidates']:
    raise SweepError(f'need hpo.batch <= min(hpo.candidates, {_lib.GP_MAX_Q}) and hpo.candidates <= {_lib.GP_MAX_M}')
  return hpo


def round_size(n_done: int, hpo: Dict[str, Any]) -> int:
  """Trials of the next round: `initial` first, then `batch`, never past max_trials."""
  return max(0, min(hpo['initial'] if n_done == 0 else hpo['batch'], hpo['max_trials'] - n_done))


def stop_reason(best_after_round: Sequence[float], n_done: int, hpo: Dict[str, Any]) -> Optional[str]:
  """'max_trials' once that many trials ran; 'patience' once the last `patience` rounds (patience > 0) did not raise the best finite
  objective (to be maximised) above the best before them; else None."""
  if n_done >= hpo['max_trials']: return 'max_trials'
  p = hpo['patience']
  if p > 0 and len(best_after_round) > p:
    before, after = best_after_round[-p - 1], best_after_round[-1]
    if not after > before: return 'patience'
  return None


def trial_objective(scores: Sequence[float]) -> float:
  """The minimum over envs of the scores, NaN when any env's score is not finite (a run that diverged on one env fails the trial)."""
  return min(scores) if all(math.isfinite(x) for x in scores) else float('nan')


def fit_data(trials: List[Dict[str, Any]], sign: float) -> Tuple[torch.Tensor, torch.Tensor]:
  """(X, y) of the trials with a finite objective (diverged trials are left out of the fit); y = sign x objective, to be maximised."""
  ok = [t for t in trials if not t['failed']]
  if not ok: return torch.zeros(0, 0, dtype=torch.float64), torch.zeros(0, dtype=torch.float64)
  return torch.tensor([t['x'] for t in ok], dtype=torch.float64), torch.tensor([sign * t['objective'] for t in ok], dtype=torch.float64)


def trial_jobs(base: Sequence[str], trials: List[Dict[str, Any]], env: str, seed0: int, R: int) -> List[SweepJob]:
  """One SweepJob per trial for one env: the fixed overrides, env, the trial's decoded values and seed = seed0 + t R (t = the trial number)."""
  return [SweepJob(t['trial'], list(base) + [f'env={env}'] + t['overrides'] + [f'seed={seed0 + t["trial"] * R}']) for t in trials]


def round_plan(out_dir: str, r: int, env_groups: Dict[str, List[List[int]]]) -> Dict[str, List[str]]:
  """How a resumed search finishes round r: checkpoint.group_plan of every program (env -> the trial numbers of each of its programs). A
  program is skipped once its trials have their metrics.pth and their scores are recorded in checkpoint/round<r>/scores.json; one with a
  checkpoint continues from it; the rest run."""
  root = os.path.join(out_dir, 'checkpoint', f'round{r}')
  done = checkpoint.read_scores(root)
  return {env: [checkpoint.group_plan([os.path.join(out_dir, str(j), env) for j in g], all(str(j) in done.get(env, {}) for j in g), os.path.join(root, env, f'group{k}'))
                for k, g in enumerate(groups)] for env, groups in env_groups.items()}


def run_trials(base: Sequence[str], trials: List[Dict[str, Any]], out_dir: str, seed0: int, R: int, round_index: Optional[int] = None, resume: bool = False) -> List[int]:
  """Trains the trials on every env (env after env; each env's trials as the programs of config.sweep_groups) and fills each trial's
  `scores` {env: train() score}. Returns the number of programs per env. round_index (checkpoint.interval set): program k of env e checkpoints
  into <out_dir>/checkpoint/round<r>/<e>/group<k>, and the scores of finished programs go to checkpoint/round<r>/scores.json; resume: finish
  the round as round_plan says."""
  from .environments import ENVS
  from .train import _train
  root = None if round_index is None else os.path.join(out_dir, 'checkpoint', f'round{round_index}')
  done = checkpoint.read_scores(root) if resume else {}
  programs = []
  for env in ENVS:
    jobs = trial_jobs(base, trials, env, seed0, R)
    groups = sweep_groups(jobs)
    programs.append(len(groups))
    print(f'env {env}: {len(jobs)} trial(s) in {len(groups)} program(s)', flush=True)
    by_num = {t['trial']: t for t in trials}
    plan = round_plan(out_dir, round_index, {env: [[j.num for j in g.jobs] for g in groups]})[env] if resume else ['run'] * len(groups)
    for k, g in enumerate(groups):
      if plan[k] == 'skip':
        for j in g.jobs: by_num[j.num]['scores'][env] = done[env][str(j.num)]
        continue
      cfg = load_config(g.overrides)
      J = len(g.jobs)
      cfg.replicas = J * R
      per_replica = {k: replica_values(k, vals, R) for k, vals in g.per_job.items()}
      blocks = []
      for i, j in enumerate(g.jobs):
        d = os.path.join(out_dir, str(j.num), env)
        os.makedirs(d, exist_ok=True)
        blocks.append((d + os.sep, f'trial {j.num} {env}: ', i * R, (i + 1) * R))
      gdir = os.path.join(root, env, f'group{k}') if root is not None and checkpoint.interval_of(cfg) else None
      for j, s in zip(g.jobs, _train(cfg, blocks, per_replica, checkpoint_dir=gdir, overrides=g.overrides, resume=plan[k] == 'continue')): by_num[j.num]['scores'][env] = s
      if root is not None:
        done.setdefault(env, {}).update({str(j.num): by_num[j.num]['scores'][env] for j in g.jobs})
        checkpoint.write_scores(root, done)
        checkpoint.remove(gdir)
  return programs


def search(argv: Sequence[str], resume_dir: Optional[str] = None) -> Dict[str, Any]:
  """`train_all.py -m algorithm=<ALG> [fixed overrides] [hpo.<key>=value]`: the whole search; returns the hpo.json record.

  With checkpoint.interval the search directory also holds multirun.yaml (`argv`) and the checkpoints of the running round (run_trials).
  resume_dir: continue that search: the rounds in its hpo.json are kept, the interrupted round is finished (round_plan), and later rounds
  are proposed as before (a proposal depends only on the trials so far, hpo.seed and the round index)."""
  from . import distributed
  from .environments import ENVS
  if int(os.environ.get('WORLD_SIZE', '1')) > 1: raise NotImplementedError('a hyper-parameter search runs on one GPU; searches across ranks are not supported')
  args = [a for a in argv if a not in MULTIRUN_FLAGS]
  for o in args:
    if '=' not in o: raise SweepError(f'override {o!r} is not key=value')
    _reject_sweep(o)
  hpo = load_hpo([o for o in args if o.lstrip('+').startswith('hpo.')])
  base = [o for o in args if not o.lstrip('+').startswith('hpo.')]
  cfg0 = load_config(base)
  if not seed_per_replica(cfg0): raise SweepError('a search gives every trial its own seed, which this configuration cannot take per replica (device_rng=false, or a subsampled expert memory)')
  space = Space.of(cfg0.algorithm, base)
  R, seed0, sign = int(cfg0.get('replicas', 1)), int(cfg0.seed), -1.0 if hpo['minimize'] else 1.0
  interval = checkpoint.interval_of(cfg0)
  out_dir = resume_dir or os.path.join(cfg0.get('output_dir', './outputs'), f'{cfg0.algorithm}_all_sweeper', time.strftime('%m-%d_%H-%M-%S'))
  os.makedirs(out_dir, exist_ok=True)
  record = dict(algorithm=cfg0.algorithm, overrides=base, hpo=hpo, envs=list(ENVS), searched=[p.key for p in space.params], group_keys=[p.key for p in space.group_params],
                d=space.d, trials=[], rounds=[])
  print(f'search: {cfg0.algorithm}, {len(space.params)} searched key(s) in {space.d} dimension(s), grouping on {record["group_keys"] or "nothing"}', flush=True)
  best_after, n_sobol, reason = [], 0, None
  if resume_dir:
    record, best_after, n_sobol = completed_rounds(resume_dir, record, space, hpo, sign)
    reason = stop_reason(best_after, len(record['trials']), hpo) if record['rounds'] else None
    print(f'resuming at round {len(record["rounds"])} with {len(record["trials"])} finished trial(s)', flush=True)
  elif interval:
    with open(os.path.join(out_dir, 'multirun.yaml'), 'w') as f: yaml.safe_dump(list(argv), f)
  resumed_round = len(record['rounds']) if resume_dir else None
  try:
    while reason is None:
      q = round_size(len(record['trials']), hpo)
      r = len(record['rounds'])
      X, y = fit_data(record['trials'], sign)
      if len(y) == 0:  # no finite objective yet: continue the Sobol sequence
        xs, used = sobol_round(space, q, hpo['seed'], n_sobol, hpo['max_groups'])
        info, n_sobol = dict(kind='sobol'), n_sobol + used
      else:
        xs, info = propose(space, X, y, q, hpo['candidates'], hpo['max_groups'], hpo['seed'] * 1000003 + r)
        info['kind'] = 'gp'
      trials = []
      for x in xs:
        values = space.decode(x)
        t = dict(trial=len(record['trials']) + len(trials), round=r, values=values, overrides=Space.overrides(values), x=x.tolist(), scores={})
        trials.append(t)
        d = os.path.join(out_dir, str(t['trial']))
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, 'overrides.yaml'), 'w') as f: yaml.safe_dump(list(base) + t['overrides'] + [f'seed={seed0 + t["trial"] * R}'], f)
      print(f'round {r} ({info["kind"]}): {len(trials)} trial(s)', flush=True)
      info['programs_per_env'] = run_trials(base, trials, out_dir, seed0, R, **(dict(round_index=r, resume=r == resumed_round) if interval else {}))
      for t in trials:
        t['objective'] = trial_objective([t['scores'][e] for e in ENVS])
        t['failed'] = not math.isfinite(t['objective'])
        print(f'trial {t["trial"]}: {" ".join(t["overrides"])}: objective {t["objective"]:.4f}' + (' (failed: excluded from the fit)' if t['failed'] else ''), flush=True)
      record['trials'].extend(trials)
      record['rounds'].append(info)
      finite = [sign * t['objective'] for t in record['trials'] if not t['failed']]
      best_after.append(max(finite) if finite else -math.inf)
      reason = stop_reason(best_after, len(record['trials']), hpo)
      if not trials: reason = 'no admissible candidate'
      with open(os.path.join(out_dir, 'hpo.json'), 'w') as f: json.dump(record, f, indent=1)
      if interval: checkpoint.remove(os.path.join(out_dir, 'checkpoint', f'round{r}'))
  finally:
    distributed.shutdown()
  ok = [t for t in record['trials'] if not t['failed']]
  best = max(ok, key=lambda t: (sign * t['objective'], -t['trial'])) if ok else None
  record['stopped'] = reason
  record['best'] = None if best is None else dict(trial=best['trial'], objective=best['objective'], values=best['values'])
  record['failed'] = [t['trial'] for t in record['trials'] if t['failed']]
  with open(os.path.join(out_dir, 'hpo.json'), 'w') as f: json.dump(record, f, indent=1)
  record['dir'] = out_dir
  print(f'search stopped ({reason}) after {len(record["trials"])} trial(s); {len(record["failed"])} failed', flush=True)
  if best is not None: print(f'best: trial {best["trial"]}: objective {best["objective"]:.4f}: {" ".join(best["overrides"])}', flush=True)
  return record


def completed_rounds(out_dir: str, record: Dict[str, Any], space: Space, hpo: Dict[str, Any], sign: float) -> Tuple[Dict[str, Any], List[float], int]:
  """(record, best objective after each round, Sobol points consumed) of the rounds a search in out_dir finished, from its hpo.json (the
  fresh `record` when it finished none). A record of another configuration or other search settings is refused."""
  path = os.path.join(out_dir, 'hpo.json')
  if not os.path.isfile(path): return record, [], 0
  with open(path) as f: saved = json.load(f)
  for k in ('algorithm', 'overrides', 'hpo', 'envs', 'searched', 'group_keys', 'd'):
    if saved.get(k) != record[k]: raise checkpoint.CheckpointError(f'{path}: {k} differs from the search\'s command line')
  best_after, n_sobol, n = [], 0, 0
  for r, info in enumerate(saved['rounds']):
    if info['kind'] == 'sobol': n_sobol += sobol_round(space, round_size(n, hpo), hpo['seed'], n_sobol, hpo['max_groups'])[1]
    n += sum(1 for t in saved['trials'] if t['round'] == r)
    finite = [sign * t['objective'] for t in saved['trials'][:n] if not t['failed']]
    best_after.append(max(finite) if finite else -math.inf)
  return saved, best_after, n_sobol


def train_all(argv: Sequence[str]) -> float:
  """`train_all.py algorithm=<ALG> [overrides]`: the configuration trained on every env with the same seed, files under
  <output_dir>/<ALG>_all/<timestamp>/<env>/; returns the minimum over envs of train()'s score."""
  from . import distributed
  from .environments import ENVS
  from .train import train
  for o in argv: _reject_sweep(o)
  cfg0 = load_config(list(argv))
  out_dir = os.path.join(cfg0.get('output_dir', './outputs'), f'{cfg0.algorithm}_all', time.strftime('%m-%d_%H-%M-%S'))
  scores = []
  try:
    for env in ENVS:
      os.makedirs(os.path.join(out_dir, env), exist_ok=True)
      scores.append(train(load_config(list(argv) + [f'env={env}']), file_prefix=os.path.join(out_dir, env) + os.sep))
  finally:
    distributed.shutdown()
  print(f'min over envs: {min(scores):.4f} ({", ".join(f"{e} {s:.4f}" for e, s in zip(ENVS, scores))})', flush=True)
  return min(scores)


def main(argv: Optional[Sequence[str]] = None):
  import sys
  argv = list(sys.argv[1:] if argv is None else argv)
  target = [a for a in argv if a.startswith('resume=')]
  if target:  # `train_all.py resume=<search dir>`
    d, others = target[0].partition('=')[2], [a for a in argv if a != target[0]]
    if others: raise SystemExit(f'resume refused: resume= takes no other override (the configuration comes from the search); got {" ".join(others)}')
    if not os.path.isfile(os.path.join(d, 'multirun.yaml')): raise SystemExit(f'resume refused: {d} holds no checkpointed search (multirun.yaml)')
    with open(os.path.join(d, 'multirun.yaml')) as f: return search(yaml.safe_load(f), resume_dir=d)
  return search(argv) if any(a in MULTIRUN_FLAGS for a in argv) else train_all(argv)
