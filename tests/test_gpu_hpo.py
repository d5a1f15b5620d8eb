"""The hyper-parameter search on the GPU: il_gp_posterior and il_gp_select against the float64 restatement (oracle/gp.py) and scikit-learn
at the block edges of the substitution and the size caps, their refusals, and `train_all.py` end to end (search rounds, grouping, files, and a
trial-env being bitwise the single `train.py` run of its overrides)."""
import ctypes as C
import glob
import json
import os

import numpy as np
import pytest
import torch

from oracle import gp as ogp

pytestmark = pytest.mark.gpu

S2, NOISE = 1.3, 0.05
GAIL_D = 22  # the encoded dimension of GAIL's search space (tests/test_hpo_cpu.py pins it)


def _problem(n, d, M, seed=0):
  rng = np.random.default_rng(seed)
  X, C_ = rng.random((n, d)), rng.random((M, d))
  y = rng.standard_normal(n)
  ls = 0.5 * np.sqrt(d) * (0.6 + 0.8 * rng.random(d))
  return X, y, C_, ls


def _fit(X, y, ls, s2=S2, noise=NOISE):
  from il_b200.hpo import GpFit
  L, alpha = ogp.posterior(X, y, X[:1], ls, s2, noise)[3:]
  t = lambda a: torch.tensor(a, dtype=torch.float64, device='cuda')
  return GpFit(t(X), t(y), 0.0, 1.0, torch.tensor(ls, dtype=torch.float64), s2, noise, t(L), t(alpha), 0.0)


def _posterior(X, y, C_, ls, extra=0):
  from il_b200.hpo import gp_posterior
  fit = _fit(X, y, ls)
  mu, var, V = gp_posterior(fit, torch.tensor(C_, dtype=torch.float64, device='cuda'), extra_rows=extra)
  return fit, mu, var, V


def _close(a, b, scale, what):
  err = np.max(np.abs(np.asarray(a) - np.asarray(b))) / scale
  assert err <= 1e-10, f'{what}: max error {err:.3g} x scale'


CASES = [(n, 7, 1000) for n in (1, 2, 31, 32, 33, 63, 64, 65, 1024, 4096)] + [(65, d, 1000) for d in (1, 7, GAIL_D, 64)] + [(64, 7, M) for M in (1, 1000, 65536 + 3)]


@pytest.mark.parametrize('n,d,M', CASES)
def test_posterior_matches_oracle(n, d, M):
  X, y, C_, ls = _problem(n, d, M)
  _, mu, var, V = _posterior(X, y, C_, ls)
  mu_o, var_o, V_o, _, _ = ogp.posterior(X, y, C_, ls, S2, NOISE)
  # relative to the scale of each quantity: the mean's largest magnitude, the prior variance, V's largest entry
  _close(mu.cpu().numpy(), mu_o, max(1.0, np.abs(mu_o).max()), 'mu')
  _close(var.cpu().numpy(), var_o, S2, 'var')
  _close(V.cpu().numpy(), V_o, max(1.0, np.abs(V_o).max()), 'V = L^-1 K*^T')


@pytest.mark.parametrize('n,d,M', [(33, 7, 1000), (65, GAIL_D, 3000)])
def test_posterior_matches_sklearn(n, d, M):
  from sklearn.gaussian_process import GaussianProcessRegressor
  from sklearn.gaussian_process.kernels import ConstantKernel, Matern
  X, y, C_, ls = _problem(n, d, M, seed=3)
  _, mu, var, _ = _posterior(X, y, C_, ls)
  gpr = GaussianProcessRegressor(ConstantKernel(S2, 'fixed') * Matern(ls, 'fixed', nu=2.5), alpha=NOISE, optimizer=None).fit(X, y)
  m, s = gpr.predict(C_, return_std=True)
  _close(mu.cpu().numpy(), m, max(1.0, np.abs(m).max()), 'mu vs sklearn')
  _close(var.cpu().numpy(), s**2, S2, 'var vs sklearn')


def _select(n, d, M, q, group=None, G=0, seed=1):
  from il_b200.hpo import gp_select
  X, y, C_, ls = _problem(n, d, M, seed)
  fit, mu, var, V = _posterior(X, y, C_, ls, extra=q)
  fstar = float(np.max(ogp.matern52(X, X, ls, S2) @ fit.alpha.cpu().numpy()))
  g = torch.tensor(np.zeros(M) if group is None else group, dtype=torch.int32, device='cuda')
  mu_o, var_o, V_o, _, _ = ogp.posterior(X, y, C_, ls, S2, NOISE)
  picks, ei = gp_select(fit, torch.tensor(C_, dtype=torch.float64, device='cuda'), mu, var, V, g, q, G, fstar)
  return X, y, C_, ls, mu_o, var_o, V_o, fstar, picks, ei, var.cpu().numpy()


def _assert_separated(C_, mu_o, var_o, V_o, ls, fstar, picks_o, group=None, G=0):
  """No two admissible candidates' EI lie within 1e-12 relative at any greedy step (so the argmax is not a rounding decision)."""
  for j in range(len(picks_o)):
    sub = picks_o[:j]
    _, _, var_j = ogp.select(C_, mu_o, var_o, V_o, ls, S2, NOISE, fstar, j, group, G)
    f = max([fstar] + [mu_o[p] for p in sub])
    ei = ogp.expected_improvement(mu_o, var_j, f)
    ok = np.ones(len(C_), bool)
    ok[list(sub)] = False
    if G > 0:
      adm = list(dict.fromkeys(group[p] for p in sub))
      if len(adm) >= G: ok &= np.isin(group, adm)
    top = np.sort(ei[ok])[-2:]
    if len(top) == 2: assert top[1] - top[0] > 1e-12 * abs(top[1]), f'step {j}: EI tie within 1e-12'


@pytest.mark.parametrize('q', [1, 8, 64])
def test_select_matches_oracle_and_sklearn_refit(q):
  from sklearn.gaussian_process import GaussianProcessRegressor
  from sklearn.gaussian_process.kernels import ConstantKernel, Matern
  X, y, C_, ls, mu_o, var_o, V_o, fstar, picks, ei, var_after = _select(50, 5, 2000, q)
  picks_o, ei_o, var_after_o = ogp.select(C_, mu_o, var_o, V_o, ls, S2, NOISE, fstar, q)
  _assert_separated(C_, mu_o, var_o, V_o, ls, fstar, picks_o)
  assert picks == picks_o.tolist()
  _close(ei, ei_o, max(1e-3, np.abs(ei_o).max()), 'EI')
  _close(var_after, var_after_o, S2, 'var after picks vs oracle')
  Xa = np.concatenate([X, C_[picks_o]])
  ya = np.concatenate([y, mu_o[picks_o]])  # the kriging believer: each pick observed at its posterior mean
  gpr = GaussianProcessRegressor(ConstantKernel(S2, 'fixed') * Matern(ls, 'fixed', nu=2.5), alpha=NOISE, optimizer=None).fit(Xa, ya)
  m, s = gpr.predict(C_, return_std=True)
  _close(var_after, s**2, S2, 'var after picks vs sklearn refit')
  _close(m, mu_o, max(1.0, np.abs(mu_o).max()), 'believed means leave the mean unchanged')


@pytest.mark.parametrize('G', [1, 2])
def test_select_max_groups(G):
  M, q = 2000, 16
  group = np.random.default_rng(5).integers(0, 10, M)
  X, y, C_, ls, mu_o, var_o, V_o, fstar, picks, ei, _ = _select(40, 4, M, q, group, G, seed=2)
  assert len({group[p] for p in picks if p >= 0}) <= G
  picks_o, ei_o, _ = ogp.select(C_, mu_o, var_o, V_o, ls, S2, NOISE, fstar, q, group, G)
  _assert_separated(C_, mu_o, var_o, V_o, ls, fstar, picks_o, group, G)
  assert picks == picks_o.tolist()
  _close(ei, ei_o, max(1e-3, np.abs(ei_o).max()), 'EI')


def test_select_runs_out_of_candidates():
  """max_groups=1 with five candidates per group: after the first group's five picks, the remaining picks are -1 with NaN EI."""
  M, q = 10, 8
  group = np.array([0, 0, 0, 0, 0, 1, 1, 1, 1, 1])
  X, y, C_, ls, mu_o, var_o, V_o, fstar, picks, ei, _ = _select(20, 3, M, q, group, 1, seed=4)
  valid = [p for p in picks if p >= 0]
  assert len(valid) == 5 and len({group[p] for p in valid}) == 1 and picks[5:] == [-1] * 3 and all(np.isnan(ei[5:]))
  assert picks == ogp.select(C_, mu_o, var_o, V_o, ls, S2, NOISE, fstar, q, group, 1)[0].tolist()


def test_abi_refusals():
  from il_b200 import _lib
  lib, h, st = _lib.lib(), _lib.handle(), _lib.stream()
  n, d, M, q = 8, 3, 16, 4
  buf = torch.zeros(1 << 16, dtype=torch.float64, device='cuda')
  p, o = buf.data_ptr(), buf[1 << 15:].data_ptr()
  ls = (C.c_double * d)(0.5, 0.5, 0.5)
  post = lambda **kw: lib.il_gp_posterior(kw.get('h', h), p, p, p, kw.get('n', n), kw.get('d', d), kw.get('Ct', p), kw.get('M', M), kw.get('ls', ls), kw.get('s2', 1.0),
                                          kw.get('noise', 0.1), o, o + 8 * M, o + 16 * M, st)
  assert post() == 0
  for kw in (dict(h=None), dict(Ct=None), dict(ls=None), dict(n=0), dict(n=_lib.GP_MAX_N + 1), dict(d=0), dict(d=_lib.GP_MAX_D + 1), dict(M=0),
             dict(M=_lib.GP_MAX_M + 1), dict(s2=float('nan')), dict(s2=0.0), dict(noise=-1.0), dict(noise=float('inf')), dict(ls=(C.c_double * d)(0.5, float('nan'), 0.5)),
             dict(ls=(C.c_double * d)(0.5, 0.0, 0.5))):
    assert post(**kw) != 0, kw
    assert _lib.last_error().startswith('il_gp_posterior')
  assert lib.il_gp_select_workspace_bytes(n, d, M, M + 1) == -1 and lib.il_gp_select_workspace_bytes(0, d, M, q) == -1
  ws_bytes = lib.il_gp_select_workspace_bytes(n, d, M, q)
  ws = torch.zeros(ws_bytes, dtype=torch.uint8, device='cuda')
  sel = lambda **kw: lib.il_gp_select(h, kw.get('n', n), d, p, M, ls, 1.0, kw.get('noise', 0.1), p, p, p, kw.get('group', p), kw.get('G', 0), kw.get('fstar', 0.0),
                                      kw.get('q', q), p, p, kw.get('ws', ws.data_ptr()), kw.get('wsb', ws_bytes), st)
  for kw in (dict(ws=None), dict(group=None), dict(wsb=ws_bytes - 1), dict(q=0), dict(q=M + 1), dict(G=-1), dict(fstar=float('nan')), dict(noise=0.0), dict(n=0)):
    assert sel(**kw) != 0, kw
    assert _lib.last_error().startswith('il_gp_select')
  torch.cuda.synchronize()


# ---- end to end -----------------------------------------------------------------------------------------------------------------
SHORT = ['steps=60', 'evaluation.interval=30', 'evaluation.episodes=1', 'logging.interval=20', 'imitation.trajectories=2', 'memory.size=100',
         'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32']
ENVS = ['ant', 'halfcheetah', 'hopper', 'walker2d']


def _min_avg(trial_dir):
  return min(float(np.mean(np.asarray(torch.load(os.path.join(trial_dir, e, 'metrics.pth'), weights_only=False)['test_returns_normalized'], dtype=np.float64)))
             for e in ENVS)


def test_search_sac_end_to_end(tmp_path, capsys):
  from il_b200.hpo import main
  from il_b200.train import main as train_main
  out = str(tmp_path / 'search')
  rec = main(['-m', 'algorithm=SAC'] + SHORT + ['training.start=20', 'training.batch_size=32', 'hpo.initial=8', 'hpo.batch=4', 'hpo.max_trials=12',
                                                'hpo.candidates=4096', f'output_dir={out}'])
  text = capsys.readouterr().out
  (run, ) = glob.glob(os.path.join(out, 'SAC_all_sweeper', '*'))
  with open(os.path.join(run, 'hpo.json')) as f: saved = json.load(f)
  assert len(saved['trials']) == 12 and [r['kind'] for r in saved['rounds']] == ['sobol', 'gp']
  assert all(r['programs_per_env'] == [1, 1, 1, 1] for r in saved['rounds']) and text.count('in 1 program(s)') == 8
  assert len(saved['rounds'][1]['picks']) == 4 and saved['rounds'][1]['gp']['lengthscales']
  for t in saved['trials']:
    d = os.path.join(run, str(t['trial']))
    assert os.path.isfile(os.path.join(d, 'overrides.yaml'))
    for e in ENVS:
      for f in ('agent.pth', 'metrics.pth'): assert os.path.isfile(os.path.join(d, e, f)), (t['trial'], e, f)
    assert t['objective'] == min(t['scores'].values())
    np.testing.assert_allclose(t['objective'], _min_avg(d), rtol=1e-5, atol=1e-6)
  assert saved['best']['trial'] == max(saved['trials'], key=lambda t: t['objective'])['trial'] and rec['best'] == saved['best']
  # one trial-env of the GP round, rerun as a single train.py command, writes the same files bit for bit
  t = saved['trials'][9]
  import yaml
  with open(os.path.join(run, '9', 'overrides.yaml')) as f: ov = yaml.safe_load(f)
  single = str(tmp_path / 'single')
  train_main(ov + ['env=hopper', f'output_dir={single}'])
  (sd, ) = glob.glob(os.path.join(single, '*', '*'))
  for f in ('agent.pth', 'metrics.pth'):
    a, b = (torch.load(os.path.join(x, f), weights_only=False) for x in (os.path.join(run, '9', 'hopper'), sd))
    _same(a, b, f)


def _same(a, b, where):
  if isinstance(a, torch.Tensor): assert torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8)), where
  elif isinstance(a, np.ndarray): assert a.dtype == b.dtype and a.tobytes() == b.tobytes(), where
  elif isinstance(a, dict):
    assert set(a) == set(b), where
    for k in a: _same(a[k], b[k], f'{where}.{k}')
  elif isinstance(a, (list, tuple)):
    assert len(a) == len(b), where
    for i, (x, y) in enumerate(zip(a, b)): _same(x, y, f'{where}[{i}]')
  else: assert a == b or (a != a and b != b), f'{where}: {a!r} != {b!r}'


def test_search_gail_max_groups(tmp_path):
  from il_b200.hpo import main
  out = str(tmp_path / 'gail')
  main(['-m', 'algorithm=GAIL'] + SHORT + ['hpo.initial=6', 'hpo.batch=6', 'hpo.max_trials=12', 'hpo.max_groups=2', 'hpo.candidates=4096', f'output_dir={out}'])
  (run, ) = glob.glob(os.path.join(out, 'GAIL_all_sweeper', '*'))
  with open(os.path.join(run, 'hpo.json')) as f: saved = json.load(f)
  assert [r['kind'] for r in saved['rounds']] == ['sobol', 'gp'] and all(max(r['programs_per_env']) <= 2 for r in saved['rounds'])
  assert len({p['group'] for p in saved['rounds'][1]['picks']}) <= 2


def test_train_all_is_min_of_train_runs(tmp_path):
  from il_b200.hpo import main
  from il_b200.train import main as train_main
  base = ['algorithm=SAC'] + SHORT + ['training.start=20', 'training.batch_size=32', 'seed=5']
  score = main(base + [f'output_dir={tmp_path / "all"}'])
  singles = [train_main(base + [f'env={e}', f'output_dir={tmp_path / e}']) for e in ENVS]
  assert score == min(singles)
  for e in ENVS: assert glob.glob(os.path.join(str(tmp_path / 'all'), 'SAC_all', '*', e, 'metrics.pth'))
