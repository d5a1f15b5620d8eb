"""The hyper-parameter search without a GPU: the shipped search spaces against the reference's (tests/golden/hp_search_spaces.json), the
encoding, grouping and Sobol round, the GP fit, round bookkeeping, the float64 oracle against scikit-learn, and scripts/print_hpo_results.py."""
import json
import math
import os
import shutil
import sys

import numpy as np
import pytest
import torch
import yaml

from il_b200 import config, hpo
from il_b200.train import check_config
from oracle import gp as ogp
from oracle import ref_search_spaces

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALGS = ref_search_spaces.ALGORITHMS
ENVS = ['ant', 'halfcheetah', 'hopper', 'walker2d']


def test_search_spaces_equal_the_reference():
  golden = ref_search_spaces.load()
  for alg in ALGS:
    spec = hpo.load_space_spec(alg)
    assert spec == golden[alg] and list(spec) == list(golden[alg]), alg


@pytest.mark.parametrize('alg', ALGS)
def test_encode_decode_round_trip_and_every_trial_loads(alg):
  base = [f'algorithm={alg}']
  space = hpo.Space.of(alg, base)
  xs, _ = hpo.sobol_round(space, 16, seed=3)
  xs = torch.cat([xs, space.snap(torch.zeros(1, space.d)), space.snap(torch.ones(1, space.d))])
  for x in xs:
    values = space.decode(x)
    assert torch.equal(space.snap(x[None])[0], x)
    again = space.decode(space.encode(values))
    for p in space.params:
      if p.kind == 'range' and p.value_type == 'float': assert math.isclose(again[p.key], values[p.key], rel_tol=1e-12, abs_tol=1e-15)
      else: assert again[p.key] == values[p.key] and type(again[p.key]) is type(values[p.key])
    cfg = config.load_config(base + ['env=hopper'] + hpo.Space.overrides(values))
    for k, v in values.items(): assert config.get_key(cfg, k) == v and type(config.get_key(cfg, k)) is type(v), k  # repr round-trips exactly
    check_config(cfg)
    config.split_per_replica(cfg, {k: [v] for k, v in values.items() if k in config.per_replica_keys(cfg)}, 1)


def test_space_dimensions_and_ignored_keys():
  gail = hpo.Space.of('GAIL', ['algorithm=GAIL'])
  keys = [p.key for p in gail.params]
  assert 'imitation.discriminator.input_dropout' not in keys and 'imitation.discriminator.dropout' not in keys
  assert gail.d == 22
  assert [p.key for p in gail.group_params] == ['training.start', 'training.batch_size', 'imitation.discriminator.hidden_size', 'imitation.discriminator.depth',
                                                 'imitation.discriminator.activation']
  red = hpo.Space.of('RED', ['algorithm=RED'])
  assert 'imitation.discriminator.dropout' in [p.key for p in red.params]


def test_fixed_overrides_leave_the_search():
  space = hpo.Space.of('SAC', ['algorithm=SAC', 'training.start=1000', 'training.batch_size=256'])
  assert [p.key for p in space.params] == ['training.learning_rate', 'reinforcement.discount', 'reinforcement.target_temperature', 'reinforcement.polyak_factor']
  assert space.d == 4 and space.group_params == []


@pytest.mark.parametrize('argv', [['-m', 'algorithm=SAC', 'training.learning_rate=0.1,0.2'], ['-m', 'algorithm=SAC', 'reinforcement.discount=range(0.9,0.99)'],
                                  ['-m', 'algorithm=SAC', 'training.start=choice(10,20)'], ['-m', 'algorithm=SAC', 'hpo.nope=1'], ['-m', 'algorithm=SAC', 'hpo.batch=0'], ['-m', 'algorithm=SAC', 'hpo.max_trials=4097'],
                                  ['algorithm=SAC', 'seed=1,2']])
def test_sweep_syntax_and_bad_settings_are_refused(argv):
  with pytest.raises(config.SweepError):
    hpo.main(argv)


def test_search_refuses_several_ranks(monkeypatch):
  monkeypatch.setenv('WORLD_SIZE', '2')
  with pytest.raises(NotImplementedError):
    hpo.search(['-m', 'algorithm=SAC'])


@pytest.mark.parametrize('alg', ['GAIL', 'RED', 'SAC'])
def test_group_ids_match_the_sweep_partition(alg):
  """Trials with equal group ids never land in different programs of config.sweep_groups."""
  base = [f'algorithm={alg}', 'env=hopper']
  space = hpo.Space.of(alg, base)
  xs, _ = hpo.sobol_round(space, 48, seed=1)
  # copies of the first 8 rows with every column outside the grouping keys redrawn: equal ids, different per-replica values
  grouped = torch.zeros(space.d, dtype=torch.bool)
  for p in space.group_params: grouped[p.col:p.col + p.width] = True
  fresh, _ = hpo.sobol_round(space, 48, seed=2)
  xs = torch.cat([xs, space.snap(torch.where(grouped, xs[:8].repeat(6, 1), fresh))])
  ids = space.group_ids(xs).tolist()
  trials = [dict(trial=i, overrides=hpo.Space.overrides(space.decode(x))) for i, x in enumerate(xs)]
  groups = config.sweep_groups(hpo.trial_jobs(base[:1], trials, 'hopper', 0, 1))
  program = {j.num: g for g, grp in enumerate(groups) for j in grp.jobs}
  for a in range(len(xs)):
    for b in range(a):
      if ids[a] == ids[b]: assert program[a] == program[b], (a, b)
  assert len(groups) <= len(set(ids))
  assert any(ids[48 + i] == ids[i] and trials[48 + i]['overrides'] != trials[i]['overrides'] for i in range(48))


def test_sobol_round_is_deterministic_and_honours_max_groups():
  space = hpo.Space.of('GAIL', ['algorithm=GAIL'])
  a, na = hpo.sobol_round(space, 8, seed=7)
  b, nb = hpo.sobol_round(space, 8, seed=7)
  assert torch.equal(a, b) and na == nb == 8 and not torch.equal(a, hpo.sobol_round(space, 8, seed=8)[0])
  c, _ = hpo.sobol_round(space, 8, seed=7, max_groups=2)
  assert len(set(space.group_ids(c).tolist())) <= 2 and len(c) == 8


def test_candidates_follow_the_documented_rule():
  space = hpo.Space.of('GAIL', ['algorithm=GAIL'])
  X, _ = hpo.sobol_round(space, 9, seed=0)
  y = torch.arange(9, dtype=torch.float64)
  Cd = hpo.candidates(space, X, y, 101, seed=5)
  assert Cd.shape == (101, space.d) and torch.equal(space.snap(Cd), Cd)
  g = torch.Generator().manual_seed(5)
  U = torch.rand(51, space.d, generator=g, dtype=torch.float64)
  assert torch.equal(Cd[:51], space.snap(U))
  parent = torch.randint(0, 5, (50, ), generator=g)
  top = X[[8, 7, 6, 5, 4]][parent]
  step = torch.randn(50, space.d, generator=g, dtype=torch.float64)
  flip = torch.rand(50, len(space.params), generator=g, dtype=torch.float64) < hpo.RESAMPLE
  for i, p in enumerate(space.params):  # a range column of a perturbed row is its parent's moved by STEP x step, clipped
    if p.kind == 'range' and p.value_type == 'float':
      assert torch.allclose(Cd[51:, p.col], (top[:, p.col] + hpo.STEP * step[:, p.col]).clamp(0, 1), rtol=0, atol=0)
    if p.kind != 'range':  # an unflipped choice keeps its parent's level
      keep = ~flip[:, i]
      assert torch.equal(Cd[51:][keep, p.col:p.col + p.width], top[keep, p.col:p.col + p.width])


def _lml_np(X, y, ls, s2, noise):
  K = ogp.matern52(X, X, ls, s2) + noise * np.eye(len(X))
  L = np.linalg.cholesky(K)
  a = np.linalg.solve(K, y)
  return -0.5 * y @ a - np.log(np.diag(L)).sum() - 0.5 * len(X) * np.log(2 * np.pi)


def test_gp_fit_on_cpu_raises_lml_and_finds_relevant_dimensions():
  rng = np.random.default_rng(0)
  X = rng.random((60, 8))
  y = np.sin(6 * X[:, 0]) + np.cos(5 * X[:, 3]) + 0.01 * rng.standard_normal(60)
  fit = hpo.fit_gp(torch.tensor(X), torch.tensor(y))
  assert fit.L.device.type == 'cpu'
  assert fit.lml >= max(fit.start_lml)
  ys = (y - y.mean()) / y.std()
  assert math.isclose(fit.lml, _lml_np(X, ys, fit.lengthscales.numpy(), fit.outputscale, fit.noise), rel_tol=1e-6)
  ls = fit.lengthscales.numpy()
  assert max(ls[[0, 3]]) < min(np.delete(ls, [0, 3])), ls
  lo, hi = hpo.GP_BOUNDS['lengthscale']
  assert (ls >= lo * (1 - 1e-9)).all() and (ls <= hi * (1 + 1e-9)).all()


def test_round_bookkeeping():
  h = dict(initial=8, batch=4, max_trials=14, patience=2)
  assert [hpo.round_size(n, h) for n in (0, 8, 12, 14)] == [8, 4, 2, 0]
  assert hpo.stop_reason([1.0], 8, h) is None and hpo.stop_reason([1.0, 2.0, 2.0], 16, h) == 'max_trials'
  assert hpo.stop_reason([1.0, 2.0, 2.0], 12, h) is None and hpo.stop_reason([1.0, 2.0, 2.0, 2.0], 12, h) == 'patience'
  assert hpo.stop_reason([1.0, 2.0, 2.0, 3.0], 12, h) is None and hpo.stop_reason([1.0] * 10, 12, dict(h, patience=0)) is None
  trials = [dict(x=[0.1], objective=0.5, failed=False), dict(x=[0.2], objective=float('nan'), failed=True), dict(x=[0.3], objective=-0.2, failed=False)]
  X, y = hpo.fit_data(trials, -1.0)
  assert X.tolist() == [[0.1], [0.3]] and y.tolist() == [-0.5, 0.2]


def test_hpo_settings_load_and_override():
  h = hpo.load_hpo([])
  assert (h['max_trials'], h['patience'], h['minimize']) == (30, 5, False)
  assert hpo.load_hpo(['hpo.batch=64', 'hpo.max_groups=2'])['batch'] == 64


@pytest.mark.parametrize('q,G', [(1, 0), (6, 0), (6, 1), (6, 2)])
def test_oracle_matches_sklearn(q, G):
  from sklearn.gaussian_process import GaussianProcessRegressor
  from sklearn.gaussian_process.kernels import ConstantKernel, Matern
  rng = np.random.default_rng(q + 10 * G)
  X, C_, y = rng.random((30, 4)), rng.random((300, 4)), rng.standard_normal(30)
  ls, s2, noise = np.array([0.4, 0.7, 1.1, 0.9]), 1.4, 0.03
  kern = lambda: ConstantKernel(s2, 'fixed') * Matern(ls, 'fixed', nu=2.5)
  mu, var, V, L, alpha = ogp.posterior(X, y, C_, ls, s2, noise)
  m, s = GaussianProcessRegressor(kern(), alpha=noise, optimizer=None).fit(X, y).predict(C_, return_std=True)
  np.testing.assert_allclose(mu, m, rtol=1e-10, atol=1e-12)
  np.testing.assert_allclose(var, s**2, rtol=1e-10, atol=1e-12)
  group = rng.integers(0, 4, len(C_))
  fstar = float(np.max(ogp.matern52(X, X, ls, s2) @ alpha))
  picks, ei, var_after = ogp.select(C_, mu, var, V, ls, s2, noise, fstar, q, group, G)
  if G: assert len(set(group[picks])) <= G
  gpr = GaussianProcessRegressor(kern(), alpha=noise, optimizer=None).fit(np.concatenate([X, C_[picks]]), np.concatenate([y, mu[picks]]))
  m2, s2_ = gpr.predict(C_, return_std=True)
  np.testing.assert_allclose(var_after, s2_**2, rtol=1e-9, atol=1e-12)
  np.testing.assert_allclose(m2, mu, rtol=1e-9, atol=1e-10)


def _fake_search(tmp, rng, replicas, diverged=None):
  """A search tree as train_all.py -m writes it, with synthetic metrics (both schemas). training.start is searched but equal in every
  trial; trial `diverged` has a NaN return on hopper (not the first env)."""
  rows = []
  for t in range(5):
    d = os.path.join(tmp, str(t))
    lr = float(rng.uniform(1e-4, 3e-4))
    with open(os.path.join(os.makedirs(d) or d, 'overrides.yaml'), 'w') as f:
      yaml.safe_dump(['algorithm=SAC', 'steps=100', 'training.start=10000', f'training.learning_rate={lr!r}', f'training.batch_size={[128, 256][t % 2]}', f'seed={t}'], f)
    per_env = []
    for e in ENVS:
      os.makedirs(os.path.join(d, e))
      r = rng.random((3, 4) if replicas == 1 else (3, replicas, 4))
      if t == diverged and e == 'hopper': r[1, ...] = np.nan
      torch.save(dict(test_steps=[10, 20, 30], test_returns_normalized=r.tolist()), os.path.join(d, e, 'metrics.pth'))
      per_env.append(r)
    rows.append((t, lr, [128, 256][t % 2], np.stack(per_env).mean(axis=tuple(range(1, per_env[0].ndim + 1))).min()))  # the reference's formula
  with open(os.path.join(tmp, 'hpo.json'), 'w') as f:
    json.dump(dict(searched=['training.start', 'training.batch_size', 'training.learning_rate']), f)
  return rows


def _conf_with(tmp_path, overlay_file):
  os.makedirs(tmp_path / 'conf' / 'optimised_hyperparameters')
  shutil.copy(os.path.join(ROOT, 'conf', 'train_config.yaml'), tmp_path / 'conf' / 'train_config.yaml')
  shutil.copytree(os.path.join(ROOT, 'conf', 'algorithm'), tmp_path / 'conf' / 'algorithm')
  shutil.copy(overlay_file, tmp_path / 'conf' / 'optimised_hyperparameters' / 'best.yaml')
  return str(tmp_path / 'conf')


@pytest.mark.parametrize('replicas,diverged', [(1, None), (3, None), (1, 2)])
def test_print_hpo_results_matches_the_reference_formula(tmp_path, replicas, diverged):
  sys.path.insert(0, os.path.join(ROOT, 'scripts'))
  import print_hpo_results
  rows = _fake_search(str(tmp_path / 'run'), np.random.default_rng(replicas), replicas, diverged)
  table = print_hpo_results.main(['--path', str(tmp_path / 'run'), '--out', str(tmp_path / 'r.json'), '--write-overlay', str(tmp_path / 'best.yaml')])
  want = sorted(rows, key=lambda r: (np.isnan(r[3]), -r[3] if not np.isnan(r[3]) else 0, r[0]))
  assert [r['trial'] for r in table] == [r[0] for r in want]
  if diverged is not None: assert np.isnan(rows[diverged][3]) and table[-1]['trial'] == diverged and np.isnan(table[-1]['min_avg_test_return'])
  for got, w in zip(table, want):
    if not np.isnan(w[3]): assert math.isclose(got['min_avg_test_return'], w[3], rel_tol=1e-12)
    assert set(got) == {'trial', 'training.learning_rate', 'training.batch_size', 'seed', 'min_avg_test_return'}  # steps and training.start never vary
  cfg = config.load_config(['optimised_hyperparameters=best'], conf_dir=_conf_with(tmp_path, tmp_path / 'best.yaml'))
  # every searched key of the best trial, the one equal across trials included; not the seed
  assert cfg.training.learning_rate == want[0][1] and cfg.training.batch_size == want[0][2] and cfg.training.start == 10000 and cfg.seed == 0


def test_print_hpo_results_overlay_needs_the_search_record(tmp_path):
  sys.path.insert(0, os.path.join(ROOT, 'scripts'))
  import print_hpo_results
  _fake_search(str(tmp_path / 'run'), np.random.default_rng(0), 1)
  os.remove(tmp_path / 'run' / 'hpo.json')
  print_hpo_results.main(['--path', str(tmp_path / 'run')])
  with pytest.raises(SystemExit):
    print_hpo_results.main(['--path', str(tmp_path / 'run'), '--write-overlay', str(tmp_path / 'best.yaml')])


def test_trial_diverged_on_a_later_env_fails_and_leaves_the_fit(tmp_path, monkeypatch):
  """A NaN score on any env, not only the first, makes the trial failed: reported and left out of fit_data."""
  assert math.isnan(hpo.trial_objective([0.5, float('nan'), 0.3])) and hpo.trial_objective([0.5, 0.2, 0.3]) == 0.2

  def fake_run_trials(base, trials, out_dir, seed0, R):
    for t in trials: t['scores'] = {e: (float('nan') if t['trial'] == 1 and e == 'hopper' else 0.1 * (t['trial'] + 1)) for e in ENVS}
    return [1] * len(ENVS)
  monkeypatch.setattr(hpo, 'run_trials', fake_run_trials)
  rec = hpo.search(['-m', 'algorithm=SAC', 'hpo.initial=3', 'hpo.max_trials=3', f'output_dir={tmp_path}'])
  assert [t['failed'] for t in rec['trials']] == [False, True, False] and rec['failed'] == [1] and math.isnan(rec['trials'][1]['objective'])
  assert rec['best']['trial'] == 2
  X, y = hpo.fit_data(rec['trials'], 1.0)
  assert X.tolist() == [rec['trials'][0]['x'], rec['trials'][2]['x']] and y.tolist() == [0.1, 0.30000000000000004]
