"""CPU checks of the seed-sweep statistics: the float64 restatement (oracle/iqm.py) against scipy and a direct per-rep loop, the host
Philox restatement against the Random123 known answers, the sweep-output loader on synthetic metrics.pth files in both formats, and the
results script's argument parsing and path resolution."""
import os
import sys

import numpy as np
import pytest
import scipy.stats
import torch

from il_b200 import results
from oracle import iqm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'scripts'))
import print_seed_sweep_results as cli  # noqa: E402


@pytest.mark.parametrize('n', range(1, 65))
def test_oracle_trim_mean_equals_scipy_with_ties(n):
  rng = np.random.default_rng(n)
  for trial in range(8):
    x = rng.integers(0, 4, size=n) * 0.37 + (rng.random(n) if trial % 2 else 0.0)  # even trials: only ties
    ref = scipy.stats.trim_mean(x, 0.25)
    assert abs(iqm.trim_mean(x) - ref) <= 1e-15 * abs(ref), (n, trial)
  x = rng.random((3, 5, n))
  np.testing.assert_allclose(iqm.trim_mean(x), scipy.stats.trim_mean(x, 0.25, axis=-1), rtol=1e-15, atol=0)


def test_oracle_bootstrap_is_the_trim_mean_of_each_gathered_resample():
  rng = np.random.default_rng(1)
  runs, envs, T, reps = 7, 3, 4, 5
  scores = rng.random((runs, envs, T))
  idx = iqm.stratified_indices(rng, reps, T, envs, runs)
  out = iqm.bootstrap_iqm(scores, idx, chunk=2)
  for r in range(reps):
    for t in range(T):
      vals = [scores[idx[r, t, e, k], e, t] for e in range(envs) for k in range(runs)]
      assert out[r, t] == pytest.approx(scipy.stats.trim_mean(vals, 0.25), rel=1e-15)
  assert np.allclose(iqm.aggregate_iqm(scores), [scipy.stats.trim_mean(scores[..., t].reshape(-1), 0.25) for t in range(T)], rtol=1e-15, atol=0)


def test_host_philox_matches_random123_known_answers_and_maps_into_range():
  z, f = np.uint64(0), np.uint64(0xFFFFFFFF)
  assert [int(v) for v in iqm._philox4x32_10(z, z, z, z, 0, 0)] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
  assert [int(v) for v in iqm._philox4x32_10(f, f, f, f, 0xFFFFFFFF, 0xFFFFFFFF)] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
  idx = iqm.philox_indices(2**40 + 5, 6, 3, 2, 11)
  assert idx.shape == (6, 3, 2, 11) and idx.min() >= 0 and idx.max() < 11
  assert not np.array_equal(idx, iqm.philox_indices(2**40 + 6, 6, 3, 2, 11))


# ---- loader ----------------------------------------------------------------------------------------------------------------------
def _job(d, steps, returns, normalized=None):
  os.makedirs(d, exist_ok=True)
  normalized = returns if normalized is None else normalized
  torch.save(dict(test_steps=list(steps), test_returns=returns, test_returns_normalized=normalized, train_steps=[]), os.path.join(d, 'metrics.pth'))


def _flat(tag, T=2, E=3):
  """replicas=1 job: one list of E episodes per evaluation; values encode (tag, t, episode)."""
  return [[tag + 0.01 * t + 0.0001 * e for e in range(E)] for t in range(T)]


def _nested(tag, R, T=2, E=3):
  return [[[tag + r + 0.01 * t + 0.0001 * e for e in range(E)] for r in range(R)] for t in range(T)]


def test_loader_reads_both_formats_job_major_replica_minor(tmp_path):
  a = tmp_path / 'flat'
  for j in (0, 1, 2, 10): _job(str(a / str(j)), [10, 20], _flat(100 * j))  # 10 sorts after 2 numerically
  os.makedirs(a / 'not_a_job')
  steps, r = results.load_sweep_returns(str(a))
  assert steps == [10, 20] and r.shape == (4, 2, 3)
  assert r[:, 0, 0].tolist() == [0, 100, 200, 1000]
  b = tmp_path / 'nested'
  for j in (0, 1): _job(str(b / str(j)), [10, 20], _nested(100 * j, R=2))
  steps, r = results.load_sweep_returns(str(b))
  assert r.shape == (4, 2, 3) and r[:, 0, 0].tolist() == [0, 1, 100, 101]
  assert r[1, 1, 2] == pytest.approx(1 + 0.01 + 0.0002)


def test_loader_unnormalise_picks_the_raw_returns(tmp_path):
  d = tmp_path / 's'
  _job(str(d / '0'), [5], [[1000.0, 2000.0]], [[0.1, 0.2]])
  assert results.load_sweep_returns(str(d))[1].tolist() == [[[0.1, 0.2]]]
  assert results.load_sweep_returns(str(d), unnormalise=True)[1].tolist() == [[[1000.0, 2000.0]]]


def test_loader_truncates_to_the_requested_seeds(tmp_path):
  dirs = []
  for env, R in (('hopper', 3), ('walker2d', 5)):
    d = tmp_path / env
    _job(str(d / '0'), [10, 20], _nested(0, R=R))
    dirs.append(str(d))
  steps, per_env = results.load_returns(dirs, seeds=3)
  assert [r.shape[0] for r in per_env] == [3, 3] and per_env[1][:, 0, 0].tolist() == [0, 1, 2]
  with pytest.raises(ValueError, match='fewer than the 4 requested'): results.load_returns(dirs, seeds=4)
  with pytest.raises(ValueError, match='5 runs, but'): results.load_returns(dirs, seeds=None)


def test_loader_refusals(tmp_path):
  d = tmp_path / 'steps'
  _job(str(d / '0'), [10, 20], _flat(0))
  _job(str(d / '1'), [10, 30], _flat(1))
  with pytest.raises(ValueError, match='test_steps'): results.load_sweep_returns(str(d))
  e1, e2 = tmp_path / 'e1', tmp_path / 'e2'
  _job(str(e1 / '0'), [10, 20], _flat(0))
  _job(str(e2 / '0'), [10], _flat(0, T=1))
  with pytest.raises(ValueError, match='test_steps'): results.load_returns([str(e1), str(e2)])
  n = tmp_path / 'nan'
  bad = _flat(0)
  bad[1][2] = float('nan')
  _job(str(n / '0'), [10, 20], bad)
  with pytest.raises(ValueError, match='non-finite'): results.load_sweep_returns(str(n))
  i = tmp_path / 'inf'
  _job(str(i / '0'), [10, 20], _flat(0), normalized=[[0.0, float('inf'), 0.0], [0.0, 0.0, 0.0]])
  results.load_sweep_returns(str(i), unnormalise=True)
  with pytest.raises(ValueError, match='non-finite'): results.load_sweep_returns(str(i))
  z = tmp_path / 'empty'
  os.makedirs(z)
  with pytest.raises(ValueError, match='no job directories'): results.load_sweep_returns(str(z))
  s = tmp_path / 'shape'
  _job(str(s / '0'), [10, 20], _flat(0, T=3))
  with pytest.raises(ValueError, match='shape'): results.load_sweep_returns(str(s))


def test_loader_pools_only_jobs_that_differ_in_the_seed(tmp_path):
  import yaml

  def job(d, overrides, tag):
    _job(str(d), [10, 20], _flat(tag))
    with open(os.path.join(str(d), 'overrides.yaml'), 'w') as f: yaml.safe_dump(overrides, f)
  ok = tmp_path / 'seeds'
  for j, s in enumerate((1, 2, 3)): job(ok / str(j), ['algorithm=GAIL', 'env=hopper', f'seed={s}', 'replicas=2'], j)
  assert results.load_sweep_returns(str(ok))[1].shape[0] == 3
  grid = tmp_path / 'grid'
  for j, (s, lr) in enumerate(((1, '1e-4'), (1, '3e-4'))): job(grid / str(j), ['algorithm=GAIL', 'env=hopper', f'seed={s}', f'training.learning_rate={lr}'], j)
  with pytest.raises(ValueError, match='more than the seed'): results.load_sweep_returns(str(grid))


# ---- script --------------------------------------------------------------------------------------------------------------------
def test_script_arguments():
  a = cli.parse_args([])
  assert a.reps == 50000 and a.seeds == 10 and not a.unnormalise and a.bootstrap_seed == 0 and a.out is None
  assert a.algorithms == cli.ALGORITHMS and a.envs == ['ant', 'halfcheetah', 'hopper', 'walker2d'] and a.trajectories == ['5', '10', '25']
  assert a.path == os.path.join('outputs', '{algorithm}_{env}_sweeper', 'traj_{trajectories}')
  a = cli.parse_args(['--reps', '100', '--algorithms', 'GAIL,RED', '--envs', 'hopper', '--seeds', '3', '--unnormalise', '--bootstrap-seed', '7', '--out', 'x.json',
                      '--path', 'runs/{algorithm}/{env}/*', '--trajectories', '10'])
  assert (a.reps, a.algorithms, a.envs, a.seeds, a.unnormalise, a.bootstrap_seed, a.out, a.path, a.trajectories) == (100, ['GAIL', 'RED'], ['hopper'], 3, True, 7, 'x.json',
                                                                                                                  'runs/{algorithm}/{env}/*', ['10'])
  assert cli.parse_args(['--algorithms', 'SAC']).trajectories == ['0']  # the reference's SAC special case
  for bad in (['--reps', '0'], ['--seeds', '0'], ['--bootstrap-seed', '-1']):
    with pytest.raises(SystemExit): cli.parse_args(bad)


def test_path_resolution_needs_exactly_one_directory(tmp_path):
  os.makedirs(tmp_path / 'GAIL_hopper_sweeper' / 'traj_5')
  os.makedirs(tmp_path / 'GAIL_walker2d_sweeper' / '01-01_00-00-00')
  os.makedirs(tmp_path / 'GAIL_walker2d_sweeper' / '01-01_00-00-01')
  (tmp_path / 'RED_hopper_sweeper').write_text('a file, not a directory')
  pattern = str(tmp_path / '{algorithm}_{env}_sweeper' / 'traj_{trajectories}')
  assert results.resolve_sweep_dir(pattern, 'GAIL', 'hopper', '5') == str(tmp_path / 'GAIL_hopper_sweeper' / 'traj_5')
  with pytest.raises(ValueError, match='matched 0'): results.resolve_sweep_dir(pattern, 'GAIL', 'hopper', '10')
  star = str(tmp_path / '{algorithm}_{env}_sweeper' / '*')
  with pytest.raises(ValueError, match='matched 2'): results.resolve_sweep_dir(star, 'GAIL', 'walker2d', '5')
  assert results.resolve_sweep_dir(star, 'GAIL', 'hopper', '5').endswith('traj_5')
  with pytest.raises(ValueError, match='matched 0'): results.resolve_sweep_dir(str(tmp_path / '{algorithm}_{env}_sweeper'), 'RED', 'hopper', '5')
