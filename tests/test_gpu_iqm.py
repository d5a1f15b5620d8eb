"""Seed-sweep statistics on the device (il_iqm, il_bootstrap_iqm, il_percentile_interval through il_b200.results) against the float64
restatement (oracle/iqm.py) and scipy / numpy, then a small seed sweep written by train.py and summarised by
scripts/print_seed_sweep_results.py, checked against the oracle computed from the written metrics.pth files."""
import glob
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import scipy.stats
import torch

from il_b200 import _lib, results
from oracle import iqm

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return float(np.max(np.abs(a - b) / np.maximum(np.abs(b), 1e-300)))


def _scores(rng, shape):
  """Positive scores with ties: a third of the values repeat a few levels, the rest are continuous."""
  x = 0.5 + rng.random(shape)
  tie = rng.random(shape) < 0.33
  x[tie] = 0.5 + rng.integers(0, 4, size=int(tie.sum())) * 0.25
  return x


@pytest.mark.parametrize('n', [1, 2, 3, 4, 5, 30, 31, 1000, _lib.IQM_MAX_N])
def test_iqm_equals_scipy_trim_mean(n):
  x = _scores(np.random.default_rng(n), (37, n))
  assert _rel(results.trim_mean(x), scipy.stats.trim_mean(x, 0.25, axis=-1)) <= 1e-13
  y = np.full((2, n), 3.0)  # all ties
  assert np.array_equal(results.trim_mean(y), [3.0, 3.0])


def test_iqm_refusals():
  lib, h = _lib.lib(), _lib.handle()
  x = torch.zeros(2, _lib.IQM_MAX_N + 1, dtype=torch.float64, device='cuda')
  out = torch.empty(2, dtype=torch.float64, device='cuda')
  assert lib.il_iqm(h, x.data_ptr(), 2, _lib.IQM_MAX_N + 1, out.data_ptr(), None) != 0 and 'IL_IQM_MAX_N' in _lib.last_error()
  assert lib.il_iqm(h, x.data_ptr(), 2, 0, out.data_ptr(), None) != 0
  assert lib.il_iqm(h, x.data_ptr(), 0, 4, out.data_ptr(), None) != 0
  assert lib.il_iqm(h, None, 2, 4, out.data_ptr(), None) != 0 and 'null' in _lib.last_error()
  with pytest.raises(ValueError): results.trim_mean(np.zeros((2, _lib.IQM_MAX_N + 1)))


# (runs, envs): N = 1, 3, 40 (the reference's 10 seeds x 4 envs), 4096 (1024 seeds x 4 envs) and the cap; N <= 256 runs the warp kernel
SIZES = [(1, 1), (3, 1), (10, 4), (1024, 4), (_lib.BOOTSTRAP_MAX_N // 4, 4)]


@pytest.mark.parametrize('T', [1, 100])
@pytest.mark.parametrize('runs,envs', SIZES)
def test_bootstrap_with_injected_indices_equals_oracle(runs, envs, T):
  rng = np.random.default_rng(runs * 7 + T)
  reps = 13 if runs * envs > 256 else 45  # not a multiple of the 8 warps per block or of any block size
  scores = _scores(rng, (runs, envs, T))
  idx = iqm.stratified_indices(rng, reps, T, envs, runs)
  dist = results.bootstrap_iqm(scores, reps, indices=torch.from_numpy(idx).cuda()).cpu().numpy()
  assert dist.shape == (reps, T)
  assert _rel(dist, iqm.bootstrap_iqm(scores, idx)) <= 1e-13


def test_bootstrap_refusals():
  lib, h = _lib.lib(), _lib.handle()
  cap = _lib.BOOTSTRAP_MAX_N
  assert lib.il_bootstrap_iqm_workspace_bytes(1, 4, cap // 4 + 1) == -1
  assert lib.il_bootstrap_iqm_workspace_bytes(0, 4, 10) == -1
  s = torch.zeros(cap + 4, dtype=torch.float64, device='cuda')
  out = torch.empty(4, dtype=torch.float64, device='cuda')
  ws = torch.empty(1 << 20, dtype=torch.uint8, device='cuda')
  call = lambda T, envs, runs, reps, scores=s.data_ptr(), o=out.data_ptr(), w=ws.data_ptr(), nb=ws.numel(): lib.il_bootstrap_iqm(h, scores, T, envs, runs, reps, 0, None, o, w, nb, None)
  assert call(1, 4, cap // 4 + 1, 1) != 0 and 'IL_BOOTSTRAP_MAX_N' in _lib.last_error()
  assert call(1, 1, cap + 1, 1) != 0
  for bad in ((0, 4, 10, 1), (1, 0, 10, 1), (1, 4, 0, 1), (1, 4, 10, 0), (1, -4, 10, 1)):
    assert call(*bad) != 0 and 'positive' in _lib.last_error(), bad
  assert call(1, 4, 10, 1, scores=None) != 0 and 'null' in _lib.last_error()
  assert call(1, 4, 10, 1, o=None) != 0 and 'null' in _lib.last_error()
  assert call(1, 4, 10, 1, w=None) != 0 and 'null' in _lib.last_error()
  assert call(1, 4, 10, 1, nb=16) != 0 and 'workspace' in _lib.last_error()
  assert call(1, 4, 10, 1) == 0
  with pytest.raises(ValueError): results.bootstrap_iqm(np.zeros((cap // 4 + 1, 4, 1)), 1)
  bad = torch.zeros(2, 1, 1, 3, dtype=torch.int32, device='cuda')
  bad[1, 0, 0, 2] = 3  # out of [0, runs): that rep's output is NaN, the other rep is computed
  dist = results.bootstrap_iqm(np.arange(3.0).reshape(3, 1, 1), 2, indices=bad).cpu().numpy()
  assert dist[0, 0] == 0.0 and np.isnan(dist[1, 0])


def test_non_finite_scores_are_refused():
  x = np.random.default_rng(0).random((10, 4, 3))
  for bad in (float('nan'), float('inf'), -float('inf')):
    y = x.copy()
    y[3, 1, 2] = bad
    for f in (lambda: results.bootstrap_iqm(y, 5), lambda: results.aggregate_iqm(y), lambda: results.trim_mean(y), lambda: results.get_interval_estimates({'a': y}, reps=5)):
      with pytest.raises(ValueError, match='non-finite'): f()


def _nan_scores(rng, shape):
  x = _scores(rng, shape)
  flat = x.reshape(-1)
  flat[rng.choice(flat.size, size=max(1, flat.size // 8), replace=False)] = np.nan
  flat[rng.choice(flat.size, size=max(1, flat.size // 16), replace=False)] = np.inf
  return x


@pytest.mark.parametrize('runs,envs', [(10, 4), (1024, 4)])
def test_kernels_rank_nan_like_numpy_sort(runs, envs):
  """Below the finite-only Python layer, the C entries rank a NaN above +inf (numpy's sort order): every sort slot is written and the
  results are those of the sort-based oracle, NaN where a NaN enters the trimmed window (scipy's trim_mean returns NaN for any NaN in
  the group instead; the Python layer refuses such input before either rule matters)."""
  lib, h, st = _lib.lib(), _lib.handle(), _lib.stream()
  rng, T, reps = np.random.default_rng(runs), 3, 29
  scores = _nan_scores(rng, (runs, envs, T))
  idx = iqm.stratified_indices(rng, reps, T, envs, runs)
  dx = torch.from_numpy(np.ascontiguousarray(scores.transpose(2, 1, 0))).cuda()
  nb = lib.il_bootstrap_iqm_workspace_bytes(T, envs, runs)
  ws = torch.full((nb, ), 0xFF, dtype=torch.uint8, device='cuda')  # stale workspace: any unwritten slot would show
  out = torch.empty(reps, T, dtype=torch.float64, device='cuda')
  _lib.check(lib.il_bootstrap_iqm(h, dx.data_ptr(), T, envs, runs, reps, 0, torch.from_numpy(idx).cuda().data_ptr(), out.data_ptr(), ws.data_ptr(), nb, st))
  ref = iqm.bootstrap_iqm(scores, idx)
  np.testing.assert_allclose(out.cpu().numpy(), ref, rtol=1e-13, atol=0, equal_nan=True)
  g = torch.from_numpy(np.ascontiguousarray(scores.reshape(-1, T).T)).cuda()
  m = torch.empty(T, dtype=torch.float64, device='cuda')
  _lib.check(lib.il_iqm(h, g.data_ptr(), T, runs * envs, m.data_ptr(), st))
  np.testing.assert_allclose(m.cpu().numpy(), iqm.trim_mean(scores.reshape(-1, T), axis=0), rtol=1e-13, atol=0, equal_nan=True)


def test_point_and_interval_cover_the_bootstrap_cap():
  """One point estimate and interval at N = IL_BOOTSTRAP_MAX_N (2048 runs x 4 envs): il_iqm takes as many values as the bootstrap."""
  assert _lib.IQM_MAX_N >= _lib.BOOTSTRAP_MAX_N
  scores = _scores(np.random.default_rng(2), (_lib.BOOTSTRAP_MAX_N // 4, 4, 2))
  points, cis = results.get_interval_estimates({'x': scores}, reps=7, seed=3)
  assert _rel(points['x'], [scipy.stats.trim_mean(scores[..., t].reshape(-1), 0.25) for t in range(2)]) <= 1e-13
  assert cis['x'].shape == (2, 2) and np.isfinite(cis['x']).all()


@pytest.mark.parametrize('runs,envs,T', [(10, 4, 3), (1024, 4, 1), (5, 3, 2)])
def test_device_draws_are_the_stated_philox_map(runs, envs, T):
  """The device resample is the stated function of (seed, rep, t, env): the oracle bootstrap over the host restatement of those draws
  (oracle.iqm.philox_indices) equals the device distribution; the restated indices are in range."""
  rng, reps, seed = np.random.default_rng(5), 37, 2**33 + 977
  scores = rng.random((runs, envs, T))  # continuous: a different resample changes the IQM
  idx = iqm.philox_indices(seed, reps, T, envs, runs)
  assert idx.min() >= 0 and idx.max() < runs
  dev = results.bootstrap_iqm(scores, reps, seed=seed).cpu().numpy()
  assert _rel(dev, iqm.bootstrap_iqm(scores, idx)) <= 1e-13


def test_device_draws_are_uniform_per_env():
  """Chi-square test of the per-env resample counts of 4000 reps x 10 runs at a fixed seed (reconstructed draws, proven equal to the
  device's by the test above): each env's counts over the 10 runs are uniform at the 0.1 % level."""
  idx = iqm.philox_indices(1234, 4000, 1, 4, 10)
  for e in range(4):
    counts = np.bincount(idx[:, 0, e].reshape(-1), minlength=10)
    assert scipy.stats.chisquare(counts).pvalue > 1e-3, (e, counts)


def test_same_seed_is_bitwise_identical():
  scores = np.random.default_rng(3).random((1024, 4, 3))
  for x, reps in ((scores[:10], 501), (scores, 33)):  # the warp kernel (N = 40) and the block kernel (N = 4096)
    a, b = results.bootstrap_iqm(x, reps, seed=9), results.bootstrap_iqm(x, reps, seed=9)
    assert torch.equal(a.view(torch.int64), b.view(torch.int64))
    assert not torch.equal(a, results.bootstrap_iqm(x, reps, seed=10))


@pytest.mark.parametrize('reps', [1, 2, 3, 40, 41, 50000])
def test_device_percentiles_equal_numpy(reps):
  rng = np.random.default_rng(reps)
  dist = np.concatenate([rng.random((reps, 3)) - 0.5, np.round(rng.random((reps, 2)) * 4) / 4, np.full((reps, 1), 0.7)], axis=1)  # signs, ties, constant
  dev = torch.from_numpy(dist).cuda()
  for conf in (0.95, 0.5, 0.999):
    lo, hi = results.interval_percentiles(conf)
    assert _rel(results.percentile_interval(dev, conf), np.percentile(dist, [lo, hi], axis=0)) <= 1e-14
    assert _rel(results.percentile_interval(dev, conf), iqm.percentile_interval(dist, conf)) <= 1e-14
  boot = results.bootstrap_iqm(rng.random((10, 4, 5)), reps, seed=1)
  assert _rel(results.percentile_interval(boot), np.percentile(boot.cpu().numpy(), [2.5, 97.5], axis=0)) <= 1e-14


def test_device_interval_agrees_with_host_bootstraps():
  """At 50 000 reps the device interval endpoints fall within 5 standard deviations of the mean of 8 independent host numpy bootstraps
  of the same data (the standard deviation taken from those 8, widened by sqrt(1 + 1/8) for the device run's own sampling noise)."""
  rng, reps, K = np.random.default_rng(11), 50000, 8
  scores = rng.random((10, 4, 3)) * np.array([1.0, 2.0, 0.5])
  host = np.stack([iqm.percentile_interval(iqm.bootstrap_iqm(scores, iqm.stratified_indices(np.random.default_rng(100 + k), reps, 3, 4, 10), chunk=4096)) for k in range(K)])
  mean, sd = host.mean(0), host.std(0, ddof=1)
  assert (sd > 0).all()
  _, ci = results.get_interval_estimates({'x': scores}, reps=reps, seed=4)
  assert (np.abs(ci['x'] - mean) <= 5 * sd * np.sqrt(1 + 1 / K)).all(), (ci['x'], mean, sd)


# ---- end to end ------------------------------------------------------------------------------------------------------------------
SMALL = ['algorithm=GAIL', 'steps=60', 'training.start=20', 'training.batch_size=32', 'evaluation.interval=30', 'evaluation.episodes=5', 'logging.interval=0',
         'imitation.trajectories=2', 'memory.size=200', 'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'imitation.discriminator.hidden_size=32']


def _run(args):
  res = subprocess.run([sys.executable, *args], cwd=ROOT, capture_output=True, text=True, timeout=1200)
  assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
  return res.stdout


@pytest.mark.parametrize('extra,seeds,runs', [(['seed=1,2,3'], '1,2,3', 3), (['replicas=2'], '1,2', 4)])
def test_seed_sweeps_summarised_by_the_script_match_the_oracle(tmp_path, extra, seeds, runs):
  out = tmp_path / 'outputs'
  for env in ('hopper', 'walker2d'):  # run_sweep names the sweeper directory after the first job's env: one command per env
    _run(['train.py', '-m', *SMALL, f'env={env}', *[e for e in extra if not e.startswith('seed=')], f'seed={seeds}', f'output_dir={out}'])
  reps, bseed = 3001, 17
  js = tmp_path / 'curves.json'
  stdout = _run(['scripts/print_seed_sweep_results.py', '--algorithms', 'GAIL', '--envs', 'hopper,walker2d', '--trajectories', '2', '--seeds', str(runs), '--reps', str(reps),
                 '--bootstrap-seed', str(bseed), '--path', str(out / '{algorithm}_{env}_sweeper' / '*'), '--out', str(js)])
  # oracle from the written files: per-run IQM over episodes, job-major then replica-minor
  per_env = []
  for env in ('hopper', 'walker2d'):
    (sweep, ) = glob.glob(str(out / f'GAIL_{env}_sweeper' / '*'))
    rows = []
    for j in sorted(os.listdir(sweep), key=int):
      m = torch.load(os.path.join(sweep, j, 'metrics.pth'), weights_only=False)
      r = np.asarray(m['test_returns_normalized'], dtype=np.float64)
      rows.extend((r[:, None, :] if r.ndim == 2 else r).transpose(1, 0, 2))
      steps = m['test_steps']
    per_env.append(iqm.trim_mean(np.stack(rows)))
  scores = np.stack(per_env, axis=1)
  assert scores.shape == (runs, 2, 2) and steps == [30, 60]
  point = iqm.aggregate_iqm(scores)
  ci = iqm.percentile_interval(iqm.bootstrap_iqm(scores, iqm.philox_indices(bseed, reps, 2, 2, runs)))
  cell = json.loads(js.read_text())['trajectories']['2']['GAIL']
  assert cell['steps'] == [30, 60]
  assert _rel(cell['iqm'], point) <= 1e-12 and _rel([cell['ci_low'], cell['ci_high']], ci) <= 1e-12
  assert 'IQM ± 1 C.I.' in stdout and '\nTrajectories: 2\n' in stdout
  line = re.search(r'^GAIL: (\S+) ± (\S+)$', stdout, flags=re.M)
  assert line.groups() == (f'{point[-1]:.2f}', f'{(ci[1, -1] - ci[0, -1]) / 2:.2f}'), stdout
