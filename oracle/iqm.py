"""float64 numpy restatement of the seed-sweep statistics of scripts/print_plot_seed_sweep_results.py (scipy's trim_mean, rliable's
stratified-bootstrap IQM and the percentile interval), with the resample indices as an input. Used by the tests and as the host timing
of scripts/iqm_bench.py; the product (imitation-learning_b200/results.py) does not import it."""
import numpy as np


def trim_mean(x, axis=-1):
  """scipy.stats.trim_mean(x, 0.25, axis): sort, drop floor(n / 4) values at each end, average the rest."""
  x = np.sort(np.asarray(x, dtype=np.float64), axis=axis)
  n = x.shape[axis]
  lc = int(0.25 * n)
  return np.mean(np.take(x, np.arange(lc, n - lc), axis=axis), axis=axis)


def aggregate_iqm(scores):
  """rliable's metrics.aggregate_iqm at every t: scores [runs, envs, T] -> [T]."""
  s = np.asarray(scores, dtype=np.float64)
  return trim_mean(s.reshape(-1, s.shape[-1]), axis=0)


def stratified_indices(rng: np.random.Generator, reps: int, T: int, envs: int, runs: int):
  """Host resample indices [reps, T, envs, runs]: runs drawn with replacement, independently per (rep, t, env)."""
  return rng.integers(0, runs, size=(reps, T, envs, runs), dtype=np.int32)


def _philox4x32_10(c0, c1, c2, c3, k0, k1):
  M0, M1, W0, W1, U32 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), np.uint64(0x9E3779B9), np.uint64(0xBB67AE85), np.uint64(0xFFFFFFFF)
  k0, k1 = np.uint64(k0), np.uint64(k1)
  for _ in range(10):
    p0, p1 = M0 * c0, M1 * c2
    c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & U32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & U32
    k0, k1 = (k0 + W0) & U32, (k1 + W1) & U32
  return c0, c1, c2, c3


def philox_indices(seed: int, reps: int, T: int, envs: int, runs: int):
  """The device draws of il_bootstrap_iqm restated, [reps, T, envs, runs]: draw k of (rep, t, e) is lane k % 4 of Philox4x32-10 at counter
  (k / 4, e, t, rep) under key (seed low word, seed high word), mapped to a run by (u * runs) >> 32."""
  rep, t, e, k = np.meshgrid(*(np.arange(n, dtype=np.uint64) for n in (reps, T, envs, runs)), indexing='ij')
  lanes = _philox4x32_10(k // np.uint64(4), e, t, rep, seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
  u = np.choose((k % np.uint64(4)).astype(np.int64), lanes)
  return ((u * np.uint64(runs)) >> np.uint64(32)).astype(np.int32)


def bootstrap_iqm(scores, indices, chunk: int = 1024):
  """[reps, T]: the IQM of each resample. scores [runs, envs, T]; indices [reps, T, envs, runs] take run indices[rep, t, e, k] of env e
  at point t."""
  x = np.asarray(scores, dtype=np.float64).transpose(2, 1, 0)  # [T, envs, runs]
  idx = np.asarray(indices)
  reps, T, envs, runs = idx.shape
  out = np.empty((reps, T))
  for r0 in range(0, reps, chunk):
    g = np.take_along_axis(x[None], idx[r0:r0 + chunk], axis=-1)
    out[r0:r0 + chunk] = trim_mean(g.reshape(g.shape[0], T, envs * runs), axis=-1)
  return out


def percentile_interval(dist, confidence=0.95):
  """[2, T]: the two-sided percentile interval of dist [reps, T] (numpy's default linear interpolation)."""
  alpha = (1.0 - confidence) / 2.0
  return np.percentile(np.asarray(dist, dtype=np.float64), [100.0 * alpha, 100.0 * (1.0 - alpha)], axis=0)
