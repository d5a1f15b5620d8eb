"""TEST INFRASTRUCTURE ONLY — a float64 numpy restatement of the GP posterior, expected improvement and greedy kriging-believer selection
that csrc/gp.cu computes (il_gp_posterior, il_gp_select). tests/test_hpo_cpu.py checks it against scikit-learn's GaussianProcessRegressor;
tests/test_gpu_hpo.py checks the kernels against it. The product never imports it."""
import numpy as np
from scipy.linalg import solve_triangular
from scipy.stats import norm


def matern52(A, B, ls, s2):
  r2 = (((A[:, None, :] - B[None, :, :]) / ls)**2).sum(-1)
  r = np.sqrt(r2)
  return s2 * (1.0 + np.sqrt(5.0) * r + (5.0 / 3.0) * r2) * np.exp(-np.sqrt(5.0) * r)


def posterior(X, y, C, ls, s2, noise):
  """(mu, var, V, L, alpha): the latent posterior mean and variance of candidates C given y at X, V = L^-1 K*^T."""
  K = matern52(X, X, ls, s2) + noise * np.eye(len(X))
  L = np.linalg.cholesky(K)
  alpha = solve_triangular(L.T, solve_triangular(L, y, lower=True), lower=False)
  Ks = matern52(C, X, ls, s2)
  V = solve_triangular(L, Ks.T, lower=True)
  return Ks @ alpha, s2 - (V * V).sum(0), V, L, alpha


def expected_improvement(mu, var, fstar):
  s = np.sqrt(np.maximum(var, 0.0))
  imp = mu - fstar
  with np.errstate(divide='ignore', invalid='ignore'):
    z = imp / s
    ei = imp * norm.cdf(z) + s * norm.pdf(z)
  return np.where(s > 0, ei, np.maximum(imp, 0.0))


def select(C, mu, var, V, ls, s2, noise, fstar, q, group=None, max_groups=0):
  """(picks, ei, var after the picks): q greedy EI picks with the kriging believer, as il_gp_select states them (first index on ties;
  picked and non-admitted candidates masked; -1 once none is admissible)."""
  var, V = var.copy(), [row for row in V]
  picked = np.zeros(len(C), bool)
  admitted, picks, eis = [], [], []
  for _ in range(q):
    ok = ~picked
    if max_groups > 0 and len(admitted) >= max_groups: ok &= np.isin(group, admitted)
    if not ok.any():
      picks.append(-1), eis.append(np.nan)
      continue
    ei = np.where(ok, expected_improvement(mu, var, fstar), -np.inf)
    w = int(np.argmax(ei))
    picks.append(w), eis.append(ei[w])
    picked[w] = True
    if max_groups > 0 and group[w] not in admitted: admitted.append(group[w])
    Vm = np.array(V)
    c = matern52(C, C[w:w + 1], ls, s2)[:, 0] - Vm.T @ Vm[:, w]
    den = var[w] + noise
    var = var - c * c / den
    V.append(c / np.sqrt(den))
    fstar = max(fstar, mu[w])
  return np.array(picks), np.array(eis), var
