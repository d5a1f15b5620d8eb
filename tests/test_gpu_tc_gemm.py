"""The wgmma (3xTF32 / TF32) dense-layer engine against the exact-fp32 FFMA engine and a float64 reference, on all
three operand layouts the MLP programs use (forward, input-gradient, weight-gradient) with their fused epilogues."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _gemm(mode, M, N, K, G, A, a_kmajor, B, b_kmajor, bias=None, act=-1, mask=None, colsum=False):
  import il_b200
  from il_b200 import _lib
  lib, h = _lib.lib(), _lib.handle()
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE[mode]))
  Cm = torch.full((G, M, N), float('nan'), device='cuda')
  cs = torch.full((G, M), float('nan'), device='cuda') if colsum else None
  lda, ldb = A.size(2), B.size(2)
  _lib.check(lib.il_debug_gemm(h, M, N, K, G, A.data_ptr(), A.stride(0), lda, int(a_kmajor), B.data_ptr(), B.stride(0), ldb, int(b_kmajor), Cm.data_ptr(), Cm.stride(0), N,
                               _lib.ptr(bias), N if bias is not None else 0, act, _lib.ptr(mask), mask.stride(0) if mask is not None else 0, N, 0, _lib.ptr(cs), M, _lib.stream()))
  torch.cuda.synchronize()
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  return Cm, cs


@pytest.mark.parametrize('layout', ['fwd', 'dx', 'dw'])
@pytest.mark.parametrize('mode,tol', [('tf32x3', 8e-6), ('tf32', 2e-3)])
def test_tc_gemm_matches_fp64(layout, mode, tol):
  torch.manual_seed(0)
  G, M, N, K = 5, 256, 256, 256
  X = torch.randn(G, M, K, device='cuda')
  W = torch.randn(G, N, K, device='cuda') / 16
  if layout == 'fwd':    # C = X W^T + b, relu
    bias = torch.randn(G, N, device='cuda')
    got, _ = _gemm(mode, M, N, K, G, X, True, W, True, bias=bias, act=0)
    ref = torch.relu(torch.einsum('gmk,gnk->gmn', X.double(), W.double()) + bias.double()[:, None, :])
  elif layout == 'dx':   # C = (dY W) * relu'(H)
    Wkn = torch.randn(G, K, N, device='cuda') / 16  # stored [K, N]
    Hm = torch.randn(G, M, N, device='cuda')
    got, _ = _gemm(mode, M, N, K, G, X, True, Wkn, False, mask=Hm)
    ref = torch.einsum('gmk,gkn->gmn', X.double(), Wkn.double()) * (Hm > 0).double()
  else:                  # C = dY^T X with column sums
    dY = torch.randn(G, K, M, device='cuda')  # stored [K = batch, M = out]
    Xb = torch.randn(G, K, N, device='cuda')  # stored [K = batch, N = in]
    got, cs = _gemm(mode, M, N, K, G, dY, False, Xb, False, colsum=True)
    ref = torch.einsum('gkm,gkn->gmn', dY.double(), Xb.double())
    np.testing.assert_allclose(cs.cpu().numpy(), dY.double().sum(1).cpu().numpy(), rtol=1e-5, atol=1e-4)
  assert not torch.isnan(got).any(), 'tile(s) never written'
  err = (got.double() - ref).abs().max().item() / ref.abs().max().item()
  print(layout, mode, 'max rel err', err)
  assert err < tol, err


def test_tc_gemm_many_groups_persistent():
  """More tiles than SMs: several waves of CTAs, every tile written."""
  torch.manual_seed(1)
  G, M, N, K = 200, 256, 256, 256
  X = torch.randn(G, M, K, device='cuda')
  W = torch.randn(G, N, K, device='cuda') / 16
  got, _ = _gemm('tf32x3', M, N, K, G, X, True, W, True)
  ref, _ = _gemm('fp32', M, N, K, G, X, True, W, True)
  assert not torch.isnan(got).any()
  err = (got - ref).abs().max().item() / ref.abs().max().item()
  assert err < 5e-6, err


@pytest.mark.parametrize('name', ['actor_hopper', 'sac_hopper'])
def test_golden_cases_with_tensor_core_engine(name, monkeypatch):
  """The reference fixtures at the real 256x256 sizes, hidden layers on the 3xTF32 tensor-core engine."""
  from conftest import load_golden
  from cuda_cases import run_cuda
  from il_b200 import _lib
  from oracle import cases
  lib, h = _lib.lib(), _lib.handle()
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['tf32x3']))
  try:
    out = run_cuda(name, [cases.make_inputs(name)])[0]
  finally:
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  g = load_golden(name)
  keys = {k.split('@')[0] for k in g} & set(out)
  bad = cases.compare(g, out, rtol=2e-4, atol=2e-5, keys=keys)
  assert not bad, '\n'.join(bad)


def test_fused_first_layer_is_schedule_independent():
  """The tensor-core engine computes the first MLP layer (K0 = 12 / 15 columns) chunk by chunk into the
  operand tile of the second. 80 replicas with IDENTICAL inputs fill more than one wave of CTAs (per-tile W1 / input
  staging): every replica must reproduce replica 0 bit for bit, and replica 0 must match the reference fixture."""
  from conftest import load_golden
  from cuda_cases import run_cuda
  from il_b200 import _lib
  from oracle import cases
  lib, h = _lib.lib(), _lib.handle()
  inp = cases.make_inputs('sac_hopper')
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['tf32x3']))
  _lib.set_option('tc_fuse_l1', 1)  # off by default; kept correct for A/B
  try:
    outs = run_cuda('sac_hopper', [inp] * 80)
  finally:
    _lib.set_option('tc_fuse_l1', 0)
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  g = load_golden('sac_hopper')
  keys = {k.split('@')[0] for k in g} & set(outs[0])
  bad = cases.compare(g, outs[0], rtol=2e-4, atol=2e-5, keys=keys)
  assert not bad, '\n'.join(bad)
  for r in (1, 37, 73, 74, 79):
    for k in keys: assert np.array_equal(outs[r][k], outs[0][k]), f'replica {r} differs from replica 0 in {k}'


def test_sign_bit_masks_equal_fp32_masks():
  """ReLU derivative masks as sign-bit words (written by the first-layer kernel and the fused-head wgmma epilogue, read by the masked dX launches)
  against fp32 activations as masks: the same `> 0` predicate on the same values, so one SAC update of the 256-wide fixture is bit-identical
  (option 1); with the input-gradient slice fused into the masked dX launch (option 2, the default) only the summation order of that thin product
  changes."""
  from cuda_cases import run_cuda
  from il_b200 import _lib
  from oracle import cases
  lib, h = _lib.lib(), _lib.handle()
  inp = cases.make_inputs('sac_hopper')
  outs = {}
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['tf32x3']))
  try:
    for level in (0, 1, 2):
      _lib.set_option('mask_bits', level)
      outs[level] = run_cuda('sac_hopper', [inp])[0]
  finally:
    _lib.set_option('mask_bits', 2)
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  for k in outs[0]:
    assert np.array_equal(outs[0][k], outs[1][k]), k
    np.testing.assert_allclose(outs[2][k], outs[0][k], rtol=2e-5, atol=2e-6, err_msg=k)
