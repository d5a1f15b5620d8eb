"""The persistent, multi-stage wgmma engine (tc_gemm_kernel): k-block counts at every alignment of tile boundaries to
the three-stage rings, tile counts below, at and just above one wave of CTAs, schedule independence (every group of a
launch computes exactly what a launch of that group alone computes) and the fused epilogues at the 256-wide sizes."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _sm_count():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _gemm(mode, M, N, K, G, A, a_kmajor, B, b_kmajor, bias=None, act=-1, mask=None, mask_act=0, colsum=False):
  from il_b200 import _lib
  lib, h = _lib.lib(), _lib.handle()
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE[mode]))
  Cm = torch.full((G, M, N), float('nan'), device='cuda')
  cs = torch.full((G, M), float('nan'), device='cuda') if colsum else None
  try:
    _lib.check(lib.il_debug_gemm(h, M, N, K, G, A.data_ptr(), A.stride(0), A.stride(1), int(a_kmajor), B.data_ptr(), B.stride(0), B.stride(1), int(b_kmajor), Cm.data_ptr(),
                                 Cm.stride(0), N, _lib.ptr(bias), bias.stride(0) if bias is not None else 0, act, _lib.ptr(mask), mask.stride(0) if mask is not None else 0, N,
                                 mask_act, _lib.ptr(cs), M, _lib.stream()))
    torch.cuda.synchronize()
  finally:
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  return Cm, cs


def _operands(layout, G, M, N, K, seed):
  """Inputs of one layout and its float64 reference. fwd: relu(X W^T + b); dx: (dY W) * relu'(H); dw: dY^T X."""
  g = torch.Generator(device='cuda').manual_seed(seed)
  rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
  if layout == 'fwd':
    X, W, b = rn(G, M, K), rn(G, N, K) / 16, rn(G, N)
    kw = dict(A=X, a_kmajor=True, B=W, b_kmajor=True, bias=b, act=0)
    ref = lambda: torch.relu(torch.einsum('gmk,gnk->gmn', X.double(), W.double()) + b.double()[:, None, :])
  elif layout == 'dx':
    dY, W, H = rn(G, M, K), rn(G, K, N) / 16, rn(G, M, N)
    kw = dict(A=dY, a_kmajor=True, B=W, b_kmajor=False, mask=H)
    ref = lambda: torch.einsum('gmk,gkn->gmn', dY.double(), W.double()) * (H > 0).double()
  else:
    dY, X = rn(G, K, M), rn(G, K, N)
    kw = dict(A=dY, a_kmajor=False, B=X, b_kmajor=False, colsum=True)
    ref = lambda: torch.einsum('gkm,gkn->gmn', dY.double(), X.double())
  return kw, ref


def _check(layout, G, M, K, seed):
  N = 256
  kw, ref = _operands(layout, G, M, N, K, seed)
  got, cs = _gemm('tf32x3', M, N, K, G, **kw)
  assert not torch.isnan(got).any(), 'output element(s) never written'
  r = ref()
  err = (got.double() - r).abs().max().item() / r.abs().max().item()
  assert err < 8e-6, err
  if cs is not None:
    assert not torch.isnan(cs).any()
    np.testing.assert_allclose(cs.cpu().numpy(), kw['A'].double().sum(1).cpu().numpy(), rtol=1e-5, atol=1e-4)


@pytest.mark.parametrize('M', [128, 256, 384])
@pytest.mark.parametrize('K', [128, 144, 160, 256, 512])
@pytest.mark.parametrize('layout', ['fwd', 'dx', 'dw'])
def test_k_blocks_around_ring_depth(layout, K, M):
  """8, 9, 10, 16 and 32 k-blocks per tile (the engine takes K >= 128), so that tile boundaries fall at every position of
  the three-stage rings, with the k-block stream of a CTA running across two to three tiles."""
  G = -(-5 * _sm_count() // 2 // (M // 128))  # about 2.5 tiles per CTA
  _check(layout, G, M, K, seed=K + M)


@pytest.mark.parametrize('tiles', ['few', 'one_wave', 'one_wave_plus_one_group', 'many_waves'])
@pytest.mark.parametrize('M', [128, 256, 384])
@pytest.mark.parametrize('layout', ['fwd', 'dx', 'dw'])
def test_tile_counts_around_one_wave(layout, M, tiles):
  tm, sm = M // 128, _sm_count()
  G = {'few': 3, 'one_wave': sm // tm, 'one_wave_plus_one_group': sm // tm + 1, 'many_waves': 7 * sm // tm + 1}[tiles]
  _check(layout, G, M, 144, seed=G)


EPILOGUES = {  # (layout, epilogue): what il_debug_gemm reaches
    ('fwd', 'plain'): dict(),
    ('fwd', 'bias_relu'): dict(bias=True, act=0),
    ('fwd', 'bias_tanh'): dict(bias=True, act=1),  # generic epilogue
    ('dx', 'relu_mask'): dict(mask=True, mask_act=0),
    ('dx', 'tanh_mask'): dict(mask=True, mask_act=1),  # generic epilogue
    ('dw', 'plain_colsum'): dict(colsum=True),
}


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('layout,epi', list(EPILOGUES))
def test_groups_are_schedule_independent(layout, epi, mode):
  """One group replicated G times (group stride 0 on every input): each group of the many-wave launch must equal the
  G = 1 launch bit for bit, whichever CTA, wave and position in a CTA's tile sequence it ran at."""
  M, N, K = 256, 256, 256
  g = torch.Generator(device='cuda').manual_seed(7)
  rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
  a_km = layout != 'dw'
  b_km = layout == 'fwd'
  A = rn(1, M, K) if a_km else rn(1, K, M)
  B = (rn(1, N, K) if b_km else rn(1, K, N)) / 16
  e = EPILOGUES[(layout, epi)]
  bias = rn(1, N) if e.get('bias') else None
  mask = rn(1, M, N) if e.get('mask') else None
  kw = dict(act=e.get('act', -1), mask_act=e.get('mask_act', 0), colsum=e.get('colsum', False))
  one, cs1 = _gemm(mode, M, N, K, 1, A, a_km, B, b_km, bias=bias, mask=mask, **kw)
  G = 2 * _sm_count() + 3
  ex = lambda t: None if t is None else t.expand(G, *t.shape[1:])
  many, csG = _gemm(mode, M, N, K, G, ex(A), a_km, ex(B), b_km, bias=ex(bias), mask=ex(mask), **kw)
  assert not torch.isnan(one).any()
  assert torch.equal(many, one.expand_as(many)), 'a group differs from the single-group launch'
  if cs1 is not None: assert torch.equal(csG, cs1.expand_as(csG))


def test_fused_epilogues_are_schedule_independent():
  """The fused bias + ReLU + head (forward), sign-bit-masked dX and masked dX + input-gradient slice epilogues, with
  operands broadcast over the twin critics (group divisor 2), at default options: 80 replicas with identical inputs
  fill more than one wave of persistent CTAs. Every replica must equal replica 0 bit for bit, and replica 0 must match
  the reference fixture."""
  from conftest import load_golden
  from cuda_cases import run_cuda
  from il_b200 import _lib
  from oracle import cases
  lib, h = _lib.lib(), _lib.handle()
  inp = cases.make_inputs('sac_hopper')
  n = 80
  assert 2 * n > _sm_count(), 'the actor launches must span more than one wave'
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['tf32x3']))
  try:
    outs = run_cuda('sac_hopper', [inp] * n)
  finally:
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  gold = load_golden('sac_hopper')
  keys = {k.split('@')[0] for k in gold} & set(outs[0])
  bad = cases.compare(gold, outs[0], rtol=2e-4, atol=2e-5, keys=keys)
  assert not bad, '\n'.join(bad)
  for r in range(1, n):
    for k in outs[0]: assert np.array_equal(outs[r][k], outs[0][k]), f'replica {r} differs from replica 0 in {k}'
