"""The warp-specialised wgmma engine (tc_gemm_kernel): a producer warpgroup hands hi/lo stages to two consumer warpgroups
through full / empty mbarrier pairs whose phase bits flip every three k-blocks, and the k-block stream of a CTA runs on
across its tiles. These tests put tile boundaries at every phase of the stage ring over many tiles per CTA, give CTAs
unequal tile counts, and check every epilogue (the fused first layer with and without its hidden store included) against
float64 and for bitwise independence of the schedule."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

N = 256


def _sm_count():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _grid(M):
  """The persistent launch's grid: one CTA per SM, rounded down to whole groups of M / 128 tiles."""
  tm, sm = M // 128, _sm_count()
  return sm // tm * tm if sm >= tm else sm


def _gemm(mode, M, K, G, A, a_kmajor, B, b_kmajor, bias=None, act=-1, mask=None, mask_act=0):
  from il_b200 import _lib
  lib, h = _lib.lib(), _lib.handle()
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE[mode]))
  Cm = torch.full((G, M, N), float('nan'), device='cuda')
  try:
    _lib.check(lib.il_debug_gemm(h, M, N, K, G, A.data_ptr(), A.stride(0), A.stride(1), int(a_kmajor), B.data_ptr(), B.stride(0), B.stride(1), int(b_kmajor), Cm.data_ptr(),
                                 Cm.stride(0), N, _lib.ptr(bias), bias.stride(0) if bias is not None else 0, act, _lib.ptr(mask), mask.stride(0) if mask is not None else 0, N,
                                 mask_act, None, M, _lib.stream()))
    torch.cuda.synchronize()
  finally:
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  return Cm


EPILOGUES = {  # name: (layout, il_debug_gemm epilogue arguments, float64 epilogue of the product P given bias b and mask H)
    'plain': ('fwd', dict(), lambda P, b, H: P),
    'bias_relu': ('fwd', dict(bias=True, act=0), lambda P, b, H: torch.relu(P + b[:, None, :])),
    'bias_tanh': ('fwd', dict(bias=True, act=1), lambda P, b, H: torch.tanh(P + b[:, None, :])),
    'relu_mask': ('dx', dict(mask=True, mask_act=0), lambda P, b, H: P * (H > 0)),
    'tanh_mask': ('dx', dict(mask=True, mask_act=1), lambda P, b, H: P * (1 - H * H)),
    'plain_dw': ('dw', dict(), lambda P, b, H: P),
}


def _case(epi, G, M, K, seed):
  layout, e, f = EPILOGUES[epi]
  g = torch.Generator(device='cuda').manual_seed(seed)
  rn = lambda *s: torch.randn(*s, device='cuda', generator=g)
  a_km, b_km = layout != 'dw', layout == 'fwd'
  A = rn(G, M, K) if a_km else rn(G, K, M)
  B = (rn(G, N, K) if b_km else rn(G, K, N)) / 16
  bias = rn(G, N) if e.get('bias') else None
  mask = (torch.tanh(rn(G, M, N)) if e.get('mask_act') == 1 else rn(G, M, N)) if e.get('mask') else None
  kw = dict(A=A, a_kmajor=a_km, B=B, b_kmajor=b_km, bias=bias, act=e.get('act', -1), mask=mask, mask_act=e.get('mask_act', 0))

  def ref():
    """The float64 output and the scale of its pre-activation values, which the engine's rounding error is relative to."""
    Ad = A.double() if a_km else A.double().transpose(1, 2)
    Bd = B.double().transpose(1, 2) if b_km else B.double()
    P = torch.bmm(Ad, Bd)
    b = None if bias is None else bias.double()
    scale = (P if b is None else P + b[:, None, :]).abs().max().item()
    return f(P, b, None if mask is None else mask.double()), scale
  return kw, ref


def _check(epi, mode, G, M, K, seed):
  kw, ref = _case(epi, G, M, K, seed)
  got = _gemm(mode, M, K, G, **kw)
  assert not torch.isnan(got).any(), 'output element(s) never written'
  r, scale = ref()
  err = (got.double() - r).abs().max().item() / scale
  assert err < {'tf32x3': 8e-6, 'tf32': 2e-3}[mode], err


@pytest.mark.parametrize('K', [128, 144, 160, 176, 512])
@pytest.mark.parametrize('epi', ['bias_relu', 'relu_mask', 'plain_dw'])
def test_stage_phases_over_many_tiles(epi, K):
  """8, 9, 10, 11 and 32 k-blocks per tile (k-block counts of every residue modulo the three stages) with about seven
  tiles per CTA, so each stage's full / empty phase bits wrap many times and every tile starts at each stage."""
  M = 256
  G = 7 * _grid(M) // 2 + 1
  _check(epi, 'tf32x3', G, M, K, seed=K)


@pytest.mark.parametrize('M', [128, 256, 384])
@pytest.mark.parametrize('epi', ['bias_relu', 'relu_mask', 'plain_dw'])
def test_unequal_tile_counts(epi, M):
  """G * M / 128 tiles just above a multiple of the grid: the first CTAs run one tile more than the rest and finish
  their k-block stream later, while the others' producers have already left."""
  tm = M // 128
  G = 2 * _grid(M) // tm + 1
  _check(epi, 'tf32x3', G, M, 144, seed=M)


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('epi', list(EPILOGUES))
def test_every_epilogue_against_float64(epi, mode):
  _check(epi, mode, 3 * _grid(256) // 2 + 1, 256, 256, seed=len(epi))


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('epi', list(EPILOGUES))
def test_replicated_group_is_schedule_independent(epi, mode):
  """One group (K = 176: 11 k-blocks, so consecutive tiles of a CTA start at different stages and phases) replicated
  over five waves with group stride 0: every group equals the single-group launch bit for bit."""
  M, K = 256, 176
  kw, _ = _case(epi, 1, M, K, seed=3)
  one = _gemm(mode, M, K, 1, **kw)
  G = 5 * _grid(M) // 2 + 1
  ex = lambda t: t.expand(G, *t.shape[1:]) if isinstance(t, torch.Tensor) else t
  many = _gemm(mode, M, K, G, **{k: ex(v) for k, v in kw.items()})
  assert not torch.isnan(one).any()
  assert torch.equal(many, one.expand_as(many)), 'a group differs from the single-group launch'


def _actor_params(S, A, H, R, seed):
  g = torch.Generator().manual_seed(seed)
  dims = [S, H, H, 2 * A]
  one = [t for l in range(3) for t in (torch.randn(dims[l + 1], dims[l], generator=g, dtype=torch.float64) * (2 / dims[l]) ** 0.5,
                                       0.1 * torch.randn(dims[l + 1], generator=g, dtype=torch.float64))]
  return [[t.float().double() for t in one] for _ in range(R)]


@pytest.mark.parametrize('fuse', [0, 1])
def test_fused_head_forward_without_hidden_store(fuse):
  """Actor forward at H = 256 and 256 rows per replica: the fused bias + ReLU + head epilogue, with the first layer
  computed inside the launch (fuse = 1) or not, and no hidden store (no backward follows). 150 replicas of one parameter
  set and one state batch give CTAs one and two tiles; every replica must equal replica 0 bit for bit, and replica 0
  must match float64 as closely as the same arithmetic in fp32 does."""
  import il_b200
  from il_b200 import _lib
  from oracle import port
  S, A, H, n, R = 11, 3, 256, 256, 150
  params = _actor_params(S, A, H, R, seed=5)
  states = torch.randn(1, n, S, generator=torch.Generator().manual_seed(6)).double()
  actor = il_b200.SoftActor(S, A, SimpleNamespace(hidden_size=H, depth=2, activation='relu'), replicas=R)
  for r, ps in enumerate(params): actor.mlp.load_params(r, 0, [t.float() for t in ps])
  _lib.check(_lib.lib().il_set_gemm_mode(_lib.handle(), _lib.GEMM_MODE['tf32x3']))
  _lib.set_option('tc_fuse_l1', fuse)
  try:
    out = actor._run(states.float().expand(R, n, S).contiguous().cuda(), want=('mean', 'log_std'))
    torch.cuda.synchronize()
  finally:
    _lib.set_option('tc_fuse_l1', 0)
    _lib.check(_lib.lib().il_set_gemm_mode(_lib.handle(), _lib.GEMM_MODE['fp32']))
  for i, key in enumerate(('mean', 'log_std')):
    got = out[key].cpu().numpy()
    for r in range(1, R): assert np.array_equal(got[r], got[0]), f'{key}: replica {r} differs from replica 0'
    f64 = port.actor_mean_logstd(params[0], states[0])[i].numpy()
    f32 = port.actor_mean_logstd([t.float() for t in params[0]], states[0].float())[i].numpy()
    err, cpu_err, scale = np.abs(got[0] - f64).max(), np.abs(f32 - f64).max(), np.abs(f64).max()
    assert err <= 8 * cpu_err + 1e-6 * scale, f'{key}: max |cuda - f64| = {err:.3e}, max |cpu fp32 - f64| = {cpu_err:.3e}'


def test_fused_first_layer_with_hidden_store_over_many_waves():
  """One SAC update of the 256-wide fixture with the first layer fused into the wgmma launch, so its hidden activation
  is stored for the backward pass: 300 identical replicas (several waves, CTAs with unequal tile counts) must each equal
  replica 0 bit for bit, and replica 0 must match the reference fixture."""
  from conftest import load_golden
  from cuda_cases import run_cuda
  from il_b200 import _lib
  from oracle import cases
  lib, h = _lib.lib(), _lib.handle()
  inp = cases.make_inputs('sac_hopper')
  n = 300
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['tf32x3']))
  _lib.set_option('tc_fuse_l1', 1)
  try:
    outs = run_cuda('sac_hopper', [inp] * n)
  finally:
    _lib.set_option('tc_fuse_l1', 0)
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  gold = load_golden('sac_hopper')
  keys = {k.split('@')[0] for k in gold} & set(outs[0])
  bad = cases.compare(gold, outs[0], rtol=2e-4, atol=2e-5, keys=keys)
  assert not bad, '\n'.join(bad)
  for r in range(1, n):
    for k in outs[0]: assert np.array_equal(outs[r][k], outs[0][k]), f'replica {r} differs from replica 0 in {k}'
