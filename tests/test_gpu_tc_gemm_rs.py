"""The wgmma engine's A operand from registers (tc_gemm_kernel): the producer copies raw A into a ring of six slots
guarded by the hi/lo stages' full / empty barriers, and each consumer warpgroup loads its A fragments from the slot and
splits them in registers, alternating two fragment sets from one k-block of a tile to the next. These tests put tile
boundaries at every phase of the A ring (k-block counts of every residue modulo 6), with tiles ending on either fragment
set (odd and even counts), over many tiles per CTA, give CTAs unequal tile counts, and run both A layouts ([rows, K]:
SWIZZLE_64B; [K, rows]: padded k-rows) in tf32x3 and tf32 with every epilogue, against float64 and for bitwise
independence of the schedule. Every case first checks that its shape is routed to tc_gemm_kernel (the dispatcher sends
K < 128 to the FFMA engine): its output must not be bitwise the FFMA engine's.
"""
import pytest
import torch

from test_gpu_tc_gemm_ws import EPILOGUES, _case, _check, _gemm, _grid

pytestmark = pytest.mark.gpu

A_LAYOUTS = ['bias_relu', 'relu_mask', 'plain_dw']  # A [rows, K] with B [rows, K] and B [K, rows]; A [K, rows]


def _assert_tc_route(epi, mode, M, K):
  """One group of the case's shape, layouts and epilogue runs on the wgmma engine (the route depends on shape, layouts
  and gemm mode, not on G). The FFMA routes compute bitwise the same in every gemm mode, so an output that differs from
  the fp32 mode's comes from tc_gemm_kernel."""
  kw, _ = _case(epi, 1, M, K, seed=0)
  tc, ffma = _gemm(mode, M, K, 1, **kw), _gemm('fp32', M, K, 1, **kw)
  assert not torch.isnan(tc).any()
  assert not torch.equal(tc, ffma), f'M={M} K={K} {epi} {mode}: bitwise the FFMA engine output, so not the wgmma engine'


def _check_tc(epi, mode, G, M, K, seed):
  _assert_tc_route(epi, mode, M, K)
  _check(epi, mode, G, M, K, seed)


@pytest.mark.parametrize('K', [128, 144, 160, 176, 208, 288])
@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('epi', A_LAYOUTS)
def test_a_ring_phases_over_many_tiles(epi, mode, K):
  """8, 9, 10, 11, 13 and 18 k-blocks per tile (residues 2, 3, 4, 5, 1 and 0 modulo the six A slots, even and odd) with
  about seven tiles per CTA, so each slot is refilled many times, tiles start at every slot, and tiles end on either
  fragment set."""
  M = 256
  G = 7 * _grid(M) // 2 + 1
  _check_tc(epi, mode, G, M, K, seed=K + 1)


@pytest.mark.parametrize('M', [128, 384])
@pytest.mark.parametrize('epi', A_LAYOUTS)
def test_a_ring_unequal_tile_counts(epi, M):
  """An odd k-block count (13) and G * M / 128 tiles just above a multiple of the grid: the first CTAs run one tile more
  than the rest and leave the A ring at another phase."""
  tm = M // 128
  G = 3 * _grid(M) // tm + 1
  _check_tc(epi, 'tf32x3', G, M, 208, seed=M + 1)


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('epi', list(EPILOGUES))
def test_every_epilogue_with_odd_k_blocks(epi, mode):
  _check_tc(epi, mode, 3 * _grid(256) // 2 + 1, 256, 208, seed=len(epi) + 7)


@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('epi', A_LAYOUTS)
def test_replicated_group_is_schedule_independent(epi, mode):
  """One group (K = 208: 13 k-blocks, so consecutive tiles of a CTA start at different A slots and stages)
  replicated over five waves with group stride 0: every group equals the single-group launch bit for bit."""
  M, K = 256, 208
  _assert_tc_route(epi, mode, M, K)
  kw, _ = _case(epi, 1, M, K, seed=11)
  one = _gemm(mode, M, K, 1, **kw)
  G = 5 * _grid(M) // 2 + 1
  ex = lambda t: t.expand(G, *t.shape[1:]) if isinstance(t, torch.Tensor) else t
  many = _gemm(mode, M, K, G, **{k: ex(v) for k, v in kw.items()})
  assert not torch.isnan(one).any()
  assert torch.equal(many, one.expand_as(many)), 'a group differs from the single-group launch'
