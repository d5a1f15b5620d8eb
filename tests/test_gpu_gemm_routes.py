"""Every route of the fp32 GEMM dispatcher (`launch_gemm`, csrc/gemm.cu) and the MLP-level kernels next to it, against float64.

Each row of the route table names the kernel instance `launch_gemm` must pick for one problem (shape, operand layouts, leading dimensions,
pointer offset, epilogue, A/B option switches), sitting on one side of a selection condition or a tile edge. For every row the test checks
- the route: the named kernel is the only kernel of the call (read from a CUDA-activity `torch.profiler` trace);
- the values: float64 reference with an elementwise bound of 2 K 2^-24 (|A| |B|)_ij (+ the bias and activation terms below): missing one k
  term, one column or one row tail exceeds it;
- coverage and bounds: every output element is written and every element around it (one extra group, row and 4+ columns) is untouched;
- the gemm mode: in `tf32x3` mode (the dense-layer wgmma engine never takes these shapes) the same kernel gives bitwise the same output.
"""
import re
import time
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                     # unit roundoff of fp32
SENTINEL = 1234.5                  # guard-band value around every output
OPTION_DEFAULTS = {'wide_tn': 1, 'first_layer_fast': 2, 'thin_hoist': 1, 'head_fused': 1}
ACT = {None: -1, 'relu': 0, 'tanh': 1, 'sigmoid': 2}
_NON_KERNEL = ('Memcpy', 'Memset')
DEV = 'cuda'


# ---- kernel names from a CUDA-activity trace -------------------------------------------------------------------------------------------
def _kernel_id(name):
  """'void (anonymous namespace)::row_dot_kernel<2, 4>(GemmArgs)' -> 'row_dot_kernel<2, 4>'."""
  s = name.replace('(anonymous namespace)::', '')
  if s.startswith('void '): s = s[5:]
  s = s.split('(', 1)[0].rsplit('::', 1)[-1]
  return re.sub(r'\s*,\s*', ', ', s.strip())


def kernels_of(fn, attempts=1, setup=None):
  """The kernels `fn` ran on the GPU, in start order, as base name + template arguments. A trace that holds no kernel event at all is taken
  again, after `setup` (outside the trace) and a pause, up to `attempts` traces in all: now and then a trace misses a kernel launched and
  finished well inside it."""
  from torch.autograd import DeviceType
  from torch.profiler import ProfilerActivity, profile
  for attempt in range(attempts):
    if setup: setup()
    torch.cuda.synchronize()
    time.sleep(0.25 * attempt)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      time.sleep(1e-3)
      fn()
      torch.cuda.synchronize()
      time.sleep(1e-3)
    evs = list(prof.profiler.kineto_results.events())
    kern = [e for e in evs if e.device_type() == DeviceType.CUDA and not e.name().startswith(_NON_KERNEL)]
    names = [_kernel_id(e.name()) for e in sorted(kern, key=lambda e: e.start_ns())]
    if names: return names
  raise AssertionError(f'{attempts} CUDA-activity trace(s) hold no kernel events: the route cannot be checked; the last one holds '
                       f'{[(e.name()[:60], str(e.device_type())) for e in evs[:8]]}')


def set_options(**opts):
  from il_b200 import _lib
  for k, v in opts.items(): _lib.set_option(k, v)


def restore_options():
  from il_b200 import _lib
  set_options(**OPTION_DEFAULTS)
  _lib.check(_lib.lib().il_set_gemm_mode(_lib.handle(), _lib.GEMM_MODE['fp32']))


# ---- the route table ------------------------------------------------------------------------------------------------------------------
def grouped(bm, bn, a, b):
  tm, tn = {(16, 128): (1, 8), (128, 16): (8, 1), (32, 128): (2, 8), (128, 128): (8, 8)}[(bm, bn)]
  return f'gemm_grouped_kernel<{bm}, {bn}, 16, {tm}, {tn}, {str(a == "k").lower()}, {str(b == "k").lower()}>'


def row_dot(K, N): return 'row_dot_kernel<2, 4>' if K <= 256 and N <= 4 else ('row_dot_kernel<2, 8>' if K <= 256 else 'row_dot_kernel<4, 8>')


def thin_k(b, hoist): return f'gemm_thin_k_kernel<{str(b == "k").lower()}, {str(hoist).lower()}>'


WIDE_TN, FIRST_RELU = 'wide_tn_kernel', 'first_layer_relu_kernel'
STREAM = {True: 'gemm_stream_tn_kernel<true>', False: 'gemm_stream_tn_kernel<false>'}


def spec(kernel, M, N, K, G=2, a='k', b='m', lda=None, ldb=None, a_off=0, bias=False, act=None, mask=None, colsum=False, opts=None):
  """One problem and the kernel that must run it. a / b: 'k' = k-major ([M, K] / [N, K]), 'm' = the other layout ([K, M] / [K, N]); a_off: A starts
  that many floats into its buffer; mask: the activation whose derivative (through its output) multiplies the product; opts: A/B option switches.
  Returns (problem, test id)."""
  lda = lda or (K if a == 'k' else M)
  ldb = ldb or (K if b == 'k' else N)
  tags = [f'M{M}', f'N{N}', f'K{K}', f'G{G}', a + b]
  if lda != (K if a == 'k' else M): tags.append(f'lda{lda}')
  if ldb != (K if b == 'k' else N): tags.append(f'ldb{ldb}')
  if a_off: tags.append(f'aoff{a_off}')
  if bias: tags.append('bias')
  if act: tags.append(act)
  if mask: tags.append(f'mask-{mask}')
  if colsum: tags.append('colsum')
  for k, v in (opts or {}).items(): tags.append(f'{k}{v}')
  short = kernel.replace('gemm_', '').replace('_kernel', '').replace(', ', '.').replace('<', '[').replace('>', ']').replace('true', 't').replace('false', 'f')
  return (dict(kernel=kernel, M=M, N=N, K=K, G=G, a=a, b=b, lda=lda, ldb=ldb, a_off=a_off, bias=bias, act=act, mask=mask, colsum=colsum, opts=opts or {}),
          short + '-' + '-'.join(tags))


def case(*args, **kw):
  p, name = spec(*args, **kw)
  return pytest.param(p, id=name)


def _route_table():
  t = []
  # row_dot_kernel: A k-major, B [K, N], N <= 8, K % 128 == 0, K <= 512, M >= 32, plain; 256 rows per CTA
  Ms = (32, 255, 256, 257)
  for i, K in enumerate((128, 256, 384, 512)):
    for j, N in enumerate((1, 3, 4, 5, 8)):
      for M in (Ms[(i + j) % 4], Ms[(i + j + 2) % 4]):
        t.append(case(row_dot(K, N), M, N, K, lda=K + 4))
  t.append(case(grouped(128, 16, 'k', 'm'), 257, 5, 200))              # K % 128 != 0
  t.append(case(grouped(128, 16, 'k', 'm'), 256, 4, 256, a_off=1))     # A not 16-byte aligned
  t.append(case(grouped(128, 16, 'k', 'm'), 256, 8, 512, lda=516, opts={'wide_tn': 0}))
  # wide_tn_kernel: both [K, *], N <= 16, M >= 64, M % 4 == 0, 64 <= K <= 1024, no epilogue but colsum
  Ms = (64, 68, 260)
  for i, N in enumerate((1, 3, 15, 16)):
    for j, K in enumerate((64, 65, 1023, 1024)):
      for cs in (False, True):
        M = Ms[(i + j + cs) % 3]
        t.append(case(WIDE_TN, M, N, K, a='m', b='m', lda=M + 4 * (j % 2), ldb=N + (j // 2), colsum=cs))
  t.append(case(STREAM[True], 66, 16, 1024, a='m', b='m', colsum=True))   # M % 4 != 0
  t.append(case(STREAM[True], 66, 3, 65, a='m', b='m'))
  t.append(case(STREAM[True], 64, 16, 1024, a='m', b='m', colsum=True, opts={'wide_tn': 0}))
  t.append(case(STREAM[True], 1000, 5, 300, a='m', b='m', colsum=True, opts={'wide_tn': 0}))
  # gemm_stream_tn_kernel<false>: both [K, *], M <= 16 < 64 <= N, 64 <= K <= 1024 (the last-layer weight gradient, colsum = head bias gradient)
  for i, M in enumerate((1, 6, 16)):
    for j, N in enumerate((64, 256, 260)):
      t.append(case(STREAM[False], M, N, (64, 71, 1024)[(i + j) % 3], a='m', b='m', colsum=True))
  t.append(case(STREAM[False], 16, 260, 1024, a='m', b='m', ldb=263, colsum=True))
  t.append(case(STREAM[False], 3, 100, 64, a='m', b='m'))
  t.append(case(grouped(16, 128, 'm', 'm'), 6, 64, 1025, a='m', b='m', colsum=True))   # K > 1024
  # first_layer_reg_kernel<K>: K in {11, 12, 14, 15, 16}, N == 256, M % 32 == 0, bias + ReLU, ldb == K
  for K in (11, 12, 14, 15, 16):
    for M in (32, 288):
      t.append(case(f'first_layer_reg_kernel<{K}, false>', M, 256, K, a='k', b='k', lda=K + (M == 288), bias=True, act='relu'))
  # first_layer_relu_kernel: K <= 16, N % 256 == 0, M % 32 == 0, bias + ReLU
  t.append(case(FIRST_RELU, 64, 512, 3, a='k', b='k', bias=True, act='relu'))
  t.append(case(FIRST_RELU, 288, 512, 13, a='k', b='k', lda=15, bias=True, act='relu'))
  t.append(case(FIRST_RELU, 160, 256, 12, a='k', b='k', bias=True, act='relu', opts={'first_layer_fast': 1}))
  t.append(case(FIRST_RELU, 96, 256, 12, a='k', b='k', ldb=16, bias=True, act='relu'))   # ldb != K: not the register-resident kernel
  t.append(case(grouped(16, 128, 'k', 'k'), 16, 256, 12, a='k', b='k', bias=True, act='relu'))
  t.append(case(thin_k('k', False), 288, 256, 12, a='k', b='k', bias=True, act='relu', opts={'first_layer_fast': 0}))
  # gemm_thin_k_kernel<B_KMAJOR, HOIST>: A k-major, K <= 32, N >= 64, N % 4 == 0, M > 16
  Ks, Ns, Ms, acts = (1, 6, 18, 31, 32), (64, 68, 300), (17, 129, 1000), ('relu', 'tanh', 'sigmoid')
  for b in ('k', 'm'):
    for i, K in enumerate(Ks):
      t.append(case(thin_k(b, False), Ms[i % 3], Ns[(i + 1) % 3], K, b=b, lda=K + 3))
      t.append(case(thin_k(b, False), Ms[(i + 1) % 3], Ns[i % 3], K, b=b, bias=True, act=acts[i % 3]))
      t.append(case(thin_k(b, True), Ms[(i + 2) % 3], Ns[(i + 2) % 3], K, b=b, mask=acts[i % 3]))
      t.append(case(thin_k(b, False), Ms[i % 3], Ns[(i + 2) % 3], K, b=b, mask=acts[(i + 1) % 3], opts={'thin_hoist': 0}))
  t.append(case(grouped(128, 128, 'k', 'm'), 129, 300, 33, b='m', mask='relu'))
  t.append(case(grouped(128, 128, 'k', 'k'), 1000, 68, 33, b='k', bias=True, act='tanh'))
  # gemm_grouped_kernel: every tile config x every layout, ragged edges, odd leading dimensions (scalar loads), every epilogue
  t += [
    case(grouped(16, 128, 'k', 'k'), 5, 130, 17, b='k', bias=True, act='tanh'),
    case(grouped(16, 128, 'k', 'm'), 16, 129, 1, b='m', mask='relu'),
    case(grouped(16, 128, 'k', 'm'), 9, 64, 40, b='m', lda=41, ldb=67, bias=True, act='sigmoid'),
    case(grouped(16, 128, 'm', 'm'), 6, 32, 48, G=3, a='m', b='m', colsum=True),      # last-layer dW of the RED / DRIL dropout nets
    case(grouped(16, 128, 'm', 'm'), 15, 32, 48, a='m', b='m', colsum=True),
    case(grouped(16, 128, 'm', 'm'), 13, 200, 1100, a='m', b='m', lda=17, colsum=True),
    case(grouped(16, 128, 'm', 'm'), 7, 130, 20, a='m', b='m', mask='tanh'),
    case(grouped(128, 16, 'k', 'k'), 300, 7, 45, b='k', bias=True, act='sigmoid'),
    case(grouped(128, 16, 'k', 'k'), 129, 16, 17, b='k', lda=19, ldb=17, mask='relu'),
    case(grouped(128, 16, 'k', 'm'), 130, 13, 20, b='m', mask='sigmoid'),
    case(grouped(128, 16, 'm', 'm'), 100, 10, 40, a='m', b='m', colsum=True),
    case(grouped(128, 16, 'm', 'm'), 66, 3, 2000, a='m', b='m', colsum=True),
    case(grouped(128, 16, 'm', 'm'), 70, 9, 100, a='m', b='m', lda=71, bias=True, act='relu'),
    case(grouped(32, 128, 'k', 'k'), 32, 100, 64, b='k', bias=True, act='relu'),
    case(grouped(32, 128, 'k', 'k'), 17, 129, 1, b='k', mask='tanh'),
    case(grouped(32, 128, 'k', 'm'), 20, 50, 40, b='m', mask='relu'),
    case(grouped(32, 128, 'k', 'm'), 31, 66, 37, b='m', lda=37, ldb=67, bias=True, act='tanh'),
    case(grouped(32, 128, 'm', 'm'), 31, 40, 50, a='m', b='m', colsum=True),
    case(grouped(32, 128, 'm', 'm'), 17, 130, 7, a='m', b='m', ldb=131, mask='sigmoid'),
    case(grouped(128, 128, 'k', 'k'), 129, 130, 17, b='k', lda=17, ldb=17, bias=True, act='relu'),
    case(grouped(128, 128, 'k', 'k'), 129, 130, 1, b='k'),
    case(grouped(128, 128, 'k', 'm'), 129, 130, 17, b='m', mask='tanh'),
    case(grouped(128, 128, 'k', 'm'), 200, 140, 300, b='m', lda=301, bias=True, act='sigmoid'),
    case(grouped(128, 128, 'm', 'm'), 129, 130, 17, a='m', b='m', colsum=True),
    case(grouped(128, 128, 'm', 'm'), 129, 130, 300, a='m', b='m', lda=129, ldb=133, colsum=True),
    case(grouped(128, 128, 'm', 'm'), 140, 129, 70, a='m', b='m', bias=True, act='tanh'),
    case(grouped(128, 128, 'm', 'm'), 130, 131, 65, a='m', b='m', mask='sigmoid'),
  ]
  return t


ROUTES = _route_table()


# ---- one il_debug_gemm call -----------------------------------------------------------------------------------------------------------
def _r4(x): return (x + 3) // 4 * 4


def _operand(rows, cols, ld, G, off, gen):
  """Random [G, rows, cols] matrix with leading dimension ld, group stride a multiple of 4, `off` floats into its buffer; padding is random too."""
  gs = _r4(rows * ld)
  buf = torch.randn(off + G * gs + 4, device=DEV, generator=gen)
  return buf, buf.as_strided((G, rows, cols), (gs, ld, 1), off), gs


class Problem:
  def __init__(self, p, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    M, N, K, G = p['M'], p['N'], p['K'], p['G']
    self.p = p
    self.a_buf, a, self.a_gs = _operand(M, K, p['lda'], G, p['a_off'], gen) if p['a'] == 'k' else _operand(K, M, p['lda'], G, p['a_off'], gen)
    self.b_buf, b, self.b_gs = _operand(N, K, p['ldb'], G, 0, gen) if p['b'] == 'k' else _operand(K, N, p['ldb'], G, 0, gen)
    self.A = a if p['a'] == 'k' else a.transpose(1, 2)  # logical [G, M, K]
    self.B = b.transpose(1, 2) if p['b'] == 'k' else b  # logical [G, K, N]
    self.ld_bias = _r4(N)
    self.bias = torch.randn(G, self.ld_bias, device=DEV, generator=gen) if p['bias'] else None
    self.mask = None
    if p['mask']:  # activation outputs: half of the ReLU ones are <= 0
      z = torch.randn(G, M, _r4(N), device=DEV, generator=gen)
      self.mask = {'relu': torch.relu(z), 'tanh': torch.tanh(z), 'sigmoid': torch.sigmoid(z)}[p['mask']].contiguous()
    self.ldc = _r4(N) + 4
    self.C = torch.empty(G + 1, M + 1, self.ldc, device=DEV)
    self.cs = torch.empty(G + 1, M + 4, device=DEV) if p['colsum'] else None
    self.inputs = [t.clone() for t in (self.a_buf, self.b_buf, self.bias, self.mask) if t is not None]

  def reset(self):
    p = self.p
    self.C.fill_(SENTINEL)
    self.C[:p['G'], :p['M'], :p['N']] = float('nan')
    if self.cs is not None:
      self.cs.fill_(SENTINEL)
      self.cs[:p['G'], :p['M']] = float('nan')

  def call(self, G=None, M=None):
    from il_b200 import _lib
    p = self.p
    G, M = p['G'] if G is None else G, p['M'] if M is None else M
    return _lib.lib().il_debug_gemm(_lib.handle(), M, p['N'], p['K'], G, self.a_buf.data_ptr() + 4 * p['a_off'], self.a_gs, p['lda'], int(p['a'] == 'k'),
                                    self.b_buf.data_ptr(), self.b_gs, p['ldb'], int(p['b'] == 'k'), self.C.data_ptr(), self.C.stride(0), self.ldc,
                                    _lib.ptr(self.bias), self.ld_bias if self.bias is not None else 0, ACT[p['act']],
                                    _lib.ptr(self.mask), self.mask.stride(0) if self.mask is not None else 0, self.mask.stride(1) if self.mask is not None else 0,
                                    ACT[p['mask']] if p['mask'] else 0, _lib.ptr(self.cs), self.cs.stride(0) if self.cs is not None else 0, _lib.stream())

  def run(self):
    """Resets the outputs, runs the call and returns the kernels it launched (one library launch per call)."""
    from il_b200 import _lib
    import il_b200
    calls = []
    def call():
      before = il_b200.launch_count()
      _lib.check(self.call())
      calls.append(il_b200.launch_count() - before)
    names = kernels_of(call, attempts=3, setup=self.reset)
    assert set(calls) == {1}, f'library launches per GEMM: {calls}'
    return names


def _ulp(x):
  a = x.abs()
  return (torch.nextafter(a, torch.full_like(a, float('inf'))) - a).double()


def _assert_within(got, ref, bound, what):
  err = (got.double() - ref).abs()
  bad = ~(err <= bound)  # NaN counts as bad
  if bad.any():
    i = tuple(int(v) for v in bad.nonzero()[0])
    raise AssertionError(f'{what}: {int(bad.sum())} of {bad.numel()} elements outside the fp32 bound; first at {i}: got {got[i].item()!r}, '
                         f'float64 {ref[i].item()!r}, |err| {err[i].item():.3e} > bound {bound[i].item():.3e}')


def check_problem(pb):
  """Values against float64, coverage of the output, the guard band and the untouched inputs."""
  p, G, M, N, K = pb.p, pb.p['G'], pb.p['M'], pb.p['N'], pb.p['K']
  for before, after in zip(pb.inputs, [t for t in (pb.a_buf, pb.b_buf, pb.bias, pb.mask) if t is not None]):
    assert torch.equal(before, after), 'an input operand was modified'
  region = torch.zeros_like(pb.C, dtype=torch.bool)
  region[:G, :M, :N] = True
  got = pb.C[:G, :M, :N]
  assert not torch.isnan(got).any(), f'{int(torch.isnan(got).sum())} output elements never written'
  guard = pb.C[~region]
  assert (guard == SENTINEL).all(), f'{int((guard != SENTINEL).sum())} elements outside the M x N x G output overwritten'
  A, B = pb.A.double(), pb.B.double()
  ref, absprod = A @ B, A.abs() @ B.abs()
  bound = 2 * K * U * absprod
  if pb.bias is not None:
    b = pb.bias[:, None, :N].double()
    ref, bound = ref + b, bound + 2 * U * b.abs()
  if p['act'] == 'relu': ref = torch.relu(ref)
  elif p['act'] == 'tanh': ref = torch.tanh(ref)
  elif p['act'] == 'sigmoid': ref = torch.sigmoid(ref)
  if p['act'] in ('tanh', 'sigmoid'): bound = bound + 4 * _ulp(got)
  if p['mask']:
    y = pb.mask[:, :M, :N].double()
    g = {'relu': (y > 0).double(), 'tanh': 1 - y * y, 'sigmoid': y * (1 - y)}[p['mask']]
    # tanh / sigmoid: act'(y) itself is evaluated in fp32 (1 - y*y, y*(1 - y)): up to 4 ulp of the unmasked value
    bound = bound * g.abs() + (4 * U * ref.abs() if p['mask'] != 'relu' else 0)
    ref = ref * g
  _assert_within(got, ref, bound, 'C')
  if pb.cs is not None:
    cs = pb.cs[:G, :M]
    assert not torch.isnan(cs).any(), f'{int(torch.isnan(cs).sum())} column sums never written'
    cregion = torch.zeros_like(pb.cs, dtype=torch.bool)
    cregion[:G, :M] = True
    assert (pb.cs[~cregion] == SENTINEL).all(), 'elements outside the G x M column sums overwritten'
    _assert_within(cs, A.sum(2), 2 * K * U * A.abs().sum(2), 'colsum')


@pytest.mark.parametrize('p', ROUTES)
def test_gemm_route(p):
  from il_b200 import _lib
  pb = Problem(p, seed=p['M'] * 7919 + p['N'] * 131 + p['K'])
  try:
    set_options(**p['opts'])
    names = pb.run()
    assert names == [p['kernel']], f'expected only {p["kernel"]}, the call ran {names}'
    check_problem(pb)
    out, cs = pb.C.clone(), None if pb.cs is None else pb.cs.clone()
    _lib.check(_lib.lib().il_set_gemm_mode(_lib.handle(), _lib.GEMM_MODE['tf32x3']))
    names = pb.run()
  finally:
    restore_options()
  assert names == [p['kernel']], f'tf32x3 mode: expected only {p["kernel"]}, the call ran {names}'
  assert torch.equal(pb.C.view(torch.int32), out.view(torch.int32)), 'tf32x3 mode changed the output of an FFMA route'
  if cs is not None: assert torch.equal(pb.cs.view(torch.int32), cs.view(torch.int32)), 'tf32x3 mode changed the column sums'


@pytest.mark.parametrize('what,p,G,M,text', [
  ('a_mmajor_b_kmajor', spec('-', 64, 64, 64, a='m', b='k')[0], None, None, 'unsupported operand layout'),
  ('colsum_a_kmajor', spec('-', 64, 64, 64, a='k', b='m', colsum=True)[0], None, None, 'colsum needs'),
  ('too_many_groups', spec('-', 32, 64, 16)[0], 65536, None, 'too many groups'),
  ('empty', spec('-', 32, 64, 16)[0], None, 0, 'empty problem'),
])
def test_gemm_refused(what, p, G, M, text):
  import il_b200
  from il_b200 import _lib
  pb = Problem(p, seed=1)
  pb.reset()
  before, c0 = il_b200.launch_count(), pb.C.clone()
  rc = pb.call(G=G, M=M)
  torch.cuda.synchronize()
  assert rc != 0, 'the call was accepted'
  assert text in _lib.last_error(), _lib.last_error()
  assert il_b200.launch_count() == before, 'a refused call launched a kernel'
  assert torch.equal(torch.isnan(pb.C), torch.isnan(c0)) and torch.equal(pb.C.nan_to_num(), c0.nan_to_num()), 'a refused call wrote its output'


# ---- MLP-level kernels --------------------------------------------------------------------------------------------------------------------
def _actor_params(S, A, H, R, seed):
  """R replicas of [W0, b0, W1, b1, W2, b2] (fp32 values held in float64, CPU): ~unit-scale activations, biases not zero."""
  g = torch.Generator().manual_seed(seed)
  dims = [S, H, H, 2 * A]
  params = [[t for l in range(3) for t in (torch.randn(dims[l + 1], dims[l], generator=g, dtype=torch.float64) * (2 / dims[l]) ** 0.5,
                                         0.1 * torch.randn(dims[l + 1], generator=g, dtype=torch.float64))] for _ in range(R)]
  return [[t.float().double() for t in ps] for ps in params]


def _actor(S, A, H, params):
  import il_b200
  actor = il_b200.SoftActor(S, A, SimpleNamespace(hidden_size=H, depth=2, activation='relu'), replicas=len(params))
  for r, ps in enumerate(params): actor.mlp.load_params(r, 0, [t.float() for t in ps])
  return actor


def _assert_vs_f64(cuda, f64, f32, what):
  """max |cuda - f64| <= 8 max |cpu_f32 - f64| + 1e-6 max |f64|: the kernel is as accurate as the same arithmetic in fp32 on the CPU."""
  cuda, f64, f32 = (np.asarray(x, np.float64) for x in (cuda, f64, f32))
  err, cpu_err, scale = np.abs(cuda - f64).max(), np.abs(f32 - f64).max(), np.abs(f64).max()
  assert err <= 8 * cpu_err + 1e-6 * scale, f'{what}: max |cuda - f64| = {err:.3e}, max |cpu fp32 - f64| = {cpu_err:.3e}, max |f64| = {scale:.3e}'


@pytest.mark.parametrize('S,A,H', [(12, 3, 32), (12, 3, 256), (18, 6, 48)])
@pytest.mark.parametrize('n', [1, 2, 8, 9, 32, 33])
def test_actor_forward_matches_float64(S, A, H, n):
  """SoftActor._run (mean, log_std) for n rows per replica: n = 1 (the acting call of every training step) and 2 <= n <= 32 run the fused
  whole-MLP kernel, n = 33 the per-layer GEMMs."""
  from oracle import port
  from il_b200 import _lib
  R = 3
  params = _actor_params(S, A, H, R, seed=100 * S + n)
  states = torch.randn(R, n, S, generator=torch.Generator().manual_seed(n)).double()
  _lib.check(_lib.lib().il_set_gemm_mode(_lib.handle(), _lib.GEMM_MODE['fp32']))
  actor = _actor(S, A, H, params)
  out = {}
  names = kernels_of(lambda: out.update(actor._run(states.float().cuda(), want=('mean', 'log_std'))), attempts=3)
  small = [k for k in names if k.startswith('mlp_small_forward_kernel')]
  if n == 1: assert small == ['mlp_small_forward_kernel<1>'], names
  elif n <= 32: assert small == ['mlp_small_forward_kernel<8>'], names
  else: assert not small and any('gemm' in k for k in names), names
  for i, key in enumerate(('mean', 'log_std')):
    f64 = np.stack([port.actor_mean_logstd(params[r], states[r])[i].numpy() for r in range(R)])
    f32 = np.stack([port.actor_mean_logstd([t.float() for t in params[r]], states[r].float())[i].numpy() for r in range(R)])
    _assert_vs_f64(out[key].cpu().numpy(), f64, f32, f'{key} (n={n})')


class _GradOnly:
  """Optimiser stand-in for oracle.port.behavioural_cloning_update: keeps the gradients, takes no step."""
  def zero_grad(self, set_to_none=True): pass
  def step(self): pass


def _bc_reference_grads(params, states, actions, weights, dtype):
  from oracle import port
  ps = [torch.nn.Parameter(t.to(dtype).clone()) for t in params]
  port.behavioural_cloning_update(ps, _GradOnly(), {'states': states.to(dtype), 'actions': actions.to(dtype), 'weights': weights.to(dtype)})
  return [p.grad.detach() for p in ps]


def _bc_case(n, A, H, head_fused):
  import il_b200
  from il_b200 import _lib
  R, S = 2, 12
  params = _actor_params(S, A, H, R, seed=7 * n + A + H)
  g = torch.Generator().manual_seed(n + 1000 * A)
  states = torch.randn(R, n, S, generator=g).double()
  actions = (torch.rand(R, n, A, generator=g, dtype=torch.float64) * 1.8 - 0.9).float().double()  # |a| <= 0.9: away from the 1 - 1e-6 clamp
  weights = torch.rand(R, n, generator=g, dtype=torch.float64).float().double() + 0.5
  actor = _actor(S, A, H, params)
  opt = il_b200.AdamW(actor.parameters(), lr=1e-3, weight_decay=0.0)
  batch = il_b200.TransitionBatch.from_dict({'states': states.float(), 'actions': actions.float(), 'weights': weights.float()}, absorbing=False, device='cuda')
  _lib.check(_lib.lib().il_set_gemm_mode(_lib.handle(), _lib.GEMM_MODE['fp32']))
  try:
    set_options(head_fused=head_fused)
    names = kernels_of(lambda: il_b200.behavioural_cloning_update(actor, batch, opt))
  finally:
    restore_options()
  fused = 'head_backward_kernel<8>' in names
  assert fused == (head_fused == 1 and n <= 1024 and 2 * A <= 8), f'n={n} A={A} head_fused={head_fused}: head_backward_kernel ran: {fused}'
  grads = [v / (1 - opt.betas[0]) for v in actor.mlp.layer_views(opt.exp_avg)[0]]  # one step from zero moments: exp_avg = (1 - beta1) grad
  for r in range(R):
    f64 = _bc_reference_grads(params[r], states[r], actions[r], weights[r], torch.float64)
    f32 = _bc_reference_grads(params[r], states[r], actions[r], weights[r], torch.float32)
    for i, (name, cuda) in enumerate(zip(('W0', 'b0', 'W1', 'b1', 'W2', 'b2'), grads)):
      _assert_vs_f64(cuda[r].cpu().numpy(), f64[i].numpy(), f32[i].numpy(), f'd{name} replica {r} (n={n}, A={A}, H={H})')


@pytest.mark.parametrize('H', [32, 40])
@pytest.mark.parametrize('A', [3, 6])
@pytest.mark.parametrize('n', [1, 17, 1024, 1025])
def test_bc_gradient_matches_float64(n, A, H):
  """One behavioural-cloning step: the gradient (first Adam moment / (1 - beta1)) against float64 autograd. A = 3 (head width 6) runs the fused head
  backward for n <= 1024; A = 6 (head width 12) and n = 1025 run the head through the GEMM routes (colsum on the 16 x 128 tile for n < 64 and
  n > 1024)."""
  _bc_case(n, A, H, head_fused=1)


def test_bc_gradient_unfused_head_matches_float64():
  _bc_case(17, 3, 32, head_fused=0)
