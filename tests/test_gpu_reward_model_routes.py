"""Every route of the RED, DRIL, GMMIL and PWIL reward programs (csrc/dropout_nets.cu, csrc/gmmil_pwil.cu) against float64.

Each row of the route tables sits on one side of a shape, mask or tie edge of one C entry, called through `_lib`:
- il_red_update: predictor / target depth 0 to 5 with every activation (and mixed per replica), input / hidden dropout masks, state-only input,
  B from 1 to 512, H from 32 to 256, zero and non-uniform row weights, weight decay; rows with B, H >= 128 run in fp32 and tf32x3 and assert
  from the trace which GEMMs the wgmma engine (tc_gemm_kernel) took. One update from zero AdamW moments leaves m = (1 - beta1) g and
  v = (1 - beta2) g^2: g is compared with the float64 autograd gradient of oracle.port.target_estimation_update under the same masks, v with
  g^2, the parameters with the AdamW formula on the kernel's own m and v; the step counter advances by one and the target stays bitwise.
- il_red_sigma / il_red_reward: the lower median of the B^2 pairwise distances. Exact rows (linear nets, small-integer weights and inputs,
  din a power of two) make every distance exact in fp32 with many ties, so sigma must equal 1 / (lower median) bitwise; random rows compare
  within tolerance after the median's neighbours are drawn clear of the distance error.
- il_actor_log_prob_dropout / il_bc_update_dropout: DRIL's dropout policy, with repeated rows, padded state rows, actions at +-1 (the clamp)
  and the published 5 x 1024-row ensemble on 256 x 2 hidden layers in both GEMM modes; the BC gradient against float64 autograd.
- il_dril_reward: ensemble sizes 2, 5, 7, shared and per-replica q, variance only, strided reward, and a row whose q is its own variance
  (it must get +1: `less_equal`, models.py:117).
- il_gmmil_bandwidth / il_gmmil_reward: B across the 32-row j tile and the 256-row i tile, d up to the shared-memory limit (195 is accepted,
  196 refused), zero and non-uniform weights, R = 3 with different data per replica. The device takes the weighted median by the exact rule:
  the smallest distance whose exact weight sum reaches half the total. The reference (models.py:40-44) normalises the weights in float32 and
  compares a float32 cumsum with 0.5; with equal weights (every shipped configuration) the two pick the same element, which the exact rows
  assert, but with unequal weights they can differ by one element. The rows check the exact rule.
- il_pwil_reward / il_pwil_reset: N from 1 to the shared-memory maximum 56 320 - d, time horizons above, at and below N, call sequences until
  the atoms run out (the device's `break`; the reference fails there on the argmin of an empty tensor), duplicate atoms across strides and
  warps (the tie goes to the first index, as torch.argmin), an `active` mask, per-replica scales and a masked reset. With integer atoms
  every distance is exact, so after every call the live weights must equal the port's bitwise (the port deletes consumed atoms; the device
  marks them -1).
Every row also counts the launches per kernel from a CUDA-activity `torch.profiler` trace, fills the workspace with NaN (with a 4 KB guard
tail), and checks that the inputs and the gaps of strided outputs stay untouched. Values use the tolerance of the MLP head tests
(_assert_vs_f64). Batch rows whose float64 ReLU pre-activation lies within 1e-4 of the kink are drawn again; DRIL thresholds, PWIL argmin
gaps and median neighbours keep a stated margin, so that a flipped comparison is never mistaken for a kernel error. Refusal rows check that a
bad call returns its error, launches nothing and writes nothing.
"""
import ctypes as C
import math
import time
import zlib
from collections import Counter

import numpy as np
import pytest
import torch

from test_gpu_gail_routes import ADAM_EPS, BETAS, DEV, KINK, LR, SENTINEL, U, _GradOnly, _ulp32
from test_gpu_gemm_routes import _assert_vs_f64, kernels_of

pytestmark = pytest.mark.gpu

S0, A0 = 12, 3  # hopper with the absorbing bit
ACTS = ('relu', 'tanh', 'sigmoid')
P_IN, P_HID = 0.05, 0.41  # RED_25_trajectories' input dropout and dropout
WS_TAIL = 4096  # bytes of SENTINEL past the workspace
TF32X3_SLACK = 8  # 3xTF32 products carry ~2^-21 relative error where fp32 carries 2^-24: the CPU fp32 error is scaled by this much
FFMA_GEMMS = ('gemm_grouped_kernel', 'gemm_thin_k_kernel', 'first_layer_relu_kernel', 'first_layer_reg_kernel', 'gemm_stream_tn_kernel', 'wide_tn_kernel', 'row_dot_kernel')
PWIL_SMEM_FLOATS = 220 * 1024 // 4  # N + d of il_pwil_reward's shared-memory check
LEAD_KERNELS = 8  # torch kernels ahead of every traced call (see _launches)


# ---- shared helpers -----------------------------------------------------------------------------------------------------------------------
def _f32(t): return t.float().double()


def _seed(request): return zlib.crc32(request.node.callspec.id.encode())


def _lib():
  from il_b200 import _lib as L
  return L


def _draw_net(dims, g, gain=1.5):
  """[W0, b0, W1, b1, ...] (fp32 values held in float64)."""
  out = []
  for l in range(len(dims) - 1):
    out += [_f32(gain * torch.randn(dims[l + 1], dims[l], generator=g, dtype=torch.float64) / dims[l] ** 0.5), _f32(0.1 * torch.randn(dims[l + 1], generator=g, dtype=torch.float64))]
  return out


def _mask(g, shape, p):
  """Pre-scaled {0, 1 / (1 - p)} dropout mask, as il_fill_dropout_mask draws it (fp32 values held in float64)."""
  keep = torch.rand(*shape, generator=g, dtype=torch.float64) >= p
  return keep.double() * float(np.float32(1 / (1 - np.float32(p))))


def _act(x, act): return torch.relu(x) if act == 'relu' else (torch.tanh(x) if act == 'tanh' else torch.sigmoid(x))


class Flat:
  """R nets of one shape in a flat [R, stride] device buffer whose padding is zero (the il_mlp layout)."""

  def __init__(self, nets, dims):
    from il_b200._lib import py_mlp_offsets
    w, b, total = py_mlp_offsets(dims)
    self.dims, self.stride, self.layout = dims, total, []
    for l in range(len(dims) - 1): self.layout += [(w[l], (dims[l + 1], dims[l])), (b[l], (dims[l + 1], ))]
    R = len(nets)
    buf, self.live = torch.zeros(R, total, dtype=torch.float64), torch.zeros(R, total, dtype=torch.bool)
    for r in range(R):
      for (off, shape), t in zip(self.layout, nets[r]):
        buf[r, off:off + t.numel()] = t.flatten()
        self.live[r, off:off + t.numel()] = True
    self.buf = buf.float().to(DEV)

  def views(self, t, r):
    flat = t[r].double().cpu()
    return [flat[off:off + math.prod(shape)].view(shape) for off, shape in self.layout]

  def struct(self, act, buf=None):
    L = _lib()
    m = L.Mlp()
    m.params, m.stride, m.n_layers, m.activation = (self.buf if buf is None else buf).data_ptr(), self.stride, len(self.dims) - 1, L.ACT[act]
    for i, x in enumerate(self.dims): m.dims[i] = x
    return m

  def padding_zero(self, t, name):
    live = self.live.to(DEV)
    assert (t[~live] == 0).all(), f'{name}: {int((t[~live] != 0).sum())} padding floats of the flat buffer not zero'


def _rows(g, R, B, S, A, ints=False, zero_every=7):
  """[R, B, row] transition rows (float64 holding fp32): random (or small-integer) states and actions, non-uniform weights with zeros."""
  from il_b200._lib import py_row_layout
  off, row = py_row_layout(S, A)
  if ints: x = torch.randint(-3, 4, (R, B, row), generator=g).double()
  else:
    x = _f32(torch.randn(R, B, row, generator=g, dtype=torch.float64))
    x[..., S:S + A] = x[..., S:S + A].clamp(-0.9, 0.9)
  w = _f32(torch.rand(R, B, generator=g, dtype=torch.float64) + 0.5)
  if zero_every: w[:, ::zero_every] = 0.0
  x[..., off['weights']] = w
  return x


def _dev_rows(x, pad=4):
  """Device copy of [R, B, row] rows, replicas B * row + pad floats apart with a SENTINEL gap."""
  R, B, row = x.shape
  buf = torch.full((R, B * row + pad), SENTINEL, dtype=torch.float64)
  buf[:, :B * row] = x.reshape(R, -1)
  return buf.float().to(DEV), B * row + pad


def _batch(buf, rs, B, S, A):
  from il_b200._lib import py_row_layout
  L = _lib()
  b = L.Batch()
  b.rows, b.replica_stride, b.B, b.S, b.A, b.row = buf.data_ptr(), rs, B, S, A, py_row_layout(S, A)[1]
  return b


class Workspace:
  """need bytes of NaN followed by WS_TAIL bytes of SENTINEL."""

  def __init__(self, need):
    self.need = need
    self.t = torch.empty(need // 4 + WS_TAIL // 4, device=DEV)
    self.fill()

  def fill(self):
    self.t[:self.need // 4].fill_(float('nan'))
    self.t[self.need // 4:].fill_(SENTINEL)

  def check_tail(self):
    tail = self.t[self.need // 4:]
    assert (tail == SENTINEL).all(), f'{int((tail != SENTINEL).sum())} floats written past the {self.need}-byte workspace'


def _tally(names):
  """Launches per kernel: FFMA GEMM routes counted together, both AdamW variants as 'adam'."""
  c = Counter(n.split('<', 1)[0] for n in names)
  out = Counter({k: v for k, v in c.items() if k not in FFMA_GEMMS and not k.startswith('adam')})
  out['ffma_gemm'] = sum(c[k] for k in FFMA_GEMMS)
  out['adam'] = sum(v for k, v in c.items() if k.startswith('adam'))
  return +out


_TRACES_COMPLETE = [True]


def _launches(call, setup):
  """Kernels of one call per kernel (see _tally), read from a CUDA-activity trace and cross-checked against the library's launch counter.
  The traced function first launches a few torch kernels, dropped from the list: a trace that loses its first events loses these rather than
  the call's. Late in a long process CUPTI can go on losing events in every trace; after a few attempts the tally is then None and
  _assert_launches checks the launch counter's total alone."""
  import il_b200
  L = _lib()
  counts, lead = [], torch.zeros(1, device=DEV)
  def fn():
    for _ in range(LEAD_KERNELS): lead.add_(1)
    before = il_b200.launch_count()
    L.check(call())
    counts.append(il_b200.launch_count() - before)
  lead_ids = set()
  for attempt in range(4 if _TRACES_COMPLETE else 1):
    try:
      if not lead_ids: lead_ids = set(kernels_of(lambda: lead.add_(1)))
      names = [n for n in kernels_of(fn, attempts=2, setup=setup) if n not in lead_ids]
    except AssertionError:  # a trace without a single kernel event
      names = []
      if not counts:
        setup()
        fn()
    assert len(set(counts)) == 1, f'library launches per call: {counts}'
    assert len(names) <= counts[-1], f'the trace holds {len(names)} kernels of a call that launched {counts[-1]}: {names}'
    if len(names) == counts[-1] and lead_ids: return _tally(names), counts[-1]
    time.sleep(0.1 * (attempt + 1))
  _TRACES_COMPLETE.clear()  # the process's traces stay lossy from here on: later calls take one trace only
  return None, counts[-1]


def _assert_launches(got, want, only=False):
  """got: (tally, total) of _launches. only: want lists some of the call's kernels (the others unchecked)."""
  tally, total = got
  keys, want = set(want), +Counter(want)
  if tally is None:
    if not only: assert total == sum(want.values()), f'{total} launches, expected {dict(want)}'
    else: assert total >= sum(want.values()), f'{total} launches, expected at least {dict(want)}'
    return
  if only: tally = Counter({k: tally[k] for k in keys})
  assert +tally == want, f'launches {dict(tally)}, expected {dict(want)}'


def _uses_tc(mode, M, N, K):
  """launch_gemm's wgmma condition for the contiguous, 16-byte aligned operands of these programs (gemm_uses_tc, tc_gemm_eligible)."""
  return mode == 'tf32x3' and M >= 128 and N == 256 and K >= 128 and M % 128 == 0 and K % 16 == 0


def _gemm_launches(mode, fwd_nets, bwd_dims, n):
  """FFMA / wgmma GEMMs (and the colsum_kernel each wgmma weight-gradient GEMM adds) of forwards over `fwd_nets` and one backward."""
  shapes, wgrad = [], []
  for dims in fwd_nets: shapes += [(n, dims[l + 1], dims[l]) for l in range(len(dims) - 1)]
  if bwd_dims:
    L = len(bwd_dims) - 1
    wgrad = [(bwd_dims[l + 1], bwd_dims[l], n) for l in range(L)]
    shapes += wgrad + [(n, bwd_dims[l], bwd_dims[l + 1]) for l in range(1, L)]
  tc = sum(_uses_tc(mode, *s) for s in shapes)
  return {'tc_gemm_kernel': tc, 'ffma_gemm': len(shapes) - tc, 'colsum_kernel': sum(_uses_tc(mode, *s) for s in wgrad)}


def _close(cuda, f64, f32, what, mode='fp32'):
  if mode != 'fp32': f32 = np.asarray(f64, np.float64) + TF32X3_SLACK * (np.asarray(f32, np.float64) - np.asarray(f64, np.float64))
  _assert_vs_f64(cuda, f64, f32, what)


def _check_adamw(prm, m, v, p0, lr, wd, what):
  """One AdamW step from zero moments: v / (1 - beta2) = g^2 for g = m / (1 - beta1), and the parameters on the kernel's own m, v."""
  g = m / float(np.float32(1 - BETAS[0]))
  vg = v / float(np.float32(1 - BETAS[1]))
  err = (vg - g ** 2).abs()
  assert (err <= 1e-6 * g ** 2).all(), f'{what}: v / (1 - beta2) differs from g^2 by up to {float(err.max()):.3e}'
  term = lr / (1 - BETAS[0]) * m / (v.sqrt() / math.sqrt(1 - BETAS[1]) + ADAM_EPS)
  ref = p0 * (1 - lr * wd) - term
  bound = 3 * _ulp32(ref) + 16 * U * term.abs()
  err = (prm - ref).abs()
  assert (err <= bound).all(), f'{what}: parameter off the AdamW step of its own m, v by {float((err / bound).max()):.2f}x the bound'
  return g


def _adam(opt, m, v, step, wd):
  opt.m, opt.v, opt.step, opt.lr, opt.beta1, opt.beta2, opt.eps, opt.weight_decay = m.data_ptr(), v.data_ptr(), step.data_ptr(), LR, BETAS[0], BETAS[1], ADAM_EPS, wd


def _hidden_pre(params, x, acts_seq, masks_in, masks_hid):
  """float64 inputs of every hidden activation (z * mask) of one dropout MLP evaluation."""
  if masks_in is not None: x = x * masks_in
  zs, L = [], len(params) // 2
  for l in range(L - 1):
    z = x @ params[2 * l].t() + params[2 * l + 1]
    if masks_hid[l] is not None: z = z * masks_hid[l]
    zs.append(z)
    x = _act(z, acts_seq)
  return zs


@pytest.fixture(autouse=True)
def _fp32_gemm():
  L = _lib()
  L.check(L.lib().il_set_gemm_mode(L.handle(), L.GEMM_MODE['fp32']))
  yield
  L.check(L.lib().il_set_gemm_mode(L.handle(), L.GEMM_MODE['fp32']))


def _set_mode(mode):
  L = _lib()
  L.check(L.lib().il_set_gemm_mode(L.handle(), L.GEMM_MODE[mode]))


# ---- RED: il_red_update ---------------------------------------------------------------------------------------------------------------------
def red_upd(B=64, H=64, depth=2, act='tanh', act_r=None, masks='both', p_in=P_IN, p=P_HID, state_only=False, wd=0.0, mode='fp32', R=2, S=S0, A=A0):
  acts = act_r or (act, )
  R = len(act_r) if act_r else R
  prm = dict(B=B, H=H, depth=depth, act=acts[0], act_r=act_r, masks=masks, p_in=p_in, p=p, state_only=state_only, wd=wd, mode=mode, R=R, S=S, A=A)
  tags = [f'B{B}', f'H{H}', f'depth{depth}', '.'.join(act_r) if act_r else act, f'mask-{masks}', f'p{p_in:g}.{p:g}', f'wd{wd:g}', mode] + (['state_only'] if state_only else [])
  return pytest.param(prm, id='-'.join(tags))


def _red_update_table():
  t, kinds = [], ('none', 'in', 'hid', 'both')
  i = 0
  t.append(red_upd(depth=0, act='relu', masks='in', H=32))
  for depth in (1, 2, 3, 5):
    for act in ACTS:
      t.append(red_upd(depth=depth, act=act, masks=kinds[i % 4], H=(32, 64)[i % 2], wd=(0.0, 2.5)[(i // 2) % 2]))
      i += 1
  t += [
    red_upd(depth=2, act_r=('relu', 'tanh', 'sigmoid'), masks='both'),
    red_upd(depth=3, act_r=('sigmoid', 'relu', 'tanh'), masks='hid', H=32, wd=2.5),
    red_upd(depth=2, act='relu', masks='both', state_only=True, p_in=0.41, p=0.05),
    red_upd(depth=1, act='tanh', masks='in', state_only=True, wd=2.5),
    red_upd(B=1, depth=2, act='relu', masks='both'),
    red_upd(B=33, depth=2, act='sigmoid', masks='hid', H=32),
    red_upd(B=257, depth=3, act='tanh', masks='both', H=64),
    red_upd(B=512, depth=2, act='tanh', masks='both', H=64, wd=2.5),  # RED_25_trajectories
  ]
  for mode in ('fp32', 'tf32x3'):
    t.append(red_upd(B=256, depth=2, act='relu', masks='both', H=128, mode=mode))
    t.append(red_upd(B=512, depth=2, act='tanh', masks='both', H=256, mode=mode, wd=2.5))
    t.append(red_upd(B=257, depth=3, act='sigmoid', masks='hid', H=256, mode=mode))
  return t


class RedProblem:
  def __init__(self, p, seed, ints=False):
    self.p, R, B, S, A = p, p['R'], p['B'], p['S'], p['A']
    self.gen = g = torch.Generator().manual_seed(seed)
    self.din = S if p['state_only'] else S + A
    self.dims = [self.din] + [p['H']] * p['depth'] + [self.din]
    self.acts = list(p['act_r']) if p['act_r'] else [p['act']] * R
    self.pred, self.targ = [_draw_net(self.dims, g) for _ in range(R)], [_draw_net(self.dims, g) for _ in range(R)]
    self.rows = _rows(g, R, B, S, A, ints=ints)
    self.use_in, self.use_hid = p['masks'] in ('in', 'both'), p['masks'] in ('hid', 'both')
    self.m_in = _mask(g, (R, B, self.din), p['p_in']) if self.use_in else None
    self.m_hid = [_mask(g, (R, B, p['H']), p['p']) if self.use_hid else None for _ in range(p['depth'])]

  def x(self, r): return self.rows[r][:, :self.din]

  def port_masks(self, r):
    return ([self.m_in[r]] if self.use_in else []) + ([m[r] for m in self.m_hid] if self.use_hid else [])

  def clear_kinks(self):
    """Draws the batch rows (and their masks) again where a float64 ReLU input of the predictor lies within KINK of 0."""
    R, B = self.p['R'], self.p['B']
    for _ in range(100):
      bad = torch.zeros(R, B, dtype=torch.bool)
      for r in range(R):
        if self.acts[r] != 'relu': continue
        zs = _hidden_pre(self.pred[r], self.x(r), 'relu', self.m_in[r] if self.use_in else None, [m[r] if m is not None else None for m in self.m_hid])
        for z in zs: bad[r] |= ((z.abs() < KINK) & (z != 0)).any(1)  # z = 0: a dropped unit, whose gradient is 0 either side
      if not bad.any(): return
      n = int(bad.sum())
      fresh = _rows(self.gen, 1, n, self.p['S'], self.p['A'], zero_every=0)[0]
      self.rows[bad] = fresh
      if self.use_in: self.m_in[bad] = _mask(self.gen, (n, self.din), self.p['p_in'])
      for m in self.m_hid:
        if m is not None: m[bad] = _mask(self.gen, (n, self.p['H']), self.p['p'])
    raise AssertionError('could not draw a batch away from the ReLU kink')

  def port_forward(self, r, dtype):
    """(prediction, target) of replica r's rows under its masks."""
    x, S = self.x(r).to(dtype), self.p['S']
    return self.port_disc(r, dtype).forward(x[:, :S], x[:, S:], masks=[m.to(dtype) for m in self.port_masks(r)])

  def port_disc(self, r, dtype, train=True):
    from oracle import port
    p = self.p
    disc = port.RedDiscriminator(self.pred[r], self.targ[r], p['state_only'], self.acts[r], p['p_in'] if self.use_in else 0.0, p['p'] if self.use_hid else 0.0)
    disc.predictor = [torch.nn.Parameter(t.to(dtype).clone()) for t in self.pred[r]]  # __init__ casts to float32
    disc.target = [t.to(dtype).clone() for t in self.targ[r]]
    disc.training = train
    return disc

  def port_update(self, r, dtype):
    from oracle import port
    from il_b200._lib import py_row_layout
    S, A = self.p['S'], self.p['A']
    x = self.rows[r].to(dtype)
    wo = py_row_layout(S, A)[0]['weights']
    disc = self.port_disc(r, dtype)
    loss = port.target_estimation_update(disc, _GradOnly(), dict(states=x[:, :S], actions=x[:, S:S + A], weights=x[:, wo]), masks=[m.to(dtype) for m in self.port_masks(r)])
    return [q.grad.detach().double() for q in disc.predictor], loss.item()


class RedDevice:
  def __init__(self, pb):
    p, R = pb.p, pb.p['R']
    self.pb = pb
    self.pred, self.targ = Flat(pb.pred, pb.dims), Flat(pb.targ, pb.dims)
    self.m, self.v = torch.zeros_like(self.pred.buf), torch.zeros_like(self.pred.buf)
    self.step = torch.zeros(1, dtype=torch.int64, device=DEV)
    self.rows, self.rs = _dev_rows(pb.rows)
    self.m_in = pb.m_in.float().to(DEV) if pb.use_in else None
    self.m_hid = [m.float().to(DEV) if m is not None else None for m in pb.m_hid]
    self.act_r = torch.tensor([_lib().ACT[a] for a in pb.acts], dtype=torch.int32, device=DEV) if p['act_r'] else None
    self.sigma = torch.full((R + 1, ), SENTINEL, device=DEV)
    self.loss = torch.full((R + 1, ), SENTINEL, device=DEV)
    self.inputs = [t.clone() for t in self._inputs()]
    self.state0 = [t.clone() for t in self._state()]

  def _inputs(self): return [t for t in [self.rows, self.m_in, self.act_r, self.targ.buf] + self.m_hid if t is not None]

  def _state(self): return [self.pred.buf, self.m, self.v, self.step, self.loss, self.sigma]

  def reset(self):
    for t, t0 in zip(self._state(), self.state0): t.copy_(t0)
    self.ws.fill()

  def disc(self, R=None):
    L, pb = _lib(), self.pb
    d = L.Red()
    d.predictor, d.target = self.pred.struct(pb.p['act']), self.targ.struct(pb.p['act'])
    d.sigma, d.state_only = self.sigma.data_ptr(), int(pb.p['state_only'])
    if self.act_r is not None: d.activation_r = self.act_r.data_ptr()
    return d

  def batch(self): return _batch(self.rows, self.rs, self.pb.p['B'], self.pb.p['S'], self.pb.p['A'])

  def workspace(self):
    d = self.disc()
    self.ws = Workspace(_lib().lib().il_red_workspace_bytes(C.byref(d), self.pb.p['R'], self.pb.p['B']))
    return self.ws

  def update_args(self):
    L, p = _lib(), self.pb.p
    a = L.RedUpdateArgs()
    a.disc, a.batch, a.R = self.disc(), self.batch(), p['R']
    _adam(a.opt, self.m, self.v, self.step, p['wd'])
    a.mask_in = L.ptr(self.m_in)
    for l, m in enumerate(self.m_hid): a.mask_hid[l] = L.ptr(m)
    a.out_loss, a.workspace, a.workspace_bytes = self.loss.data_ptr(), self.ws.t.data_ptr(), self.ws.need
    return a

  def check_inputs(self):
    for i, (before, after) in enumerate(zip(self.inputs, self._inputs())): assert torch.equal(before, after), f'input {i} (rows, masks, activations, target) modified'
    self.ws.check_tail()


@pytest.mark.parametrize('p', _red_update_table())
def test_red_update_route(p, request):
  L = _lib()
  lib = L.lib()
  pb = RedProblem(p, _seed(request))
  pb.clear_kinks()
  dv = RedDevice(pb)
  dv.workspace()
  a = dv.update_args()
  _set_mode(p['mode'])
  got = _launches(lambda: lib.il_red_update(L.handle(), C.byref(a), L.stream()), dv.reset)
  depth, B = p['depth'], p['B']
  want = dict(tick_kernel=1, input_mask_kernel=int(pb.use_in), dropout_act_kernel=2 * depth, red_loss_kernel=1, dropout_bwd_kernel=depth, adam=1,
              **_gemm_launches(p['mode'], [pb.dims, pb.dims], pb.dims, B))
  _assert_launches(got, want)
  assert int(dv.step.item()) == 1, f'step counter {int(dv.step.item())} after one update'
  for name, t in (('params', dv.pred.buf), ('m', dv.m), ('v', dv.v)): dv.pred.padding_zero(t, name)
  assert dv.loss[p['R']].item() == SENTINEL, 'loss written past its R slots'
  dv.check_inputs()
  names = [f'{"Wb"[i % 2]}{i // 2}' for i in range(2 * (depth + 1))]
  for r in range(p['R']):
    what = f'replica {r} ({pb.acts[r]})'
    g64, l64 = pb.port_update(r, torch.float64)
    g32, l32 = pb.port_update(r, torch.float32)
    _close(dv.loss[r].item(), l64, l32, f'loss {what}', p['mode'])
    m, v, prm = (dv.pred.views(t, r) for t in (dv.m, dv.v, dv.pred.buf))
    for i, name in enumerate(names):
      g = _check_adamw(prm[i], m[i], v[i], pb.pred[r][i], LR, p['wd'], f'{name} {what}')
      _close(g.numpy(), g64[i].numpy(), g32[i].numpy(), f'd{name} {what}', p['mode'])


# ---- RED: il_red_sigma / il_red_reward --------------------------------------------------------------------------------------------------------
def red_sig(B, exact, depth=0, act='tanh', masks='in', act_r=None, state_only=False, R=2, H=32):
  S, A = (5, 3) if not state_only else (8, 3)  # din = 8 either way: a power of two, so exact rows' distance means stay exact
  base = red_upd(B=B, H=H, depth=depth, act=act, act_r=act_r, masks=masks, p_in=0.5 if exact else P_IN, state_only=state_only, R=R, S=S, A=A).values[0]
  prm = dict(base, exact=exact)
  return pytest.param(prm, id=f'{"exact" if exact else "random"}-B{B}-depth{depth}-{".".join(act_r) if act_r else act}-mask-{masks}' + ('-state_only' if state_only else ''))


SIGMA_ROUTES = ([red_sig(B, True) for B in (1, 2, 3, 64, 512, 1024)] + [red_sig(33, True, masks='none', state_only=True)] +
                [red_sig(64, False, depth=2, act='tanh', masks='both'), red_sig(257, False, depth=3, act_r=('relu', 'sigmoid', 'tanh'), masks='both', R=3),
                 red_sig(512, False, depth=1, act='relu', masks='hid', H=64)])


SIGMA_EPS = 2e-5


def _lower_median(v):
  s = torch.sort(v.flatten()).values
  k = (s.numel() - 1) // 2
  return s, k


@pytest.mark.parametrize('p', SIGMA_ROUTES)
def test_red_sigma_route(p, request):
  """Exact rows: sigma is 1 / (lower median) bitwise. Random rows: the device's median has rank (B^2 - 1) / 2 among the float64 distances up
  to SIGMA_EPS, a bound on their relative fp32 error (among 10^5 to 10^6 distances, neighbours of the median always lie closer than that)."""
  from oracle import port
  L = _lib()
  lib = L.lib()
  R, B = p['R'], p['B']
  pb = RedProblem(p, _seed(request), ints=p['exact'])
  if p['exact']:  # small-integer linear nets: every prediction, difference and mean over din = 8 is exact in fp32
    pb.pred = [[torch.randint(-2, 3, t.shape, generator=pb.gen).double() for t in net] for net in pb.pred]
    pb.targ = [[torch.randint(-2, 3, t.shape, generator=pb.gen).double() for t in net] for net in pb.targ]
  dv = RedDevice(pb)
  dv.workspace()
  d, b = dv.disc(), dv.batch()
  call = lambda: lib.il_red_sigma(L.handle(), C.byref(d), R, C.byref(b), L.ptr(dv.m_in), L.mask_array(dv.m_hid), dv.ws.t.data_ptr(), dv.ws.need, L.stream())
  got = _launches(call, dv.reset)
  _assert_launches(got, dict(input_mask_kernel=int(pb.use_in), dropout_act_kernel=2 * p['depth'], red_pairwise_kernel=1, red_median_kernel=1,
                             **_gemm_launches('fp32', [pb.dims, pb.dims], None, B)))
  dv.check_inputs()
  for i, (t, t0) in enumerate(zip(dv._state()[:5], dv.state0[:5])): assert torch.equal(t, t0), f'il_red_sigma wrote state {i} (predictor, m, v, step, loss)'
  assert dv.sigma[R].item() == SENTINEL, 'sigma written past its R slots'
  for r in range(R):
    D64 = port.squared_distance_mean(*pb.port_forward(r, torch.float64))
    assert D64.dtype == torch.float64
    s, k = _lower_median(D64)
    if p['exact']:
      med32 = s.float()[k]
      assert med32.double().item() == s[k].item(), 'an exact row\'s distance is not exact in fp32'
      want = (1 / med32).item()  # fp32 division, as the kernel's 1.f / median
      assert dv.sigma[r].item() == want, f'replica {r}: sigma {dv.sigma[r].item()!r}, 1 / lower median {want!r} (median {s[k].item()}, k = {k} of {s.numel()})'
    else:
      med = 1 / dv.sigma[r].double().item()
      below, upto = int((s < med * (1 - SIGMA_EPS)).sum()), int((s <= med * (1 + SIGMA_EPS)).sum())
      assert below <= k < upto, f'replica {r}: 1 / sigma = {med!r} has rank {below}..{upto - 1} among the float64 distances, the lower median has rank {k} ({s[k].item()!r})'


@pytest.mark.parametrize('B,ld,depth,act', [(1, 1, 0, 'relu'), (64, 2, 2, 'tanh'), (257, 3, 3, 'sigmoid'), (512, 1, 2, 'relu')])
def test_red_reward_route(B, ld, depth, act, request):
  """Eval mode (no masks), per-replica sigma, a strided output with reward_rs > B * ld."""
  L = _lib()
  lib = L.lib()
  R = 3
  pb = RedProblem(red_upd(B=B, depth=depth, act=act, masks='none', R=R).values[0], _seed(request))
  dv = RedDevice(pb)
  sig = torch.tensor([0.5, 3.0, 0.125], device=DEV)
  dv.sigma[:R] = sig
  dv.state0 = [t.clone() for t in dv._state()]
  dv.workspace()
  rs = B * ld + 5
  reward = torch.full((R * rs + 1, ), SENTINEL, device=DEV)
  d, b = dv.disc(), dv.batch()
  def setup():
    dv.reset()
    reward.fill_(SENTINEL)
  got = _launches(lambda: lib.il_red_reward(L.handle(), C.byref(d), R, C.byref(b), reward.data_ptr(), rs, ld, dv.ws.t.data_ptr(), dv.ws.need, L.stream()), setup)
  _assert_launches(got, dict(dropout_act_kernel=2 * depth, red_reward_kernel=1, **_gemm_launches('fp32', [pb.dims, pb.dims], None, B)))
  dv.check_inputs()
  for i, (t, t0) in enumerate(zip(dv._state(), dv.state0)): assert torch.equal(t, t0), f'il_red_reward wrote state {i}'
  written = torch.zeros_like(reward, dtype=torch.bool)
  for r in range(R):
    idx = r * rs + torch.arange(B, device=DEV) * ld
    written[idx] = True
    ref = []
    for dtype in (torch.float64, torch.float32):
      disc = pb.port_disc(r, dtype, train=False)
      disc.sigma_1 = sig[r].item()
      x = pb.x(r).to(dtype)
      with torch.no_grad(): ref.append(disc.predict_reward(x[:, :S0], x[:, S0:]).double().numpy())
    _assert_vs_f64(reward[idx].double().cpu().numpy(), ref[0], ref[1], f'reward replica {r}')
  assert (reward[~written] == SENTINEL).all(), f'{int((reward[~written] != SENTINEL).sum())} reward floats outside the strided output written'


# ---- DRIL: il_actor_log_prob_dropout -----------------------------------------------------------------------------------------------------------
def actor_lp(rows, repeat, H=32, depth=2, act='tanh', act_r=None, masks='both', mode='fp32', A=A0, R=2):
  R = len(act_r) if act_r else R
  prm = dict(rows=rows, repeat=repeat, H=H, depth=depth, act=act, act_r=act_r, masks=masks, mode=mode, A=A, R=R)
  return pytest.param(prm, id=f'n{rows * repeat}-repeat{repeat}-H{H}-depth{depth}-{".".join(act_r) if act_r else act}-mask-{masks}-A{A}-{mode}')


ACTOR_ROUTES = [
  actor_lp(64, 1, act='relu', masks='none'),
  actor_lp(64, 1, act='sigmoid', masks='in'),
  actor_lp(33, 5, act='tanh', masks='hid', depth=1, H=64),
  actor_lp(29, 5, act_r=('relu', 'tanh', 'sigmoid'), masks='both'),
  actor_lp(7, 5, act='relu', masks='both', depth=3, A=1),
  actor_lp(1024, 5, H=256, depth=2, act='tanh', masks='both', mode='fp32'),  # DRIL: batch 1024 x the 5-member ensemble
  actor_lp(1024, 5, H=256, depth=2, act='tanh', masks='both', mode='tf32x3'),
  actor_lp(1024, 5, H=256, depth=2, act_r=('relu', 'sigmoid'), masks='both', mode='tf32x3'),
]


@pytest.mark.parametrize('p', ACTOR_ROUTES)
def test_actor_log_prob_dropout_route(p, request):
  from oracle import port
  L = _lib()
  lib = L.lib()
  R, rows, rep, A, S = p['R'], p['rows'], p['repeat'], p['A'], S0
  n = rows * rep
  g = torch.Generator().manual_seed(_seed(request))
  dims = [S] + [p['H']] * p['depth'] + [2 * A]
  acts = list(p['act_r']) if p['act_r'] else [p['act']] * R
  nets = [_draw_net(dims, g, gain=1.0) for _ in range(R)]
  ld = S + 5  # padded state rows
  states = _f32(torch.randn(R, rows, S, generator=g, dtype=torch.float64))
  actions = _f32(torch.rand(R, rows, A, generator=g, dtype=torch.float64) * 1.8 - 0.9)
  actions[:, ::3, 0], actions[:, 1::3, -1] = 1.0, -1.0  # at the clamp (1 - 1e-6 in fp32)
  use_in, use_hid = p['masks'] in ('in', 'both'), p['masks'] in ('hid', 'both')
  p_in, p_h = 0.21, 0.21
  m_in = _mask(g, (R, n, S), p_in) if use_in else None
  m_hid = [_mask(g, (R, n, p['H']), p_h) if use_hid else None for _ in range(p['depth'])]
  flat = Flat(nets, dims)
  srs = rows * ld + 7
  sbuf = torch.full((R, srs), SENTINEL, dtype=torch.float64)
  sbuf[:, :rows * ld].view(R, rows, ld)[..., :S] = states
  sdev = sbuf.float().to(DEV)
  adev = actions.float().to(DEV).contiguous()
  mdev_in = m_in.float().to(DEV) if use_in else None
  mdev_hid = [m.float().to(DEV) if m is not None else None for m in m_hid]
  act_r = torch.tensor([L.ACT[a] for a in acts], dtype=torch.int32, device=DEV) if p['act_r'] else None
  inputs = [t.clone() for t in [sdev, adev, flat.buf] + ([mdev_in] if use_in else []) + [m for m in mdev_hid if m is not None]]
  m = flat.struct(p['act'])
  ws = Workspace(lib.il_actor_dropout_workspace_bytes(C.byref(m), R, n))
  out = torch.full((R * n + 1, ), SENTINEL, device=DEV)
  def setup():
    ws.fill()
    out.fill_(SENTINEL)
  _set_mode(p['mode'])
  call = lambda: lib.il_actor_log_prob_dropout(L.handle(), C.byref(m), R, n, rep, sdev.data_ptr(), srs, ld, adev.data_ptr(), L.ptr(mdev_in), L.mask_array(mdev_hid), out.data_ptr(),
                                               ws.t.data_ptr(), ws.need, L.stream(), L.ptr(act_r))
  got = _launches(call, setup)
  _assert_launches(got, dict(input_mask_kernel=2, dropout_act_kernel=p['depth'], actor_head_kernel=1, **_gemm_launches(p['mode'], [dims], None, n)))
  for i, (t, t0) in enumerate(zip([sdev, adev, flat.buf] + ([mdev_in] if use_in else []) + [m for m in mdev_hid if m is not None], inputs)):
    assert torch.equal(t, t0), f'input {i} modified'
  ws.check_tail()
  assert out[R * n].item() == SENTINEL, 'log_prob written past its R x n outputs'
  lp = out[:R * n].view(R, n).double().cpu()
  for r in range(R):
    x, a = torch.repeat_interleave(states[r], rep, 0), torch.repeat_interleave(actions[r], rep, 0)
    pm = ([m_in[r]] if use_in else []) + ([mm[r] for mm in m_hid] if use_hid else [])
    drop = dict(input_dropout=p_in if use_in else 0.0, dropout=p_h if use_hid else 0.0, training=True)
    # the reference runs in fp32: its clamp bound is fl32(1 - 1e-6), below 1 - 1e-6, so the float64 density takes the fp32-clamped action
    a32 = a.float().clamp(-1 + 1e-6, 1 - 1e-6).double()
    mean, log_std = port.actor_mean_logstd(nets[r], x, acts[r], masks=list(pm), **drop)
    f64 = port.tanh_gaussian_logprob_from_pre_tanh(mean, log_std, torch.atanh(a32))
    f32 = port.actor_log_prob([t.float() for t in nets[r]], x.float(), a.float(), acts[r], masks=[t.float() for t in pm], **drop).double()
    _close(lp[r].numpy(), f64.numpy(), f32.numpy(), f'log_prob replica {r} ({acts[r]})', p['mode'])


# ---- DRIL: il_bc_update_dropout ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('B,A,act,masks,with_loss', [(1, 3, 'tanh', 'both', True), (17, 1, 'relu', 'in', False), (17, 6, 'sigmoid', 'hid', True), (1024, 8, 'tanh', 'both', True),
                                                     (1025, 3, 'relu', 'both', False), (1025, 6, 'tanh', 'none', True)])
def test_bc_update_dropout_route(B, A, act, masks, with_loss, request):
  from oracle import port
  from il_b200._lib import py_row_layout
  L = _lib()
  lib = L.lib()
  R, S, H, depth, wd = 2, S0, 32, 2, 0.5
  g = torch.Generator().manual_seed(_seed(request))
  dims = [S] + [H] * depth + [2 * A]
  nets = [_draw_net(dims, g, gain=1.0) for _ in range(R)]
  rows = _rows(g, R, B, S, A)
  wo = py_row_layout(S, A)[0]['weights']
  use_in, use_hid = masks in ('in', 'both'), masks in ('hid', 'both')
  p_in, p_h = 0.21, 0.2
  m_in = _mask(g, (R, B, S), p_in) if use_in else None
  m_hid = [_mask(g, (R, B, H), p_h) if use_hid else None for _ in range(depth)]
  if act == 'relu':  # draw rows again whose ReLU input lies within KINK of 0
    for _ in range(100):
      bad = torch.zeros(R, B, dtype=torch.bool)
      for r in range(R):
        for z in _hidden_pre(nets[r], rows[r][:, :S], 'relu', m_in[r] if use_in else None, [mm[r] if use_hid else None for mm in m_hid]): bad[r] |= ((z.abs() < KINK) & (z != 0)).any(1)
      if not bad.any(): break
      k = int(bad.sum())
      rows[bad] = _rows(g, 1, k, S, A, zero_every=0)[0]
      if use_in: m_in[bad] = _mask(g, (k, S), p_in)
      for mm in m_hid:
        if mm is not None: mm[bad] = _mask(g, (k, H), p_h)
    else: raise AssertionError('could not draw a batch away from the ReLU kink')
  flat = Flat(nets, dims)
  mom, vel = torch.zeros_like(flat.buf), torch.zeros_like(flat.buf)
  step = torch.zeros(1, dtype=torch.int64, device=DEV)
  rdev, rs = _dev_rows(rows)
  mdev_in = m_in.float().to(DEV) if use_in else None
  mdev_hid = [mm.float().to(DEV) if mm is not None else None for mm in m_hid]
  loss = torch.full((R + 1, ), SENTINEL, device=DEV)
  a = L.BcArgs()
  a.actor, a.batch, a.R = flat.struct(act), _batch(rdev, rs, B, S, A), R
  _adam(a.opt, mom, vel, step, wd)
  a.out_loss = loss.data_ptr() if with_loss else None
  ws = Workspace(lib.il_actor_dropout_workspace_bytes(C.byref(a.actor), R, B))
  a.workspace, a.workspace_bytes = ws.t.data_ptr(), ws.need
  state = [flat.buf, mom, vel, step, loss]
  state0, inputs = [t.clone() for t in state], [t.clone() for t in [rdev] + ([mdev_in] if use_in else []) + [mm for mm in mdev_hid if mm is not None]]
  def setup():
    for t, t0 in zip(state, state0): t.copy_(t0)
    ws.fill()
  got = _launches(lambda: lib.il_bc_update_dropout(L.handle(), C.byref(a), L.ptr(mdev_in), L.mask_array(mdev_hid), L.stream(), None), setup)
  _assert_launches(got, dict(tick_kernel=1, input_mask_kernel=int(use_in), dropout_act_kernel=depth, dropout_bwd_kernel=depth, adam=1), only=True)
  assert int(step.item()) == 1
  for i, (t, t0) in enumerate(zip([rdev] + ([mdev_in] if use_in else []) + [mm for mm in mdev_hid if mm is not None], inputs)): assert torch.equal(t, t0), f'input {i} modified'
  ws.check_tail()
  for name, t in (('params', flat.buf), ('m', mom), ('v', vel)): flat.padding_zero(t, name)
  assert loss[R].item() == SENTINEL and (with_loss or (loss[:R] == SENTINEL).all()), 'loss slots written outside [R] (or without out_loss)'
  names = [f'{"Wb"[i % 2]}{i // 2}' for i in range(2 * (depth + 1))]
  for r in range(R):
    ref = []
    for dtype in (torch.float64, torch.float32):
      ps = [torch.nn.Parameter(t.to(dtype).clone()) for t in nets[r]]
      x = rows[r].to(dtype)
      pm = ([m_in[r].to(dtype)] if use_in else []) + ([mm[r].to(dtype) for mm in m_hid] if use_hid else [])
      l = port.behavioural_cloning_update(ps, _GradOnly(), dict(states=x[:, :S], actions=x[:, S:S + A], weights=x[:, wo]), act, input_dropout=p_in if use_in else 0.0,
                                          dropout=p_h if use_hid else 0.0, training=True, masks=pm)
      ref.append(([q.grad.detach().double() for q in ps], l.item()))
    if with_loss: _assert_vs_f64(loss[r].item(), ref[0][1], ref[1][1], f'loss replica {r}')
    m, v, prm = (flat.views(t, r) for t in (mom, vel, flat.buf))
    for i, name in enumerate(names):
      gr = _check_adamw(prm[i], m[i], v[i], nets[r][i], LR, wd, f'{name} replica {r}')
      _assert_vs_f64(gr.numpy(), ref[0][0][i].numpy(), ref[1][0][i].numpy(), f'd{name} replica {r} (B={B}, A={A})')


# ---- DRIL: il_dril_reward -----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('E,q_shared,with_reward,ld', [(2, 0, True, 1), (5, 1, True, 2), (5, 0, False, 1), (7, 0, True, 3), (7, 1, True, 1)])
def test_dril_reward_route(E, q_shared, with_reward, ld, request):
  L = _lib()
  lib = L.lib()
  R, B = 3, 300
  g = torch.Generator().manual_seed(_seed(request))
  lp = _f32(torch.randn(R, B * E, generator=g, dtype=torch.float64) * 0.7 - 1.0)
  var64 = lp.view(R, B, E).exp().var(dim=2)
  q = torch.quantile(var64, 0.6, dim=1)
  q = q[:1].expand(R).clone() if q_shared else q
  # no variance within 1e-4 (relative) of its threshold: a flipped comparison is then a kernel error
  near = (var64 - q[:, None]).abs() < 1e-4 * q[:, None]
  lp[near.repeat_interleave(E, 1)] -= 0.5
  lp = _f32(lp)
  lp_dev = lp.float().to(DEV)
  var64, var32 = lp.view(R, B, E).exp().var(dim=2), lp.float().view(R, B, E).exp().var(dim=2).double()
  assert not ((var64 - q[:, None]).abs() < 1e-4 * q[:, None]).any()
  q_dev = torch.tensor(q.numpy(), dtype=torch.float32, device=DEV)
  rs = B * ld + 3
  reward = torch.full((R * rs + 1, ), SENTINEL, device=DEV)
  variance = torch.full((R * B + 1, ), SENTINEL, device=DEV)
  lp0, q0 = lp_dev.clone(), q_dev.clone()
  def setup():
    reward.fill_(SENTINEL)
    variance.fill_(SENTINEL)
  call = lambda: lib.il_dril_reward(L.handle(), lp_dev.data_ptr(), R, B, E, q_dev.data_ptr() if with_reward else None, q_shared, reward.data_ptr() if with_reward else None, rs, ld,
                                    variance.data_ptr(), L.stream())
  _assert_launches(_launches(call, setup), dict(dril_reward_kernel=1))
  assert torch.equal(lp_dev, lp0) and torch.equal(q_dev, q0), 'an input was modified'
  assert variance[R * B].item() == SENTINEL, 'variance written past its R x B outputs'
  _assert_vs_f64(variance[:R * B].view(R, B).double().cpu().numpy(), var64.numpy(), var32.numpy(), f'variance (E = {E})')
  if not with_reward:
    assert (reward == SENTINEL).all(), 'reward written without a reward output'
    return
  written = torch.zeros_like(reward, dtype=torch.bool)
  for r in range(R):
    idx = r * rs + torch.arange(B, device=DEV) * ld
    written[idx] = True
    want = torch.where(var64[r] <= float(q_dev[0 if q_shared else r]), 1.0, -1.0)
    assert torch.equal(reward[idx].double().cpu(), want), f'replica {r}: {int((reward[idx].double().cpu() != want).sum())} rewards differ from the float64 variance test'
  assert (reward[~written] == SENTINEL).all(), 'reward gaps written'
  # a threshold equal to a row's own variance (read back from the device): var <= q holds, so that row gets +1
  row = 17
  v_dev = variance[:R * B].view(R, B)
  tie_q = v_dev[:, row].clone() if not q_shared else v_dev[:1, row].clone().expand(R).contiguous()
  reward.fill_(SENTINEL)
  L.check(lib.il_dril_reward(L.handle(), lp_dev.data_ptr(), R, B, E, tie_q.data_ptr(), q_shared, reward.data_ptr(), rs, ld, None, L.stream()))
  torch.cuda.synchronize()
  for r in range(R if not q_shared else 1):
    assert reward[r * rs + row * ld].item() == 1.0, f'replica {r}: the row whose variance equals q got {reward[r * rs + row * ld].item()} (models.py:117 uses less_equal)'


# ---- GMMIL ---------------------------------------------------------------------------------------------------------------------------------------
def gm(B, S, A, state_only=False, R=1, exact=False, weights='random', pad=4):
  d = S if state_only else S + A
  prm = dict(B=B, S=S, A=A, state_only=state_only, R=R, exact=exact, weights=weights, pad=pad)
  return pytest.param(prm, id=f'B{B}-d{d}-R{R}-{weights}' + ('-exact' if exact else '') + ('-state_only' if state_only else '') + (f'-pad{pad}' if pad != 4 else ''))


# exact rows: integer features with d a power of two (every D exact in fp32); random rows: the d edges 3, 15, 24, 119, 120 and 195
GMMIL_ROUTES = [
  gm(1, 13, 3, exact=True, weights='ones'), gm(2, 5, 3, exact=True, weights='ones'), gm(31, 13, 3, exact=True, weights='int'), gm(32, 24, 8, exact=True, weights='int'),
  gm(33, 5, 3, exact=True, weights='ones', R=3), gm(255, 5, 3, R=3, weights='int', exact=True), gm(256, 8, 3, state_only=True, exact=True, weights='ones'),
  gm(257, 13, 3, exact=True, weights='ones'), gm(300, 16, 3, state_only=True, exact=True, weights='int', pad=1001), gm(513, 16, 8, state_only=True, R=3, exact=True, weights='int'),
  gm(40, 2, 1, R=3), gm(33, 12, 3), gm(300, 12, 3, R=3, pad=1001), gm(96, 18, 6, weights='ones'), gm(257, 111, 8), gm(64, 112, 8), gm(64, 120, 8, state_only=True),
  gm(33, 187, 8),  # d = 195: the widest feature row the shared memory holds
]


def _exact_median(D, w_i, w_j):
  """Smallest element x of D with sum_{D_ij <= x} w_i w_j >= 0.5 sum w_i w_j (exact in float64 for the small-integer weights)."""
  W = torch.outer(w_i, w_j).flatten()
  s, idx = torch.sort(D.flatten(), stable=True)
  c = torch.cumsum(W[idx], 0)
  k = int(torch.nonzero(c >= 0.5 * W.sum())[0])
  return s[k].item(), s, k


@pytest.mark.parametrize('p', GMMIL_ROUTES)
def test_gmmil_route(p, request):
  from oracle import port
  from il_b200._lib import py_row_layout
  L = _lib()
  lib = L.lib()
  R, B, S, A = p['R'], p['B'], p['S'], p['A']
  d = S if p['state_only'] else S + A
  off, row = py_row_layout(S, A)
  g = torch.Generator().manual_seed(_seed(request))
  ints = p['exact']
  if ints: assert d & (d - 1) == 0, 'an exact row needs d a power of two'
  pol, exp = _rows(g, R, B, S, A, ints=ints, zero_every=0), _rows(g, R, B, S, A, ints=ints, zero_every=0)
  for x in (pol, exp):
    if p['weights'] == 'ones': x[..., off['weights']] = 1.0
    elif p['weights'] == 'int': x[..., off['weights']] = torch.randint(0, 3, (R, B), generator=g).double()
    else: x[..., off['weights']] = _f32(torch.rand(R, B, generator=g, dtype=torch.float64) + 0.25)
    x[:, ::5, off['weights']] = 0.0 if p['weights'] != 'ones' else 1.0
    x[..., off['weights']] += (x[..., off['weights']].sum(1, keepdim=True) == 0).double()  # never an all-zero batch
  pdev, rs = _dev_rows(pol, p['pad'])
  edev, _ = _dev_rows(exp, p['pad'])
  pb, eb = _batch(pdev, rs, B, S, A), _batch(edev, rs, B, S, A)
  need = lib.il_gmmil_workspace_bytes(R, B)
  ws = Workspace(need)
  gamma = torch.full((R * 2 + 2, ), SENTINEL, device=DEV)
  inputs = [pdev.clone(), edev.clone()]
  def setup():
    ws.fill()
    gamma.fill_(SENTINEL)
  call = lambda: lib.il_gmmil_bandwidth(L.handle(), R, C.byref(pb), C.byref(eb), int(p['state_only']), gamma.data_ptr(), ws.t.data_ptr(), need, L.stream())
  _assert_launches(_launches(call, setup), dict(gmmil_kernel=2, weighted_median_kernel=2))
  assert torch.equal(pdev, inputs[0]) and torch.equal(edev, inputs[1]), 'a batch was modified'
  ws.check_tail()
  assert (gamma[2 * R:] == SENTINEL).all(), 'gamma written past its [R, 2] slots'
  gam = gamma[:2 * R].view(R, 2).double().cpu()
  feats = lambda x, r: x[r][:, :d]
  for r in range(R):
    wp, we = pol[r][:, off['weights']], exp[r][:, off['weights']]
    for col, (xi, wi) in enumerate(((pol, wp), (exp, we))):
      D64 = port.squared_distance_mean(feats(xi, r), feats(exp, r))
      assert D64.dtype == torch.float64
      med, s, k = _exact_median(D64, wi, we)
      want = float(np.float32(1 / (med + 1e-8)))
      if p['exact']:  # integer features, d a power of two or a sum of exactly representable squares: D is exact in fp32
        assert torch.equal(D64.float().double(), D64)
        assert gam[r, col].item() == want, f'replica {r} gamma_{col + 1}: {gam[r, col].item()!r}, (float)(1 / (median + 1e-8)) = {want!r} under the exact rule'
        if p['weights'] == 'ones':  # equal weights: the reference's float32 rule picks the same element
          assert port.weighted_median(D64.float(), torch.outer(wi, we).float()).item() == med
      else:  # the device's median is the exact-rule element up to eps, a bound on the relative fp32 error of a mean of d squares
        eps = 2 * (d + 8) * U
        m = 1 / gam[r, col].item() - 1e-8
        W = torch.outer(wi, we).flatten()
        half = 0.5 * W.sum().item()
        below, upto = W[D64.flatten() < m * (1 - eps)].sum().item(), W[D64.flatten() <= m * (1 + eps)].sum().item()
        assert below < half <= upto, f'replica {r} gamma_{col + 1}: 1 / gamma - 1e-8 = {m!r} holds weight {below}..{upto} below it, half the total is {half} (median {med!r})'

  # reward with the device's own bandwidths, strided
  ld = 2
  rrs = B * ld + 3
  reward = torch.full((R * rrs + 1, ), SENTINEL, device=DEV)
  gamma_in = gamma[:2 * R].clone()
  call = lambda: lib.il_gmmil_reward(L.handle(), R, C.byref(pb), C.byref(eb), int(p['state_only']), gamma_in.data_ptr(), reward.data_ptr(), rrs, ld, L.stream())
  _assert_launches(_launches(call, lambda: reward.fill_(SENTINEL)), dict(gmmil_kernel=1))
  assert torch.equal(pdev, inputs[0]) and torch.equal(edev, inputs[1]), 'a batch was modified'
  written = torch.zeros_like(reward, dtype=torch.bool)
  for r in range(R):
    idx = r * rrs + torch.arange(B, device=DEV) * ld
    written[idx] = True
    ref = []
    for dtype in (torch.float64, torch.float32):
      disc = port.GmmilDiscriminator(p['state_only'])
      disc.gamma_1, disc.gamma_2 = gam[r, 0].item(), gam[r, 1].item()
      x, y = pol[r].to(dtype), exp[r].to(dtype)
      ref.append(disc.predict_reward(x[:, :S], x[:, S:S + A], y[:, :S], y[:, S:S + A], x[:, off['weights']], y[:, off['weights']]).double().numpy())
    _assert_vs_f64(reward[idx].double().cpu().numpy(), ref[0], ref[1], f'GMMIL reward replica {r}')
  assert (reward[~written] == SENTINEL).all(), 'reward gaps written'


# ---- PWIL ------------------------------------------------------------------------------------------------------------------------------------------
def pw(N, T, S=12, A=3, state_only=False, calls=3, exact=True, dup=False, active=None, per_replica=False, R=2):
  d = S if state_only else S + A
  prm = dict(N=N, T=T, S=S, A=A, state_only=state_only, calls=calls, exact=exact, dup=dup, active=active, per_replica=per_replica, R=len(active) if active else R)
  tags = [f'N{N}', f'T{T}', f'd{d}', f'calls{calls}', 'exact' if exact else 'random'] + (['dup'] if dup else []) + (['active'] if active else []) + (['per_replica'] if per_replica else [])
  return pytest.param(prm, id='-'.join(tags) + ('-state_only' if state_only else ''))


PWIL_ROUTES = [
  pw(1, 3, calls=4),                      # T > N: part of the one atom per call, then the atoms run out
  pw(3, 2, calls=4),                      # T < N: whole atoms and a partial one, then the break
  pw(255, 255, calls=6),                  # T = N: every call partial, ~1e-6 of the atom left behind
  pw(256, 1000, calls=5, dup=True),
  pw(257, 64, calls=6, state_only=True, active=[1, 0, 1]),
  pw(4097, 1000, calls=4, dup=True, per_replica=True, R=3),
  pw(4097, 300, S=112, A=8, calls=3, exact=False),
  pw(25000, 1000, calls=3, dup=True),
  pw(25000, 25000, S=17, A=6, calls=2, exact=False),
  pw(PWIL_SMEM_FLOATS - 15, 1000, calls=2, dup=True),   # the shared-memory maximum N = 56 320 - d
]


def _pwil_state(g, p, exact):
  N, S, A = p['N'], p['S'], p['A']
  d = S if p['state_only'] else S + A
  if exact: atoms = torch.randint(-4, 5, (N, d), generator=g).double()
  else: atoms = _f32(torch.randn(N, d, generator=g, dtype=torch.float64))
  return atoms, d


@pytest.mark.parametrize('p', PWIL_ROUTES)
def test_pwil_route(p, request):
  from oracle import port
  L = _lib()
  lib = L.lib()
  R, N, T, S, A = p['R'], p['N'], p['T'], p['S'], p['A']
  g = torch.Generator().manual_seed(_seed(request))
  raw, d = _pwil_state(g, p, p['exact'])
  raw = raw.float()
  if p['exact']: scale, offset = torch.ones(d), torch.zeros(d)
  else: scale, offset = 1 / (raw.std(0) + 0.1), -raw.mean(0)
  # the agent's (state, action) of every call and replica; with dup the first call's nearest atom is repeated across strides and warps
  queries = []
  for _ in range(p['calls']):
    if p['exact']: queries.append(torch.randint(-4, 5, (R, d), generator=g).float())
    else: queries.append((raw[torch.randint(0, N, (R, ), generator=g)].double() + 0.3 * torch.randn(R, d, generator=g, dtype=torch.float64)).float())
  if p['dup']:
    for i in (i for i in (N - 1, 2 * 256 + 37, 700, 256 + 3, 5) if i < N): raw[i] = queries[0][0]
  bw32 = [float(np.float32(5.0 * T / math.sqrt(d) * f)) for f in ((1.0, 0.5, 2.0)[:R] if p['per_replica'] else (1.0, ) * R)]
  rscale = [float(np.float32(5.0 * f)) for f in ((1.0, 0.25, 3.0)[:R] if p['per_replica'] else (1.0, ) * R)]
  # one port per replica on the same atoms, in float32 as the reference runs, with the row's scale and offset in place of its data statistics
  ports = []
  for r in range(R):
    pd = port.PwilDiscriminator(raw[:, :S], raw[:, S:] if not p['state_only'] else None, T, state_only=p['state_only'])
    pd.scale, pd.offset, pd.reward_scale, pd.reward_bandwidth = scale[None], offset[None], rscale[r], bw32[r]
    pd.reset()
    ports.append(pd)
  atoms = ports[0].atoms
  if p['exact']: assert torch.equal(atoms, raw)
  adev, sdev, odev = atoms.float().to(DEV).contiguous(), scale.float().to(DEV), offset.float().to(DEV)
  wdev = torch.full((R, N), SENTINEL, device=DEV)
  st = L.Pwil()
  st.atoms, st.scale, st.offset, st.weights, st.N, st.d, st.S, st.A = adev.data_ptr(), sdev.data_ptr(), odev.data_ptr(), wdev.data_ptr(), N, d, S, A
  st.state_only, st.time_horizon, st.reward_scale, st.reward_bandwidth = int(p['state_only']), T, rscale[0], bw32[0]
  if p['per_replica']:
    rs_r, bw_r = torch.tensor(rscale, dtype=torch.float32, device=DEV), torch.tensor(bw32, dtype=torch.float32, device=DEV)
    st.reward_scale_r, st.reward_bandwidth_r = rs_r.data_ptr(), bw_r.data_ptr()
  _assert_launches(_launches(lambda: lib.il_pwil_reset(L.handle(), C.byref(st), R, None, L.stream()), lambda: wdev.fill_(SENTINEL)), dict(pwil_reset_kernel=1))
  assert torch.equal(wdev, torch.full_like(wdev, float(np.float32(1) / np.float32(N)))), 'reset: weights are not 1 / N'
  active = torch.tensor(p['active'], dtype=torch.int32, device=DEV) if p['active'] else None
  live = [r for r in range(R) if not p['active'] or p['active'][r]]
  inputs0 = [adev.clone(), sdev.clone(), odev.clone()]
  for c, q in enumerate(queries):
    state, action = q[:, :S].to(DEV).contiguous(), (q[:, S:] if not p['state_only'] else torch.zeros(R, A)).to(DEV).contiguous()
    reward = torch.full((R + 1, ), SENTINEL, device=DEV)
    w_before = wdev.clone()
    def setup():
      wdev.copy_(w_before)
      reward.fill_(SENTINEL)
    call = lambda: lib.il_pwil_reward(L.handle(), C.byref(st), R, state.data_ptr(), action.data_ptr(), reward.data_ptr(), L.ptr(active), L.stream())
    _assert_launches(_launches(call, setup), dict(pwil_reward_kernel=1))
    for t, t0 in zip((adev, sdev, odev), inputs0): assert torch.equal(t, t0), f'call {c}: atoms / scale / offset modified'
    assert reward[R].item() == SENTINEL, 'reward written past its R slots'
    for r in range(R):
      what = f'call {c} replica {r}'
      if r not in live:
        assert torch.equal(wdev[r], w_before[r]) and reward[r].item() == SENTINEL, f'{what}: an inactive replica was written'
        continue
      pd = ports[r]
      agent = q[r:r + 1]
      dists = torch.linalg.norm(pd.atoms - pd.scale * (agent + pd.offset), dim=1)
      if not p['exact']:  # the atoms this call consumes are clear of their neighbours by 1e-5 (relative): far above the fp32 distance error
        dd = torch.sort(torch.linalg.norm(pd.atoms.double() - (pd.scale * (agent + pd.offset)).double(), dim=1)).values
        n_take = min(dd.numel() - 1, int(math.ceil(N / T)) + 1)
        assert n_take <= 0 or ((dd[1:n_take + 1] - dd[:n_take]) > 1e-5 * dd[n_take]).all(), f'{what}: an argmin gap lies within the margin (draw another seed)'
      cost = None
      if float(pd.weights.double().sum()) < 1 / T - 1e-6:
        # the atoms run out in this call: the device breaks out of its loop; the reference would take the argmin of an empty tensor and fail
        cost = float((pd.weights.double() * dists.double()).sum())
        pd.atoms, pd.weights = pd.atoms[:0], pd.weights[:0]
        want = pd.reward_scale * math.exp(-pd.reward_bandwidth * cost)
      else:
        want = pd.compute_reward(agent[:, :S], agent[:, S:])
        cost = -math.log(want / pd.reward_scale) / pd.reward_bandwidth
      w = wdev[r].cpu()
      kept = w[w >= 0]
      assert (w[w < 0] == -1).all(), f'{what}: a consumed atom holds {w[w < 0][w[w < 0] != -1][:3].tolist()} instead of -1'
      assert torch.equal(kept, pd.weights), (f'{what}: {kept.numel()} live atoms on the device, {pd.weights.numel()} in the port; first differing weights '
                                              f'{[(a, b) for a, b in zip(kept.tolist(), pd.weights.tolist()) if a != b][:3]}')
      got = reward[r].item()
      # the device holds the bandwidth in fp32 (the port takes it as given here) and may fuse the cost's multiply-adds: ~1e-7 of bandwidth x cost
      bound = 4 * float(_ulp32(torch.tensor([want]))[0]) + 1e-6 * abs(want) * (1 + pd.reward_bandwidth * cost)
      assert abs(got - want) <= bound, f'{what}: reward {got!r}, port {want!r}'
  # a masked reset restores exactly the masked replicas
  mask = torch.tensor([r % 2 for r in range(R)], dtype=torch.int32, device=DEV)
  before = wdev.clone()
  L.check(lib.il_pwil_reset(L.handle(), C.byref(st), R, mask.data_ptr(), L.stream()))
  torch.cuda.synchronize()
  for r in range(R):
    want = torch.full_like(before[r], float(np.float32(1) / np.float32(N))) if r % 2 else before[r]
    assert torch.equal(wdev[r], want), f'masked reset: replica {r} ({"reset" if r % 2 else "kept"})'


# ---- refused calls ------------------------------------------------------------------------------------------------------------------------------
def _refused(call, text, outputs):
  import il_b200
  L = _lib()
  before, snap = il_b200.launch_count(), [t.clone() for t in outputs]
  rc = call()
  torch.cuda.synchronize()
  assert rc != 0, 'the call was accepted'
  assert text in L.last_error(), L.last_error()
  assert il_b200.launch_count() == before, 'a refused call launched a kernel'
  for t, t0 in zip(outputs, snap): assert torch.equal(t.nan_to_num(), t0.nan_to_num()) and torch.equal(t.isnan(), t0.isnan()), 'a refused call wrote an output'


def _red_refusal_device(R=2):
  pb = RedProblem(red_upd(B=16, H=32, depth=2, act='tanh', masks='both', R=R).values[0], 3)
  dv = RedDevice(pb)
  dv.workspace()
  return dv


@pytest.mark.parametrize('what', ['embedding_dims', 'workspace_one_byte_short', 'activation_r_past_grid'])
def test_red_update_refused(what):
  L = _lib()
  dv = _red_refusal_device()
  dv.act_r = torch.zeros(2, dtype=torch.int32, device=DEV)
  a = dv.update_args()
  text = {'embedding_dims': 'embedding networks must map', 'workspace_one_byte_short': 'bad optimiser state / workspace', 'activation_r_past_grid': 'per-replica activations need'}[what]
  if what == 'embedding_dims': a.batch.S, a.batch.row = a.batch.S - 1, _lib().py_row_layout(a.batch.S - 1, a.batch.A)[1]
  if what == 'workspace_one_byte_short': a.workspace_bytes -= 1
  if what == 'activation_r_past_grid': a.R = 65536
  _refused(lambda: L.lib().il_red_update(L.handle(), C.byref(a), L.stream()), text, dv._state() + [dv.ws.t])


@pytest.mark.parametrize('entry', ['sigma', 'reward'])
def test_red_sigma_and_reward_refused(entry):
  L = _lib()
  lib = L.lib()
  dv = _red_refusal_device()
  d, b = dv.disc(), dv.batch()
  reward = torch.full((2, 16), SENTINEL, device=DEV)
  for text, S, need in (('workspace too small', S0, dv.ws.need - 1), ('embedding networks must map', S0 + 1, dv.ws.need)):
    bb = _batch(dv.rows, dv.rs, 16, S, A0)
    if entry == 'sigma': call = lambda: lib.il_red_sigma(L.handle(), C.byref(d), 2, C.byref(bb), L.ptr(dv.m_in), L.mask_array(dv.m_hid), dv.ws.t.data_ptr(), need, L.stream())
    else: call = lambda: lib.il_red_reward(L.handle(), C.byref(d), 2, C.byref(bb), reward.data_ptr(), 16, 1, dv.ws.t.data_ptr(), need, L.stream())
    _refused(call, text, [dv.sigma, reward, dv.ws.t])


def test_actor_and_dril_refused():
  L = _lib()
  lib = L.lib()
  R, S, A, n = 2, S0, A0, 10
  flat = Flat([_draw_net([S, 32, 2 * A], torch.Generator().manual_seed(1)) for _ in range(R)], [S, 32, 2 * A])
  m = flat.struct('tanh')
  ws = Workspace(lib.il_actor_dropout_workspace_bytes(C.byref(m), R, n))
  states, actions, out = torch.zeros(R, n, S, device=DEV), torch.zeros(R, n, A, device=DEV), torch.full((R, n), SENTINEL, device=DEV)
  _refused(lambda: lib.il_actor_log_prob_dropout(L.handle(), C.byref(m), R, n, 3, states.data_ptr(), n * S, S, actions.data_ptr(), None, L.mask_array([]), out.data_ptr(),
                                                 ws.t.data_ptr(), ws.need, L.stream(), None), 'il_actor_log_prob_dropout: bad argument', [out, ws.t])
  lp, q, reward, var = torch.zeros(R, n), torch.zeros(R, device=DEV), torch.full((R, n), SENTINEL, device=DEV), torch.full((R, n), SENTINEL, device=DEV)
  lp = lp.to(DEV)
  _refused(lambda: lib.il_dril_reward(L.handle(), lp.data_ptr(), R, n, 1, q.data_ptr(), 0, reward.data_ptr(), n, 1, var.data_ptr(), L.stream()), 'il_dril_reward: bad argument',
           [reward, var])


@pytest.mark.parametrize('what', ['d196', 'shape_mismatch'])
def test_gmmil_refused(what):
  L = _lib()
  lib = L.lib()
  B, R = 8, 1
  S, A = (188, 8) if what == 'd196' else (12, 3)
  g = torch.Generator().manual_seed(2)
  pdev, rs = _dev_rows(_rows(g, R, B, S, A))
  edev, _ = _dev_rows(_rows(g, R, B + 1, S, A))
  pb, eb = _batch(pdev, rs, B, S, A), _batch(edev, rs, B if what == 'd196' else B + 1, S, A)
  need = lib.il_gmmil_workspace_bytes(R, B + 1)
  ws = Workspace(need)
  gamma, reward = torch.full((2 * R, ), SENTINEL, device=DEV), torch.full((R, B), SENTINEL, device=DEV)
  text = 'feature width 196 too large' if what == 'd196' else 'policy/expert batch shape mismatch'
  _refused(lambda: lib.il_gmmil_bandwidth(L.handle(), R, C.byref(pb), C.byref(eb), 0, gamma.data_ptr(), ws.t.data_ptr(), need, L.stream()), text, [gamma, ws.t])
  _refused(lambda: lib.il_gmmil_reward(L.handle(), R, C.byref(pb), C.byref(eb), 0, gamma.data_ptr(), reward.data_ptr(), B, 1, L.stream()), text, [reward])
  if what == 'd196':  # one feature fewer fits: d = 195
    pdev, rs = _dev_rows(_rows(g, R, B, 187, 8))
    pb = eb = _batch(pdev, rs, B, 187, 8)
    L.check(lib.il_gmmil_bandwidth(L.handle(), R, C.byref(pb), C.byref(eb), 0, gamma.data_ptr(), ws.t.data_ptr(), need, L.stream()))
    torch.cuda.synchronize()
    assert torch.isfinite(gamma).all()


@pytest.mark.parametrize('what', ['N_past_shared_memory', 'd_not_S_plus_A', 'd_not_S_state_only'])
def test_pwil_refused(what):
  L = _lib()
  lib = L.lib()
  R, S, A = 2, S0, A0
  d = S if what == 'd_not_S_state_only' else S + A
  N = PWIL_SMEM_FLOATS - d + 1 if what == 'N_past_shared_memory' else 16
  atoms = torch.zeros(N, d, device=DEV)
  sc, of = torch.ones(d, device=DEV), torch.zeros(d, device=DEV)
  w = torch.full((R, N), 0.5, device=DEV)
  st = L.Pwil()
  st.atoms, st.scale, st.offset, st.weights, st.N, st.S, st.A = atoms.data_ptr(), sc.data_ptr(), of.data_ptr(), w.data_ptr(), N, S, A
  st.state_only, st.time_horizon, st.reward_scale, st.reward_bandwidth = int(what == 'd_not_S_state_only'), 100, 5.0, 1.0
  st.d = d if what == 'N_past_shared_memory' else d + 1
  state, action, reward = torch.zeros(R, S, device=DEV), torch.zeros(R, A, device=DEV), torch.full((R, ), SENTINEL, device=DEV)
  text = 'do not fit in shared memory' if what == 'N_past_shared_memory' else 'inconsistent with S='
  _refused(lambda: lib.il_pwil_reward(L.handle(), C.byref(st), R, state.data_ptr(), action.data_ptr(), reward.data_ptr(), None, L.stream()), text, [w, reward])
  if what == 'N_past_shared_memory':  # one atom fewer fits
    st.N = N - 1
    L.check(lib.il_pwil_reward(L.handle(), C.byref(st), R, state.data_ptr(), action.data_ptr(), reward.data_ptr(), None, L.stream()))
    torch.cuda.synchronize()
