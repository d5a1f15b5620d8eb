"""Every branch of the general GAIL discriminator program (csrc/gail_general.cu: il_gailx_update, il_gailx_reward) against float64.

The general program runs every discriminator configuration the fused kernels do not: any depth (0 to 5 hidden layers) and activation, reward
shaping (a linear g plus a shaping MLP h), the log-policy term, with every loss, gradient penalty, entropy bonus and spectral norm. Each row
of the route table is one such configuration; the kernels it must launch follow from it:
- one sn_access_kernel per spectral-norm access (g once per pass, h twice: h(s') then h(s)), one mix_batch_kernel per mixed batch;
- in the gradient-penalty pass, per net: gp_linear_gx_kernel for a linear net, else gp_top_kernel, L - 2 gp_mask_kernel launches, L - 1
  gp_second_kernel launches and, with a tanh / sigmoid activation, L - 2 add_kernel launches (the second-derivative chain zbar).
For every update row the test checks
- the launches, counted per kernel from a CUDA-activity `torch.profiler` trace;
- the gradient: one update from zero AdamW moments leaves m = (1 - beta1) g and v = (1 - beta2) g^2; g of every g and h parameter is compared
  with the float64 autograd gradient of oracle.port.gail_update (which pins the reference), v with g^2;
- the parameters: the AdamW formula on the kernel's own m and v within a few ulp; the step counter advances by one;
- both losses, and the spectral-norm u and v of every layer of g and h after all of the call's accesses (the unused h(s') of the
  gradient-penalty pass included);
- the bounds: the zero padding of the flat parameter buffer stays exactly zero in the parameters, m and v; the u / v slots past each net's
  vectors, the inputs and a 4 KB tail past the workspace stay untouched. The workspace is filled with NaN before every call, so a read before
  a write shows up in the outputs.
Reward rows check logits and every reward function in eval mode with the same bounds; refusal rows check that a bad call writes nothing.
Values use the tolerance of the MLP head tests: per output tensor, 8 max|port in fp32 on the CPU - float64| + 1e-6 max|float64|. Batch rows
whose float64 ReLU pre-activation lies within 1e-4 of the kink in any differentiated pass are drawn again, and every PUGAIL row asserts that
its clamp is at least 1e-3 from -margin (and active where the row says so), so a mask flip is never mistaken for a kernel error.
"""
import ctypes as C
import math
import zlib
from collections import Counter
from itertools import product

import numpy as np
import pytest
import torch

from test_gpu_gail_routes import ADAM_EPS, BETAS, CLAMP_GAP, DEV, ENV, KINK, LR, PRIOR, SENTINEL, U, WD, _GradOnly, _ulp32
from test_gpu_gemm_routes import _assert_vs_f64, kernels_of

pytestmark = pytest.mark.gpu

DISCOUNT = float(np.float32(0.97))
LOSSES = ('BCE', 'PUGAIL', 'PUGAILm', 'Mixup')  # PUGAIL: margin inf; PUGAILm: margin 0.05 with the clamp active
MARGIN = {'PUGAIL': float('inf'), 'PUGAILm': 0.05}
WS_TAIL = 4096  # bytes of SENTINEL past the workspace
ACTS = ('relu', 'tanh', 'sigmoid')


# ---- the route table ------------------------------------------------------------------------------------------------------------------
def upd(env='hopper', H=64, B=64, depth=2, act='tanh', shaping=False, loss='BCE', gp=1.0, ent=0.0, sn=True, logp=False, state_only=False, R=2,
        per_replica=None, S=None, A=None):
  """One il_gailx_update problem. depth: hidden layers of g (no shaping) or of h (shaping; g is then linear). per_replica: the [R] value
  arrays the call passes ('ent', 'discount', 'lr_wd', 'gp')."""
  S, A = (S, A) if S is not None else ENV[env]
  p = dict(kind='update', S=S, A=A, H=H, B=B, depth=depth, act=act, shaping=shaping, loss=loss, gp=gp, ent=ent, sn=sn, logp=logp, state_only=state_only,
           R=R, per_replica=per_replica or ())
  d = S if state_only else S + A
  net = f'h{depth}' if shaping else f'g{depth}'
  tags = [env or f'S{S}A{A}', f'd{d}', f'H{H}', f'B{B}', net + (act if depth else ''), loss, f'gp{gp:g}', f'ent{ent:g}', 'sn' if sn else 'nosn']
  if logp: tags.append('logp')
  if state_only: tags.append('state_only')
  tags += [f'{k}_r' for k in p['per_replica']]
  return pytest.param(p, id='-'.join(tags))


def rew(env='hopper', H=64, B=64, depth=2, act='tanh', shaping=False, rf='AIRL', sn=True, logp=False, ld=1, logits=True, R=2):
  S, A = ENV[env]
  p = dict(kind='reward', S=S, A=A, H=H, B=B, depth=depth, act=act, shaping=shaping, rf=rf, sn=sn, logp=logp, state_only=False, ld=ld, logits=logits, R=R,
           loss='BCE', gp=0.0, ent=0.0, per_replica=())
  net = f'h{depth}' if shaping else f'g{depth}'
  tags = [env, f'd{S + A}', f'H{H}', f'B{B}', net + (act if depth else ''), rf, 'sn' if sn else 'nosn', f'ld{ld}'] + (['logp'] if logp else []) + ([] if logits else ['nologits'])
  return pytest.param(p, id='reward-' + '-'.join(tags))


PRODUCT = list(product(LOSSES, (0.0, 1.0), (0.0, 0.05), (False, True)))  # loss x gradient penalty x entropy bonus x spectral norm


def _opts(i):
  """A spread of loss, entropy bonus and spectral norm for the structure rows (they all take the gradient-penalty pass)."""
  loss, _, ent, sn = PRODUCT[(11 * i + 5) % len(PRODUCT)]
  return dict(loss=loss, ent=ent, sn=sn)


def _route_table():
  t = []
  # structure without shaping: g of depth 0 (linear: gp_linear_gx_kernel, gp_kappa_colsum_kernel with kappa = 1), 1 (gp_top_kernel, zbar without
  # add_kernel), 2, 3 and 5 (the middle branch of the double backward and gp_mask_kernel more than once)
  i = 0
  for depth in (0, 1, 2, 3, 5):
    for act in (ACTS if depth else ('relu', )):
      t.append(upd(depth=depth, act=act, **_opts(i)))
      i += 1
  # structure with shaping: linear g + h of depth 0 (the accumulating gp_linear_gx_kernel), 1 and 2, kappa = -(1 - t) on h(s)
  for depth in (0, 1, 2):
    for act in ACTS:
      t.append(upd(depth=depth, act=act, shaping=True, **_opts(i)))
      i += 1
  # the full option product on two anchors: depth-2 tanh g on hopper at H = 64, B = 256; shaping with a depth-1 tanh h and the log-policy term on
  # halfcheetah at H = 128, B = 512
  for loss, gp, ent, sn in PRODUCT:
    t.append(upd('hopper', 64, 256, 2, 'tanh', False, loss, gp, ent, sn))
    t.append(upd('halfcheetah', 128, 512, 1, 'tanh', True, loss, gp, ent, sn, logp=True))
  # shape edges: B (1, not a multiple of the 256-thread blocks, the published 1024), H, d (Ant: 120), state-only (no gradient penalty)
  t += [
    upd(B=1, depth=2, act='relu'),
    upd(B=33, depth=3, act='sigmoid', loss='Mixup'),
    upd(B=257, depth=2, act='tanh', shaping=True, loss='PUGAILm'),
    upd(B=1024, depth=2, act='relu', ent=0.05),
    upd(H=32, depth=2, act='sigmoid', B=100),
    upd(H=128, depth=3, act='tanh', B=128, loss='Mixup'),
    upd(H=128, depth=1, act='relu', shaping=True, B=96, sn=False),
    upd('halfcheetah', 64, 256, 2, 'relu', loss='PUGAIL', ent=0.05),
    upd('ant', 64, 256, 2, 'tanh', loss='Mixup'),
    upd('ant', 128, 128, 1, 'sigmoid', shaping=True, loss='BCE', ent=0.05),
    upd('ant', 32, 64, 0, 'relu', sn=False),
    upd('halfcheetah', 64, 64, 2, 'sigmoid', gp=0.0, state_only=True, loss='Mixup', ent=0.05),
    upd('hopper', 64, 64, 1, 'tanh', shaping=True, gp=0.0, state_only=True),
    upd('ant', 128, 48, 3, 'relu', gp=0.0, state_only=True, loss='PUGAILm'),
  ]
  # the log-policy term with every loss (Mixup through logp_mix), with and without shaping
  for shaping, loss in product((False, True), ('BCE', 'PUGAILm', 'Mixup')):
    t.append(upd(depth=2 - shaping, act='tanh', shaping=shaping, loss=loss, logp=True, ent=0.05))
  # per-replica values, every replica against its own float64 update (grad_penalty_r stays > 0: the program keeps the penalty pass uniform)
  t += [
    upd(depth=2, act='tanh', R=3, per_replica=('ent', ), ent=0.05),
    upd(depth=1, act='sigmoid', shaping=True, R=3, per_replica=('discount', ), loss='Mixup'),
    upd(depth=3, act='relu', R=3, per_replica=('lr_wd', ), loss='PUGAIL'),
    upd(depth=2, act='tanh', shaping=True, R=3, per_replica=('gp', ), logp=True),
  ]
  # il_gailx_reward: every reward function, with and without shaping and spectral norm, then the log-policy term, a strided output, no logits and B
  for rf, shaping, sn in product(('AIRL', 'GAIL', 'FAIRL'), (False, True), (False, True)):
    t.append(rew(depth=2 - shaping, act='tanh', shaping=shaping, rf=rf, sn=sn, ld=1 + sn))
  t += [
    rew(depth=1, act='tanh', shaping=True, rf='AIRL', logp=True, ld=2),
    rew(depth=3, act='sigmoid', rf='FAIRL', logp=True),
    rew(depth=2, act='relu', rf='GAIL', logits=False, ld=2),
    rew(depth=0, act='relu', rf='AIRL', B=1),
    rew('ant', 128, 257, depth=2, act='tanh', shaping=True, rf='GAIL', ld=2),
  ]
  return t


ROUTES = _route_table()


# ---- problems ---------------------------------------------------------------------------------------------------------------------------
def _dims(p):
  """Layer widths of g and h (None without shaping)."""
  d = p['S'] if p['state_only'] else p['S'] + p['A']
  hid = [p['H']] * p['depth']
  return ([d, 1], [p['S']] + hid + [1]) if p['shaping'] else ([d] + hid + [1], None)


def _normalise(x): return x / x.norm()


def _f32(t): return t.float().double()


def _act(x, act): return torch.relu(x) if act == 'relu' else (torch.tanh(x) if act == 'tanh' else torch.sigmoid(x))


def _draw_net(dims, g):
  """[W0, b0, W1, b1, ...] and the spectral-norm (u, v) of every layer (fp32 values held in float64), not converged."""
  params, sn = [], []
  for l in range(len(dims) - 1):
    n_in, n_out = dims[l], dims[l + 1]
    params += [_f32(1.5 * torch.randn(n_out, n_in, generator=g, dtype=torch.float64) / n_in ** 0.5), _f32(0.1 * torch.randn(n_out, generator=g, dtype=torch.float64))]
    sn.append(tuple(_f32(_normalise(torch.randn(n, generator=g, dtype=torch.float64))) for n in (n_out, n_in)))
  return params, sn


def _accesses(params, sn, n, use_sn, training=True):
  """Effective parameters of n successive spectral-norm accesses (train mode: one power iteration each), float64."""
  vecs, out = [(u.clone(), v.clone()) for u, v in sn], []
  for _ in range(n):
    eff = []
    for l in range(len(params) // 2):
      W = params[2 * l]
      if use_sn:
        u, v = vecs[l]
        if training:
          u = _normalise(W @ v)
          v = _normalise(W.t() @ u)
          vecs[l] = (u, v)
        W = W / (u @ W @ v)
      eff += [W, params[2 * l + 1]]
    out.append(eff)
  return out


def _forward(eff, x, act):
  """Hidden pre-activations and the output of one MLP evaluation."""
  zs = []
  L = len(eff) // 2
  for l in range(L):
    x = x @ eff[2 * l].t() + eff[2 * l + 1]
    if l < L - 1:
      zs.append(x)
      x = _act(x, act)
  return zs, x[:, 0]


class Problem:
  """Parameters, spectral-norm vectors, batches, noise, actors and per-replica values of one row (CPU float64 holding fp32 values)."""

  def __init__(self, p, seed):
    from il_b200._lib import py_row_layout
    self.p, R, S, A, B = p, p['R'], p['S'], p['A'], p['B']
    self.d = S if p['state_only'] else S + A
    self.off, self.row = py_row_layout(S, A)
    self.g_dims, self.h_dims = _dims(p)
    self.gen = torch.Generator().manual_seed(seed)
    self.g = [_draw_net(self.g_dims, self.gen) for _ in range(R)]
    self.h = [_draw_net(self.h_dims, self.gen) for _ in range(R)] if self.h_dims else None
    # small actors: log pi(a|s) of a few units, so that the discriminator logits stay away from sigmoid saturation
    self.actor = [[0.3 * t for t in _draw_net([S, 32, 32, 2 * A], self.gen)[0]] for _ in range(R)] if p['logp'] else None
    self.pol, self.exp = self._rows(R, B), self._rows(R, B)
    self.eps_gp, self.eps_mix = self._unit(R, B), self._unit(R, B)
    f32 = lambda xs: [float(np.float32(x)) for x in xs]
    pr = p['per_replica']
    self.ent_r = f32([0.0, 0.05, 0.3]) if 'ent' in pr else None
    self.discount_r = f32([0.9, 0.97, 0.995]) if 'discount' in pr else None
    self.lr_r, self.wd_r = ([3e-4, 1e-3, 2e-3], [0.0, 0.1, 10.0]) if 'lr_wd' in pr else (None, None)
    self.gp_r = f32([0.25, 1.0, 2.0]) if 'gp' in pr else None

  def _rows(self, *shape):
    o = self.off
    x = torch.randn(*shape, self.row, generator=self.gen, dtype=torch.float64)
    A = self.p['A']
    x[..., o['actions']:o['actions'] + A] = 0.9 * torch.tanh(x[..., o['actions']:o['actions'] + A])  # away from the atanh clamp of the log-policy
    x[..., o['terminals']] = (torch.rand(*shape, generator=self.gen, dtype=torch.float64) < 0.25).double()
    x[..., o['weights']] = torch.rand(*shape, generator=self.gen, dtype=torch.float64) + 0.5
    return _f32(x)

  def _unit(self, *shape): return _f32(torch.rand(*shape, generator=self.gen, dtype=torch.float64))

  # per-replica hyper-parameters
  def discount(self, r): return self.discount_r[r] if self.discount_r else DISCOUNT
  def ent(self, r): return self.ent_r[r] if self.ent_r else self.p['ent']
  def gp(self, r): return self.gp_r[r] if self.gp_r else self.p['gp']
  def lr(self, r): return self.lr_r[r] if self.lr_r else LR
  def wd(self, r): return self.wd_r[r] if self.wd_r else WD

  def fields(self, rows):
    o, S, A = self.off, self.p['S'], self.p['A']
    return dict(states=rows[:, :S], actions=rows[:, S:S + A], next_states=rows[:, o['next_states']:o['next_states'] + S], terminals=rows[:, o['terminals']],
                weights=rows[:, o['weights']])

  def mix(self, r, eps): return eps[r][:, None] * self.exp[r] + (1 - eps[r][:, None]) * self.pol[r]

  def loss_rows(self, r):
    """Rows of every loss pass of replica r, with the key of its log-policy input."""
    if self.p['loss'] == 'Mixup': return [(self.mix(r, self.eps_mix), 'mix')]
    return [(self.pol[r], 'policy'), (self.exp[r], 'expert')]

  def pass_rows(self, r):
    rows = [x for x, _ in self.loss_rows(r)]
    return rows + ([self.mix(r, self.eps_gp)] if self.p['gp'] > 0 else [])

  def log_policy(self, r, rows):
    from oracle import port
    f = self.fields(rows)
    return port.actor_log_prob(self.actor[r], f['states'], f['actions'])

  def logits(self, r, passes, training=True):
    """float64 (pre-activations of every differentiated evaluation, logits without the log-policy term) of each pass of replica r."""
    p, n = self.p, len(passes)
    g_eff = _accesses(*self.g[r], n, p['sn'], training)
    h_eff = _accesses(*self.h[r], 2 * n, p['sn'], training) if self.h else None
    o, S = self.off, p['S']
    out = []
    for k, rows in enumerate(passes):
      zs, f = _forward(g_eff[k], rows[:, :self.d], p['act'])
      if h_eff:
        _, hn = _forward(h_eff[2 * k], rows[:, o['next_states']:o['next_states'] + S], p['act'])  # h(s') is never differentiated by the penalty
        zh, hs = _forward(h_eff[2 * k + 1], rows[:, :S], p['act'])
        zs = zs + zh
        f = f + (1 - rows[:, o['terminals']]) * (self.discount(r) * hn - hs)
      out.append((zs, f))
    return out

  def clear_kinks(self):
    """Draws the batch rows (and their noise) again where a float64 ReLU pre-activation of a differentiated evaluation lies within KINK of 0."""
    if self.p['act'] != 'relu' or self.p['depth'] == 0: return
    R, B = self.p['R'], self.p['B']
    for _ in range(100):
      bad = torch.zeros(R, B, dtype=torch.bool)
      for r in range(R):
        for zs, _ in self.logits(r, self.pass_rows(r)):
          for z in zs: bad[r] |= (z.abs() < KINK).any(1)
      if not bad.any(): return
      n = int(bad.sum())
      self.pol[bad], self.exp[bad] = self._rows(n), self._rows(n)
      self.eps_gp[bad], self.eps_mix[bad] = self._unit(n), self._unit(n)
    raise AssertionError('could not draw a batch away from the ReLU kink')

  def pugail_inner(self, r):
    """The clamped quantity of training.py:102 in float64."""
    sp = torch.nn.functional.softplus
    (fp_rows, _), (fe_rows, _) = self.loss_rows(r)
    (_, fp), (_, fe) = self.logits(r, [fp_rows, fe_rows])
    if self.actor:
      fp, fe = fp - self.log_policy(r, fp_rows), fe - self.log_policy(r, fe_rows)
    wo = self.off['weights']
    return (PRIOR * (fe_rows[:, wo] * sp(fe)).mean() - (fp_rows[:, wo] * sp(fp)).mean()).item()

  def prepare_update(self):
    """Clears the kinks; a PUGAIL row draws its whole batch again until every replica's clamp is CLAMP_GAP from -margin (and active at a
    finite margin)."""
    R, B = self.p['R'], self.p['B']
    for _ in range(20):
      self.clear_kinks()
      if not self.p['loss'].startswith('PUGAIL'): return
      margin = MARGIN[self.p['loss']]
      inner = [self.pugail_inner(r) for r in range(R)]
      if all(abs(x + margin) > CLAMP_GAP and (margin == float('inf') or x < -margin) for x in inner): return
      self.pol, self.exp = self._rows(R, B), self._rows(R, B)
      self.eps_gp, self.eps_mix = self._unit(R, B), self._unit(R, B)
    raise AssertionError(f'could not draw a batch whose PUGAIL clamp is clear of -margin {margin} (and active): {inner}')


# ---- float64 / fp32 references (oracle.port on the CPU) --------------------------------------------------------------------------------
def _port_disc(pb, r, dtype, rf='AIRL'):
  from oracle import port
  p = pb.p
  cast = lambda ts: [t.to(dtype).clone() for t in ts]
  disc = port.GailDiscriminator(pb.g[r][0], None, discount=pb.discount(r), activation=p['act'], reward_function=rf, state_only=p['state_only'],
                                subtract_log_policy=p['logp'], h=pb.h[r][0] if pb.h else None)
  disc.g = [torch.nn.Parameter(t) for t in cast(pb.g[r][0])]  # __init__ casts to float32
  if pb.h: disc.h = [torch.nn.Parameter(t) for t in cast(pb.h[r][0])]
  if p['sn']:
    disc.g_sn = [tuple(cast(uv)) for uv in pb.g[r][1]]
    if pb.h: disc.h_sn = [tuple(cast(uv)) for uv in pb.h[r][1]]
  return disc


def port_update(pb, r, dtype):
  """Gradients of every g then h parameter, losses (bce / mixup, gp) and the per-layer (u, v) of g then h after one update of replica r."""
  from oracle import port
  p = pb.p
  disc = _port_disc(pb, r, dtype)
  pol, exp = (pb.fields(x[r].to(dtype)) for x in (pb.pol, pb.exp))
  loss = 'PUGAIL' if p['loss'].startswith('PUGAIL') else p['loss']
  actor = [t.to(dtype) for t in pb.actor[r]] if pb.actor else None
  out = port.gail_update(disc, _GradOnly(), pol, exp, pb.eps_gp[r].to(dtype) if p['gp'] > 0 else None, loss_function=loss, grad_penalty=pb.gp(r),
                         entropy_bonus=pb.ent(r), pos_class_prior=PRIOR, nonnegative_margin=MARGIN.get(p['loss'], float('inf')),
                         eps_mixup=pb.eps_mix[r].to(dtype) if loss == 'Mixup' else None, actor=actor)
  grads = [q.grad.detach().double() for q in disc.parameters()]
  losses = [out['bce_loss'].item(), out['gp_loss'].item() if 'gp_loss' in out else 0.0]
  uv = [tuple(t.double() for t in x) for x in (disc.g_sn or []) + (disc.h_sn or [])] if p['sn'] else []
  return grads, losses, uv


def port_reward(pb, r, dtype, logp):
  disc = _port_disc(pb, r, dtype, pb.p['rf'])
  f = pb.fields(pb.pol[r].to(dtype))
  args = (f['states'], f['actions'], f['next_states'], f['terminals'], None if logp is None else logp[r].to(dtype))
  with torch.no_grad():
    return disc.forward(*args).double(), disc.predict_reward(*args).double()


# ---- device problems ----------------------------------------------------------------------------------------------------------------------
def _mlp_struct(ptr, stride, dims, act):
  from il_b200 import _lib
  m = _lib.Mlp()
  m.params, m.stride, m.n_layers, m.activation = ptr, stride, len(dims) - 1, _lib.ACT[act]
  for i, x in enumerate(dims): m.dims[i] = x
  return m


def _net_layout(dims):
  """[(offset, shape)] of W0, b0, W1, b1, ... and the net's total floats (il_mlp_param_offsets)."""
  from il_b200._lib import py_mlp_offsets
  w, b, total = py_mlp_offsets(dims)
  out = []
  for l in range(len(dims) - 1): out += [(w[l], (dims[l + 1], dims[l])), (b[l], (dims[l + 1], ))]
  return out, total


class Device:
  """The device buffers of one problem: g and h in one flat [R, stride] buffer whose padding is zero, u / v rows with a SENTINEL tail, batch
  replicas `rs` floats apart with a SENTINEL gap, and a workspace filled with NaN followed by WS_TAIL bytes of SENTINEL."""

  def __init__(self, pb):
    p, R, B = pb.p, pb.p['R'], pb.p['B']
    self.pb, self.p = pb, p
    g_lay, g_total = _net_layout(pb.g_dims)
    h_lay, h_total = _net_layout(pb.h_dims) if pb.h_dims else ([], 0)
    self.h_off, self.stride = g_total, g_total + h_total + 12
    self.layout = [(off, shape) for off, shape in g_lay] + [(g_total + off, shape) for off, shape in h_lay]  # every parameter tensor, g then h
    prm = torch.zeros(R, self.stride, dtype=torch.float64)
    self.live = torch.zeros(R, self.stride, dtype=torch.bool)
    for r in range(R):
      tensors = pb.g[r][0] + (pb.h[r][0] if pb.h else [])
      for (off, shape), t in zip(self.layout, tensors):
        prm[r, off:off + t.numel()] = t.flatten()
        self.live[r, off:off + t.numel()] = True
    self.params = prm.float().to(DEV)
    self.m, self.v = torch.zeros_like(self.params), torch.zeros_like(self.params)
    self.sn = {}  # net -> (u, v) buffers
    if p['sn']:
      for net, dims, nets in (('g', pb.g_dims, pb.g), ('h', pb.h_dims, pb.h)):
        if dims is None: continue
        uu, vv = torch.full((R, sum(dims[1:]) + 5), SENTINEL, dtype=torch.float64), torch.full((R, sum(dims[:-1]) + 3), SENTINEL, dtype=torch.float64)
        for r in range(R):
          u_cat, v_cat = torch.cat([u for u, _ in nets[r][1]]), torch.cat([v for _, v in nets[r][1]])
          uu[r, :u_cat.numel()], vv[r, :v_cat.numel()] = u_cat, v_cat
        self.sn[net] = (uu.float().to(DEV), vv.float().to(DEV))
    self.step = torch.zeros(1, dtype=torch.int64, device=DEV)
    self.rs = B * pb.row + 4  # batch replica stride: 16-byte aligned, not B * row
    self.pol, self.exp = (self._batch(x) for x in (pb.pol, pb.exp))
    self.eps_gp, self.eps_mix = pb.eps_gp.float().to(DEV), pb.eps_mix.float().to(DEV)
    self.logp = {}
    if pb.actor:  # the log-policy inputs in fp32, from the float64 actor
      with torch.no_grad():
        for key, fn in (('policy', lambda r: pb.pol[r]), ('expert', lambda r: pb.exp[r]), ('mix', lambda r: pb.mix(r, pb.eps_mix))):
          self.logp[key] = torch.stack([pb.log_policy(r, fn(r)) for r in range(R)]).float().to(DEV)
    self.losses = torch.full((R, 2), SENTINEL, device=DEV)
    arr = lambda xs, dt: None if xs is None else torch.tensor(xs, dtype=dt, device=DEV)
    self.ent_r, self.discount_r, self.gp_r = (arr(x, torch.float32) for x in (pb.ent_r, pb.discount_r, pb.gp_r))
    self.lr_r, self.wd_r = arr(pb.lr_r, torch.float64), arr(pb.wd_r, torch.float64)
    self.ws = None
    self.inputs = [t.clone() for t in self._inputs()]
    self.state0 = [t.clone() for t in self._state()]

  def _batch(self, x):
    R, B, row = x.shape
    buf = torch.full((R, self.rs), SENTINEL, dtype=torch.float64)
    buf[:, :B * row] = x.reshape(R, -1)
    return buf.float().to(DEV)

  def _inputs(self):
    return [self.pol, self.exp, self.eps_gp, self.eps_mix] + list(self.logp.values()) + [t for t in (self.ent_r, self.discount_r, self.gp_r, self.lr_r, self.wd_r) if t is not None]

  def _state(self):
    return [self.params, self.m, self.v, self.step, self.losses] + [t for uv in self.sn.values() for t in uv]

  def workspace(self, need):
    self.need = need
    self.ws = torch.empty(need // 4 + WS_TAIL // 4, device=DEV)
    self.fill_ws()
    return self.ws

  def fill_ws(self):
    self.ws[:self.need // 4].fill_(float('nan'))
    self.ws[self.need // 4:].fill_(SENTINEL)

  def reset(self):
    for t, t0 in zip(self._state(), self.state0): t.copy_(t0)
    if self.ws is not None: self.fill_ws()

  def batch_struct(self, buf):
    from il_b200 import _lib
    b = _lib.Batch()
    b.rows, b.replica_stride, b.B, b.S, b.A, b.row = buf.data_ptr(), self.rs, self.p['B'], self.p['S'], self.p['A'], self.pb.row
    return b

  def disc_struct(self, rf='AIRL'):
    from il_b200 import _lib
    p, pb, d = self.p, self.pb, _lib.Gailx()
    d.g = _mlp_struct(self.params.data_ptr(), self.stride, pb.g_dims, p['act'])
    if pb.h_dims: d.h = _mlp_struct(self.params.data_ptr() + 4 * self.h_off, self.stride, pb.h_dims, p['act'])
    if 'g' in self.sn:
      (gu, gv) = self.sn['g']
      d.g_u, d.g_v, d.g_u_stride, d.g_v_stride = gu.data_ptr(), gv.data_ptr(), gu.stride(0), gv.stride(0)
    if 'h' in self.sn:
      (hu, hv) = self.sn['h']
      d.h_u, d.h_v, d.h_u_stride, d.h_v_stride = hu.data_ptr(), hv.data_ptr(), hu.stride(0), hv.stride(0)
    d.state_only, d.reward_function, d.subtract_log_policy, d.discount = int(p['state_only']), _lib.REWARD[rf], int(p['logp']), DISCOUNT
    if self.discount_r is not None: d.discount_r = self.discount_r.data_ptr()
    return d

  def update_args(self):
    from il_b200 import _lib
    p, R, a = self.p, self.p['R'], _lib.GailxUpdateArgs()
    a.disc, a.params_floats = self.disc_struct(), R * self.stride
    a.policy, a.expert = self.batch_struct(self.pol), self.batch_struct(self.exp)
    o = a.opt
    o.m, o.v, o.step, o.lr, o.beta1, o.beta2, o.eps, o.weight_decay = self.m.data_ptr(), self.v.data_ptr(), self.step.data_ptr(), LR, BETAS[0], BETAS[1], ADAM_EPS, WD
    if self.lr_r is not None: o.lr_r, o.weight_decay_r, o.replica_floats = self.lr_r.data_ptr(), self.wd_r.data_ptr(), self.stride
    mixup = p['loss'] == 'Mixup'
    a.eps_gp = self.eps_gp.data_ptr() if p['gp'] > 0 else None
    a.eps_mix = self.eps_mix.data_ptr() if mixup else None
    if self.logp:
      if mixup: a.logp_mix = self.logp['mix'].data_ptr()
      else: a.logp_policy, a.logp_expert = self.logp['policy'].data_ptr(), self.logp['expert'].data_ptr()
    a.R, a.loss_function, a.training = R, _lib.LOSS['PUGAIL' if p['loss'].startswith('PUGAIL') else p['loss']], 1
    a.grad_penalty, a.entropy_bonus, a.pos_class_prior, a.nonnegative_margin = p['gp'], p['ent'], PRIOR, MARGIN.get(p['loss'], float('inf'))
    if self.gp_r is not None: a.grad_penalty_r = self.gp_r.data_ptr()
    if self.ent_r is not None: a.entropy_bonus_r = self.ent_r.data_ptr()
    a.out_losses = self.losses.data_ptr()
    return a

  def check_bounds(self):
    """Inputs, the zero padding of the flat buffer, the u / v tails and the workspace tail."""
    for i, (before, after) in enumerate(zip(self.inputs, self._inputs())): assert torch.equal(before, after), f'input {i} (rows, eps, logp, per-replica values) modified'
    live = self.live.to(DEV)
    for name, t in (('params', self.params), ('m', self.m), ('v', self.v)):
      assert (t[~live] == 0).all(), f'{name}: {int((t[~live] != 0).sum())} padding floats of the flat buffer not zero'
    for net, (uu, vv) in self.sn.items():
      dims = self.pb.g_dims if net == 'g' else self.pb.h_dims
      assert (uu[:, sum(dims[1:]):] == SENTINEL).all(), f'{net}: u written past its {sum(dims[1:])} slots'
      assert (vv[:, sum(dims[:-1]):] == SENTINEL).all(), f'{net}: v written past its {sum(dims[:-1])} slots'
    assert (self.ws[self.need // 4:] == SENTINEL).all(), f'{int((self.ws[self.need // 4:] != SENTINEL).sum())} floats written past the {self.need}-byte workspace'


def _views(flat, layout):
  return [flat[off:off + math.prod(shape)].view(shape) for off, shape in layout]


def _names(pb):
  out = []
  for net, dims in (('g', pb.g_dims), ('h', pb.h_dims)):
    if dims: out += [f'{net}.{"Wb"[i % 2]}{i // 2}' for i in range(2 * (len(dims) - 1))]
  return out


def _output_bias_scale(pb, r, net):
  """Size of the terms an output-bias gradient sums: per loss pass and row, |d loss / d logit| <= w (1 + 0.23 entropy_bonus) / B, times
  (1 + discount) for h, which enters through h(s') and h(s). The sum cancels (policy against expert rows, h(s') against h(s)), so its float32
  rounding error scales with these terms rather than with the result: a sequential sum over B rows on the device is as correct as torch's
  pairwise one on the CPU, yet its error can be 30x larger relative to the result."""
  wo = pb.off['weights']
  s = sum(rows[:, wo].mean().item() for rows, _ in pb.loss_rows(r)) * (1 + 0.23 * pb.ent(r))
  return s * (1 + pb.discount(r)) if net == 'h' else s


def check_update(dv):
  """Gradient, v, AdamW step, losses and u / v of every replica against float64."""
  p, pb = dv.p, dv.pb
  assert int(dv.step.item()) == 1, f'step counter {int(dv.step.item())} after one update'
  w1c, w2c = np.float32(1 - BETAS[0]), np.float32(1 - BETAS[1])
  names = _names(pb)
  out_biases = {f'{net}.b{len(dims) - 2}' for net, dims in (('g', pb.g_dims), ('h', pb.h_dims)) if dims}
  for r in range(p['R']):
    what = f'replica {r}'
    m, v, prm = (_views(t[r].double().cpu(), dv.layout) for t in (dv.m, dv.v, dv.params))
    p0 = pb.g[r][0] + (pb.h[r][0] if pb.h else [])
    g = [t / float(w1c) for t in m]
    f64, f32 = port_update(pb, r, torch.float64), port_update(pb, r, torch.float32)
    lr, wd = pb.lr(r), pb.wd(r)
    step_size, bc2 = lr / (1 - BETAS[0]), math.sqrt(1 - BETAS[1])
    for i, name in enumerate(names):
      if name in out_biases:
        got_g, want, cpu = g[i].numpy(), f64[0][i].numpy(), f32[0][i].numpy()
        err, cpu_err, scale = np.abs(got_g - want).max(), np.abs(cpu - want).max(), max(np.abs(want).max(), _output_bias_scale(pb, r, name[0]))
        assert err <= 8 * cpu_err + 1e-6 * scale, f'd{name} {what}: max |cuda - f64| = {err:.3e}, max |cpu fp32 - f64| = {cpu_err:.3e}, summed terms {scale:.3e}'
      else:
        _assert_vs_f64(g[i].numpy(), f64[0][i].numpy(), f32[0][i].numpy(), f'd{name} {what}')
      vg = v[i] / float(w2c)
      err = (vg - g[i] ** 2).abs()
      assert (err <= 1e-6 * g[i] ** 2).all(), f'{name} {what}: v / (1 - beta2) differs from g^2 by up to {float(err.max()):.3e}'
      term = step_size * m[i] / (v[i].sqrt() / bc2 + ADAM_EPS)
      ref = p0[i] * (1 - lr * wd) - term
      bound = 3 * _ulp32(ref) + 16 * U * term.abs()
      err = (prm[i] - ref).abs()
      assert (err <= bound).all(), f'{name} {what}: parameter off the AdamW step of its own m, v by {float((err / bound).max()):.2f}x the bound'
    got = dv.losses[r].double().cpu()
    _assert_vs_f64(got[0].item(), f64[1][0], f32[1][0], f'{p["loss"]} loss {what}')
    if p['gp'] > 0: _assert_vs_f64(got[1].item(), f64[1][1], f32[1][1], f'gradient-penalty loss {what}')
    else: assert got[1].item() == SENTINEL, f'gradient-penalty loss slot written ({got[1].item()}) without a penalty pass ({what})'
    l = 0
    for net, dims in (('g', pb.g_dims), ('h', pb.h_dims)):
      if not p['sn'] or dims is None: continue
      uu, vv = dv.sn[net]
      uo = vo = 0
      for k in range(len(dims) - 1):
        for name, buf, o, n, i in (('u', uu, uo, dims[k + 1], 0), ('v', vv, vo, dims[k], 1)):
          _assert_vs_f64(buf[r, o:o + n].double().cpu().numpy(), f64[2][l][i].numpy(), f32[2][l][i].numpy(), f'spectral-norm {name} of {net} layer {k} {what}')
        uo, vo, l = uo + dims[k + 1], vo + dims[k], l + 1


def expected_launches(p, g_dims, h_dims):
  """Launches per kernel of il_gailx_update that follow from the configuration."""
  gp, mixup = p['gp'] > 0, p['loss'] == 'Mixup'
  per, n_loss = (3 if h_dims else 1), (1 if mixup else 2)
  Ls = [len(d) - 1 for d in (g_dims, h_dims) if d is not None] if gp else []  # the nets of the penalty pass
  deep = [L for L in Ls if L >= 2]
  return {'sn_access_kernel': (n_loss + gp) * per, 'mix_batch_kernel': mixup + gp, 'gailx_loss_kernel': 1, 'sn_project_kernel': n_loss * per + len(Ls),
          'gp_penalty_kernel': int(gp), 'gp_linear_gx_kernel': sum(L == 1 for L in Ls), 'gp_kappa_colsum_kernel': len(Ls), 'gp_top_kernel': len(deep),
          'gp_mask_kernel': sum(L - 2 for L in deep), 'gp_second_kernel': sum(L - 1 for L in deep),
          'add_kernel': 0 if p['act'] == 'relu' else sum(L - 2 for L in deep)}


def _run(dv, call):
  import il_b200
  from il_b200 import _lib
  launches = []
  def fn():
    before = il_b200.launch_count()
    _lib.check(call())
    launches.append(il_b200.launch_count() - before)
  for _ in range(3):  # now and then a trace misses one of the call's kernels (the launch counter still shows it): take it again
    names = kernels_of(fn, attempts=3, setup=dv.reset)
    if len(names) >= launches[-1]: break
  assert len(set(launches)) == 1, f'library launches per call: {launches}'
  return names


def _seed(request): return zlib.crc32(request.node.callspec.id.encode())


@pytest.fixture(autouse=True)
def _fp32_gemm():
  from il_b200 import _lib
  _lib.check(_lib.lib().il_set_gemm_mode(_lib.handle(), _lib.GEMM_MODE['fp32']))
  yield


@pytest.mark.parametrize('p', ROUTES)
def test_gailx_route(p, request):
  from il_b200 import _lib
  lib = _lib.lib()
  pb = Problem(p, _seed(request))
  if p['kind'] == 'update': pb.prepare_update()
  dv = Device(pb)
  if p['kind'] == 'update':
    a = dv.update_args()
    ws = dv.workspace(lib.il_gailx_workspace_bytes(C.byref(a)))
    a.workspace, a.workspace_bytes = ws.data_ptr(), dv.need
    names = _run(dv, lambda: lib.il_gailx_update(_lib.handle(), C.byref(a), _lib.stream()))
    got, want = Counter(names), expected_launches(p, pb.g_dims, pb.h_dims)
    assert {k: got[k] for k in want} == want, f'launches {dict(got)}, expected {want}'
    check_update(dv)
    dv.check_bounds()
    return
  # reward rows: eval-mode forward; parameters, u / v and the batch are read only
  R, B, ld = p['R'], p['B'], p['ld']
  d = dv.disc_struct(p['rf'])
  ws = dv.workspace(lib.il_gailx_reward_workspace_bytes(C.byref(d), R, B))
  rs = B * ld + 3  # padded replica stride of the reward output
  reward = torch.full((R * rs + 1, ), SENTINEL, device=DEV)
  logits = torch.full((R, B), SENTINEL, device=DEV) if p['logits'] else None
  logp = dv.logp.get('policy')
  b = dv.batch_struct(dv.pol)
  base_reset = dv.reset
  def reset():
    base_reset()
    reward.fill_(SENTINEL)
    if logits is not None: logits.fill_(SENTINEL)
  dv.reset = reset
  names = _run(dv, lambda: lib.il_gailx_reward(_lib.handle(), C.byref(d), R, C.byref(b), _lib.ptr(logp), reward.data_ptr(), rs, ld, _lib.ptr(logits), ws.data_ptr(), dv.need,
                                               _lib.stream()))
  got = Counter(names)
  assert got['sn_access_kernel'] == (3 if p['shaping'] else 1) and got['gailx_reward_kernel'] == 1, f'launches {dict(got)}'
  for i, (t, t0) in enumerate(zip(dv._state(), dv.state0)): assert torch.equal(t, t0), f'il_gailx_reward wrote its state ({i})'
  dv.check_bounds()
  written = torch.zeros_like(reward, dtype=torch.bool)
  logp64 = None if logp is None else logp.double().cpu()
  for r in range(R):
    idx = r * rs + torch.arange(B, device=DEV) * ld
    written[idx] = True
    f64, f32 = port_reward(pb, r, torch.float64, logp64), port_reward(pb, r, torch.float32, logp64)
    if logits is not None: _assert_vs_f64(logits[r].double().cpu().numpy(), f64[0].numpy(), f32[0].numpy(), f'logits replica {r}')
    _assert_vs_f64(reward[idx].double().cpu().numpy(), f64[1].numpy(), f32[1].numpy(), f'{p["rf"]} reward replica {r}')
  assert (reward[~written] == SENTINEL).all(), f'{int((reward[~written] != SENTINEL).sum())} reward floats outside the B x ld x R output written'


# ---- refused calls ------------------------------------------------------------------------------------------------------------------------
REFUSALS = [
  # (id, row changes, args change, error text)
  ('state_only_grad_penalty', dict(state_only=True), None, 'grad_penalty with a state-only discriminator'),
  ('missing_eps_gp', {}, lambda a, dv, h: setattr(a, 'eps_gp', None), 'missing eps_gp / eps_mix'),
  ('missing_eps_mix', dict(loss='Mixup'), lambda a, dv, h: setattr(a, 'eps_mix', None), 'missing eps_gp / eps_mix'),
  ('logp_missing', dict(logp=True), lambda a, dv, h: setattr(a, 'logp_expert', None), 'subtract_log_policy needs the log-policy inputs'),
  ('logp_mix_missing', dict(logp=True, loss='Mixup'), lambda a, dv, h: setattr(a, 'logp_mix', None), 'subtract_log_policy needs the log-policy inputs'),
  ('workspace_one_byte_short', {}, lambda a, dv, h: setattr(a, 'workspace_bytes', a.workspace_bytes - 1), 'workspace too small'),
  ('h_outside_the_flat_buffer', {}, lambda a, dv, h: (setattr(a.disc.h, 'params', h.data_ptr()), setattr(a.disc.h, 'stride', h.stride(0))),
   'g / h must live in one flat [R, stride] parameter buffer'),
  ('spectral_norm_on_g_only', {}, lambda a, dv, h: (setattr(a.disc, 'h_u', None), setattr(a.disc, 'h_v', None)), 'spectral norm must cover both g and h'),
  ('loss_code_3', {}, lambda a, dv, h: setattr(a, 'loss_function', 3), 'bad loss function 3'),
]


@pytest.mark.parametrize('what,changes,edit,text', REFUSALS, ids=[x[0] for x in REFUSALS])
def test_gailx_update_refused(what, changes, edit, text):
  import il_b200
  from il_b200 import _lib
  lib = _lib.lib()
  p = upd(B=16, depth=1, act='tanh', shaping=True, gp=1.0).values[0]
  p = dict(p, **changes)
  pb = Problem(p, seed=7)
  dv = Device(pb)
  a = dv.update_args()
  ws = dv.workspace(lib.il_gailx_workspace_bytes(C.byref(a)))
  a.workspace, a.workspace_bytes = ws.data_ptr(), dv.need
  h_elsewhere = torch.zeros(p['R'], dv.stride + 4, device=DEV)  # a copy of h with its own stride: not the flat buffer AdamW covers
  h_elsewhere[:, :dv.stride - dv.h_off] = dv.params[:, dv.h_off:]
  if edit: edit(a, dv, h_elsewhere)
  before = il_b200.launch_count()
  rc = lib.il_gailx_update(_lib.handle(), C.byref(a), _lib.stream())
  torch.cuda.synchronize()
  assert rc != 0, 'the call was accepted'
  assert text in _lib.last_error(), _lib.last_error()
  assert il_b200.launch_count() == before, 'a refused call launched a kernel'
  for i, (t, t0) in enumerate(zip(dv._state(), dv.state0)): assert torch.equal(t, t0), f'a refused call wrote its state ({i}: params, m, v, step, losses, u, v)'
  dv.check_bounds()
