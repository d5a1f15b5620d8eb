"""Every route of the fused GAIL discriminator kernels (csrc/gail.cu: il_gail_update, il_gail_reward) against float64.

il_gail_update picks one of seven kernels from the input width d, the hidden width H, the batch size B and the shared memory each needs
(gail_update_plan); il_gail_reward picks one of two. Both walk the batch in chunks of RB rows, the last of which can be partial. Each row of
the route table names the kernel the call must run and sits on one side of a selection condition or a chunk edge. For every row the test checks
- the route: the named kernel is the only discriminator kernel of the call (after gail_tick_kernel for an update), read from a CUDA-activity
  `torch.profiler` trace;
- the gradient: one update from zero AdamW moments leaves m = (1 - beta1) g and v = (1 - beta2) g^2; g is compared with the float64 autograd
  gradient of oracle.port.gail_update (BCE / PUGAIL / Mixup, closed-form gradient-penalty double backward, entropy bonus, spectral-norm
  backward), and v with g^2;
- the parameters: the AdamW formula in float64 on the kernel's own m, v and the old parameters, within a few ulp (after one step the update
  is about lr sign(g), so a plain comparison would hide a wrong gradient); the step counter advances by one;
- the side outputs: the BCE / Mixup and gradient-penalty losses, and the spectral-norm u, v written back;
- the reward rows: logits and reward of every reward function;
- the bounds: the stride padding of every parameter block, the u / v slots past each replica's vectors, the replicas a call does not run, the
  reward guard band and the inputs stay untouched.
Values use the tolerance of the MLP head tests: per output tensor, 8 max|port in fp32 on the CPU - float64| + 1e-6 max|float64|. Inputs are
drawn from seeded generators; batch rows whose float64 hidden pre-activation lies within 1e-4 of the ReLU kink in any pass are drawn again, and
every PUGAIL row asserts that its clamp is at least 1e-3 from the margin, so a mask flip is never mistaken for a kernel error.
"""
import ctypes as C
import math
from itertools import product

import numpy as np
import pytest
import torch

from test_gpu_gemm_routes import _assert_vs_f64, kernels_of

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
SENTINEL = 1234.5
ENV = {'hopper': (12, 3), 'halfcheetah': (18, 6), 'ant': (112, 8)}  # state (with the absorbing bit), action
LR, WD, BETAS, ADAM_EPS, PRIOR = 1e-3, 0.1, (0.9, 0.999), 1e-8, 0.7
KINK, CLAMP_GAP = 1e-4, 1e-3
DEV = 'cuda'
LOSSES = ('BCE', 'PUGAIL', 'PUGAIL0', 'Mixup', 'PUGAILm')  # PUGAIL: margin inf; PUGAIL0: margin 0 and PUGAILm: margin 0.05, where the clamp is active
MARGIN = {'PUGAIL': float('inf'), 'PUGAIL0': 0.0, 'PUGAILm': 0.05}
TICK = 'gail_tick_kernel'
REW_TILED, REW = 'gail_reward_tiled_kernel', 'gail_reward_kernel'


def tiled(nt): return f'gail_update_tiled_kernel<{nt}>'


def untiled(ne): return f'gail_update_kernel<{ne}>'


# ---- the route table ------------------------------------------------------------------------------------------------------------------
def upd(kernel, env, H, B, loss='BCE', gp=1.0, ent=0.0, sn=True, state_only=False, tiled_on=1, order=False, S=None, A=None):
  """One update problem and the kernel that must run it; S / A override the environment's sizes. order: the call runs replicas [2, 0] of a
  3-replica buffer through replica_order (replica 1 must stay untouched); otherwise replicas 0, 1 in block order (replica 2 untouched)."""
  S, A = (S, A) if S is not None else ENV[env]
  p = dict(kind='update', kernel=kernel, S=S, A=A, H=H, B=B, loss=loss, gp=gp, ent=ent, sn=sn, state_only=state_only, tiled=tiled_on, order=order)
  d = S if state_only else S + A
  tags = [env or f'S{S}A{A}', f'd{d}', f'H{H}', f'B{B}', loss, f'gp{gp:g}', f'ent{ent:g}', 'sn' if sn else 'nosn']
  if state_only: tags.append('state_only')
  if not tiled_on: tags.append('untiled_opt')
  if order: tags.append('order')
  short = kernel.replace('gail_update_', '').replace('_kernel', '').replace('<', '').replace('>', '')
  return pytest.param(p, id=short + '-' + '-'.join(tags))


def rew(kernel, env, H, B, rf='AIRL', sn=True, ld=1, order=False, tiled_on=1):
  S, A = ENV[env]
  p = dict(kind='reward', kernel=kernel, S=S, A=A, H=H, B=B, rf=rf, sn=sn, ld=ld, state_only=False, tiled=tiled_on, order=order)
  tags = [env, f'd{S + A}', f'H{H}', f'B{B}', rf, 'sn' if sn else 'nosn', f'ld{ld}'] + (['order'] if order else [])
  return pytest.param(p, id=kernel.replace('gail_', '').replace('_kernel', '') + '-' + '-'.join(tags))


PRODUCT = list(product(LOSSES, (0.0, 1.0), (0.0, 0.05), (False, True)))  # loss x gradient penalty x entropy bonus x spectral norm
SPREAD = PRODUCT[:32]  # the first four losses: the spread of the rows outside the full product predates PUGAILm


def _opts(i):
  """A spread of the option product for the rows outside the two full-product routes."""
  loss, gp, ent, sn = SPREAD[(11 * i + 5) % len(SPREAD)]
  return dict(loss=loss, gp=gp, ent=ent, sn=sn)


def _route_table():
  t = []
  # the full option product on the bench route (hopper, H = 64, B = 256: two 128-row chunks) and on the Ant route of GAIL_25_trajectories
  # (H = 128: gail_update_kernel<64>, 16 chunks of 16 rows)
  for loss, gp, ent, sn in PRODUCT:
    t.append(upd(tiled(1), 'hopper', 64, 256, loss, gp, ent, sn))
    t.append(upd(untiled(64), 'ant', 128, 256, loss, gp, ent, sn))
  rows = [
    # gail_tiled = 1: d <= 32, H in {32, 64, 128}, B % 4 == 0, tiles <= 256 and the carve-up within 110 KB
    dict(kernel=tiled(1), env='hopper', H=64, B=132),                       # last chunk 4 rows
    dict(kernel=tiled(1), env='hopper', H=64, B=20),                        # RB 32: 12 zero-padded rows
    dict(kernel=tiled(1), env='hopper', H=64, B=1024, order=True),          # 8 chunks
    dict(kernel=tiled(1), env='hopper', H=32, B=256),
    dict(kernel=tiled(2), env='hopper', H=128, B=256),
    dict(kernel=tiled(2), env='halfcheetah', H=64, B=256),
    dict(kernel=tiled(4), env='halfcheetah', H=128, B=256),                 # RB 32: 8 chunks
    dict(kernel=tiled(4), env='halfcheetah', H=128, B=256, state_only=True),  # d = 18: RB 64
    dict(kernel=tiled(4), env='halfcheetah', H=128, B=100, order=True),     # RB 32, last chunk 4 rows
    dict(kernel=tiled(4), env=None, S=22, A=6, H=128, B=256),               # d = 28: the last d that fits at H = 128
    dict(kernel=tiled(4), env=None, S=22, A=6, H=128, B=72),                # RB 80 halved twice: 20-row chunks, the last 12 rows
    dict(kernel=untiled(16), env=None, S=24, A=6, H=128, B=256),            # d = 30: 117 KB tiled even at RB 32
    dict(kernel=untiled(16), env=None, S=26, A=6, H=128, B=64),             # d = 32
    # fall-backs to the untiled kernel
    dict(kernel=untiled(4), env='hopper', H=64, B=254),                     # B % 4 != 0
    dict(kernel=untiled(4), env='hopper', H=64, B=1),
    dict(kernel=untiled(4), env='hopper', H=48, B=256),                     # not a tiled width
    dict(kernel=untiled(4), env='hopper', H=64, B=256, tiled_on=0),         # gail_tiled off
    dict(kernel=untiled(16), env='halfcheetah', H=128, B=256, tiled_on=0),
    # untiled instances <NE>: NE = ceil(H d / 256)
    dict(kernel=untiled(16), env='ant', H=32, B=256),
    dict(kernel=untiled(32), env='ant', H=64, B=256),
    dict(kernel=untiled(32), env='ant', H=64, B=65, order=True),            # RB 64: last chunk 1 row
    dict(kernel=untiled(64), env='ant', H=128, B=17),                       # RB 16: 2 chunks, last 1 row
    dict(kernel=untiled(64), env='ant', H=128, B=256, order=True),
    dict(kernel=untiled(64), env='ant', H=128, B=33, state_only=True),      # d = 112
  ]
  for i, r in enumerate(rows):
    o = _opts(i)
    if r.get('state_only'): o['gp'] = 0.0  # refused with a state-only discriminator (test_gail_update_refused)
    t.append(upd(r.pop('kernel'), r.pop('env'), r.pop('H'), r.pop('B'), **o, **r))
  # il_gail_reward: the tiled forward for d <= 32, H in {32, 64, 128} within 72 KB (RB 64, or B rounded up to 16); the untiled kernel otherwise
  for rf, sn in product(('AIRL', 'GAIL', 'FAIRL'), (False, True)):
    t.append(rew(REW_TILED, 'hopper', 64, 256, rf, sn, ld=1 + sn))
    t.append(rew(REW, 'ant', 128, 256, rf, sn, ld=2 - sn))                    # RB 16
  t += [
    rew(REW_TILED, 'halfcheetah', 128, 65, 'GAIL', True, ld=2, order=True),   # RB 64: last chunk 1 row
    rew(REW_TILED, 'hopper', 32, 20, 'FAIRL', False, ld=2),                  # RB 32
    rew(REW_TILED, 'hopper', 64, 1, 'AIRL', True),                           # RB 16
    rew(REW, 'hopper', 48, 256, 'FAIRL', True, ld=2),
    rew(REW, 'hopper', 64, 256, 'GAIL', True, tiled_on=0),
    rew(REW, 'ant', 128, 17, 'AIRL', False, order=True),
  ]
  return t


ROUTES = _route_table()


# ---- inputs -----------------------------------------------------------------------------------------------------------------------------
def _layout(d, H):
  from il_b200._lib import py_mlp_offsets
  w, b, total = py_mlp_offsets([d, H, 1])
  return dict(w1=w[0], b1=b[0], w2=w[1], b2=b[1], total=total)


def _normalise(x): return x / x.norm()


def _draw_params(d, H, g):
  """W1, b1, w2, b2 and the spectral-norm vectors u1, v1, u2, v2 (fp32 values held in float64): not converged, so the power iterations move them."""
  f = lambda t: t.float().double()
  W1, b1 = f(torch.randn(H, d, generator=g, dtype=torch.float64) / d ** 0.5), f(0.1 * torch.randn(H, generator=g, dtype=torch.float64))
  w2, b2 = f(torch.randn(1, H, generator=g, dtype=torch.float64) / H ** 0.5), f(0.1 * torch.randn(1, generator=g, dtype=torch.float64))
  u1, v1, v2 = (f(_normalise(torch.randn(n, generator=g, dtype=torch.float64))) for n in (H, d, H))
  u2 = torch.tensor([1.0 if torch.rand(1, generator=g).item() < 0.5 else -1.0], dtype=torch.float64)
  return [W1, b1, w2, b2], [u1, v1, u2, v2]


def _sigmas(params, sn_vecs, n):
  """The float64 (sigma1, sigma2) of n train-mode forwards (one power iteration per layer each)."""
  W1, _, w2, _ = params
  u1, v1, u2, v2 = sn_vecs
  out = []
  for _ in range(n):
    u1 = _normalise(W1 @ v1); v1 = _normalise(W1.t() @ u1)
    u2 = _normalise(w2 @ v2); v2 = _normalise(w2.t() @ u2)
    out.append(((u1 @ W1 @ v1).item(), (u2 @ (w2 @ v2)).item()))
  return out


class Inputs:
  """Parameters, spectral-norm vectors, batches and noise of one problem, CPU float64 holding fp32 values. NB replicas in every buffer."""

  def __init__(self, p, Hs, seed):
    from il_b200._lib import py_row_layout
    S, A, B = p['S'], p['A'], p['B']
    self.d = S if p['state_only'] else S + A
    self.off, self.row = py_row_layout(S, A)
    self.g = torch.Generator().manual_seed(seed)
    self.Hs = Hs
    self.params, self.sn = zip(*[_draw_params(self.d, H, self.g) for H in Hs])
    NB = len(Hs)
    self.pol, self.exp = self._rows(NB, B), self._rows(NB, B)
    self.eps_gp, self.eps_mix = self._unit(NB, B), self._unit(NB, B)

  def _rows(self, *shape):
    x = torch.randn(*shape, self.row, generator=self.g, dtype=torch.float64)
    x[..., self.off['weights']] = torch.rand(*shape, generator=self.g, dtype=torch.float64) + 0.5
    return x.float().double()

  def _unit(self, *shape): return torch.rand(*shape, generator=self.g, dtype=torch.float64).float().double()

  def fields(self, rows, S, A):
    o = self.off
    return dict(states=rows[:, :S], actions=rows[:, S:S + A], next_states=rows[:, o['next_states']:o['next_states'] + S], terminals=rows[:, o['terminals']],
                weights=rows[:, o['weights']])

  def pass_inputs(self, p, r):
    """[(x, w)] of every forward of the update, in the kernel's pass order."""
    d, wo = self.d, self.off['weights']
    pol, exp = self.pol[r], self.exp[r]
    mix = lambda e: (e[:, None] * exp[:, :d] + (1 - e[:, None]) * pol[:, :d], e * exp[:, wo] + (1 - e) * pol[:, wo])
    passes = [mix(self.eps_mix[r])] if p['loss'] == 'Mixup' else [(pol[:, :d], pol[:, wo]), (exp[:, :d], exp[:, wo])]
    if p['gp'] > 0: passes.append(mix(self.eps_gp[r]))
    return passes

  def forwards(self, p, r):
    """float64 hidden pre-activations z and logits f of every pass of replica r's update."""
    params = self.params[r]
    passes = self.pass_inputs(p, r)
    sig = _sigmas(params, self.sn[r], len(passes)) if p['sn'] else [(1.0, 1.0)] * len(passes)
    W1, b1, w2, b2 = params
    out = []
    for (x, w), (s1, s2) in zip(passes, sig):
      z = x @ (W1 / s1).t() + b1
      out.append((z, torch.relu(z) @ (w2 / s2).t()[:, 0] + b2, w))
    return out

  def clear_kinks(self, p, replicas):
    """Draws the batch rows (and their noise) again where a float64 pre-activation of any pass lies within KINK of the ReLU kink."""
    B = p['B']
    for _ in range(100):
      bad = torch.zeros(len(self.Hs), B, dtype=torch.bool)
      for r in replicas:
        for z, _, _ in self.forwards(p, r): bad[r] |= (z.abs() < KINK).any(1)
      if not bad.any(): return
      n = int(bad.sum())
      self.pol[bad], self.exp[bad] = self._rows(n), self._rows(n)
      self.eps_gp[bad], self.eps_mix[bad] = self._unit(n), self._unit(n)
    raise AssertionError('could not draw a batch away from the ReLU kink')

  def pugail_inner(self, p, r):
    """The clamped quantity of training.py:102 in float64."""
    fs = self.forwards(p, r)
    sp = torch.nn.functional.softplus
    (_, fp, wp), (_, fe, we) = fs[0], fs[1]
    return (PRIOR * (we * sp(fe)).mean() - (wp * sp(fp)).mean()).item()


# ---- float64 / fp32 references (oracle.port on the CPU) --------------------------------------------------------------------------------
class _GradOnly:
  """Optimiser stand-in for oracle.port.gail_update: keeps the gradients, takes no step."""
  def zero_grad(self, set_to_none=True): pass
  def step(self): pass


def _port_disc(params, sn_vecs, sn, state_only, rf, dtype):
  from oracle import port
  disc = port.GailDiscriminator(params, None, discount=0.97, reward_function=rf, state_only=state_only)
  disc.g = [torch.nn.Parameter(t.to(dtype).clone()) for t in params]  # __init__ casts to float32
  if sn:
    u1, v1, u2, v2 = (t.to(dtype).clone() for t in sn_vecs)
    disc.g_sn = [(u1, v1), (u2, v2)]
  return disc


def port_update(p, inp, r, dtype):
  """Gradients [dW1, db1, dw2, db2], losses (bce / mixup, gp) and the u, v after one update of replica r."""
  from oracle import port
  S, A = p['S'], p['A']
  disc = _port_disc(inp.params[r], inp.sn[r], p['sn'], p['state_only'], 'AIRL', dtype)
  pol, exp = (inp.fields(x[r].to(dtype), S, A) for x in (inp.pol, inp.exp))
  loss = 'PUGAIL' if p['loss'].startswith('PUGAIL') else p['loss']
  margin = MARGIN.get(p['loss'], float('inf'))
  out = port.gail_update(disc, _GradOnly(), pol, exp, inp.eps_gp[r].to(dtype) if p['gp'] > 0 else None, loss_function=loss, grad_penalty=p['gp'],
                         entropy_bonus=p['ent'], pos_class_prior=PRIOR, nonnegative_margin=margin,
                         eps_mixup=inp.eps_mix[r].to(dtype) if loss == 'Mixup' else None)
  grads = [q.grad.detach().double() for q in disc.g]
  losses = [out['bce_loss'].item(), out['gp_loss'].item() if 'gp_loss' in out else 0.0]
  uv = None
  if p['sn']:
    (u1, v1), (u2, v2) = disc.g_sn
    uv = (torch.cat([u1, u2]).double(), torch.cat([v1, v2]).double())
  return grads, losses, uv


def port_reward(p, inp, r, dtype):
  S, A = p['S'], p['A']
  disc = _port_disc(inp.params[r], inp.sn[r], p['sn'], False, p['rf'], dtype)
  f = inp.fields(inp.pol[r].to(dtype), S, A)
  with torch.no_grad():
    return disc.forward(f['states'], f['actions']).double(), disc.predict_reward(f['states'], f['actions']).double()


# ---- device problems ----------------------------------------------------------------------------------------------------------------------
class Device:
  """The device buffers of one problem with a guard of SENTINEL in every gap: parameter blocks of `stride` floats (the live layout of
  replica r's width first), u / v rows longer than H + 1 / d + H, and batch replicas `replica_stride` floats apart."""

  def __init__(self, p, inp, stride, u_stride, v_stride, params=None, u=None, v=None):
    dev, NB, d, B = DEV, len(inp.Hs), inp.d, p['B']
    self.p, self.inp, self.stride = p, inp, stride
    self.live = torch.zeros(NB, stride, dtype=torch.bool)
    prm = torch.full((NB, stride), SENTINEL, dtype=torch.float64)
    for r, H in enumerate(inp.Hs):
      L = _layout(d, H)
      for key, t in zip(('w1', 'b1', 'w2', 'b2'), inp.params[r]):
        prm[r, L[key]:L[key] + t.numel()] = t.flatten()
        self.live[r, L[key]:L[key] + t.numel()] = True
    self.params = params if params is not None else torch.empty(NB, stride, device=dev)
    self.params.copy_(prm)
    self.m = torch.where(self.live, 0.0, SENTINEL).float().to(dev)
    self.v = self.m.clone()
    self.u = self.vv = None
    if p['sn']:
      uu, vv = torch.full((NB, u_stride), SENTINEL, dtype=torch.float64), torch.full((NB, v_stride), SENTINEL, dtype=torch.float64)
      for r, H in enumerate(inp.Hs):
        u1, v1, u2, v2 = inp.sn[r]
        uu[r, :H + 1], vv[r, :d + H] = torch.cat([u1, u2]), torch.cat([v1, v2])
      self.u = u if u is not None else torch.empty(NB, u_stride, device=dev)
      self.vv = v if v is not None else torch.empty(NB, v_stride, device=dev)
      self.u.copy_(uu)
      self.vv.copy_(vv)
    self.step = torch.zeros(1, dtype=torch.int64, device=dev)
    self.rs = B * inp.row + 4  # batch replica stride: 16-byte aligned, not B * row
    self.pol, self.exp = (self._batch(x) for x in (inp.pol, inp.exp))
    self.eps_gp, self.eps_mix = inp.eps_gp.float().to(dev), inp.eps_mix.float().to(dev)
    self.losses = torch.full((NB, 2), SENTINEL, device=dev)
    self.inputs = [t.clone() for t in (self.pol, self.exp, self.eps_gp, self.eps_mix)]
    self.state0 = [None if t is None else t.clone() for t in (self.params, self.m, self.v, self.u, self.vv, self.step, self.losses)]

  def _batch(self, x):
    NB, B, row = x.shape
    buf = torch.full((NB, self.rs), SENTINEL, dtype=torch.float64)
    buf[:, :B * row] = x.reshape(NB, -1)
    return buf.float().to(DEV)

  def reset(self):
    for t, t0 in zip((self.params, self.m, self.v, self.u, self.vv, self.step, self.losses), self.state0):
      if t is not None: t.copy_(t0)

  def batch_struct(self, buf):
    from il_b200 import _lib
    b = _lib.Batch()
    b.rows, b.replica_stride, b.B, b.S, b.A, b.row = buf.data_ptr(), self.rs, self.p['B'], self.p['S'], self.p['A'], self.inp.row
    return b

  def gail_struct(self, order=None, rf='AIRL'):
    from il_b200 import _lib
    p, g = self.p, _lib.Gail()
    g.g.params, g.g.stride, g.g.n_layers, g.g.activation = self.params.data_ptr(), self.stride, 2, _lib.ACT['relu']
    g.g.dims[0], g.g.dims[1], g.g.dims[2] = self.inp.d, max(self.inp.Hs), 1
    if p['sn']: g.u, g.v, g.u_stride, g.v_stride = self.u.data_ptr(), self.vv.data_ptr(), self.u.stride(0), self.vv.stride(0)
    g.state_only, g.reward_function = int(p['state_only']), _lib.REWARD[rf]
    if order is not None:  # one width class over a slice of the replicas
      g.n_width_classes, g.width_class_H[0], g.width_class_begin[0], g.replica_order = 1, max(self.inp.Hs), 0, order.data_ptr()
    return g

  def update_args(self, gail, R, eps_gp=True, eps_mix=True, loss=None):
    from il_b200 import _lib
    p, a = self.p, _lib.GailUpdateArgs()
    loss = loss or p['loss']
    a.disc, a.policy, a.expert = gail, self.batch_struct(self.pol), self.batch_struct(self.exp)
    o = a.opt
    o.m, o.v, o.step, o.lr, o.beta1, o.beta2, o.eps, o.weight_decay = self.m.data_ptr(), self.v.data_ptr(), self.step.data_ptr(), LR, BETAS[0], BETAS[1], ADAM_EPS, WD
    a.eps_gp = self.eps_gp.data_ptr() if eps_gp and p['gp'] > 0 else None
    a.eps_mix = self.eps_mix.data_ptr() if eps_mix and loss == 'Mixup' else None
    a.R, a.loss_function, a.training = R, _lib.LOSS['PUGAIL' if loss.startswith('PUGAIL') else loss], 1
    a.grad_penalty, a.entropy_bonus, a.pos_class_prior = p['gp'], p['ent'], PRIOR
    a.nonnegative_margin = MARGIN.get(loss, float('inf'))
    a.out_losses = self.losses.data_ptr()
    return a

  def check_untouched(self, active):
    """Inputs, padding, u / v slots past each replica's vectors and every replica outside `active`."""
    for before, after, name in zip(self.inputs, (self.pol, self.exp, self.eps_gp, self.eps_mix), ('policy rows', 'expert rows', 'eps_gp', 'eps_mix')):
      assert torch.equal(before, after), f'{name} modified'
    idle = [r for r in range(len(self.inp.Hs)) if r not in active]
    live = self.live.to(self.params.device)
    for name, t, t0 in (('params', self.params, self.state0[0]), ('m', self.m, self.state0[1]), ('v', self.v, self.state0[2])):
      assert torch.equal(t[~live], t0[~live]), f'{name}: {int((t[~live] != t0[~live]).sum())} stride-padding floats written'
      for r in idle: assert torch.equal(t[r], t0[r]), f'{name}: replica {r}, outside the call, written'
    if self.u is not None:
      d = self.inp.d
      for r, H in enumerate(self.inp.Hs):
        keep_u, keep_v = (slice(0, None), slice(0, None)) if r in idle else (slice(H + 1, None), slice(d + H, None))
        assert torch.equal(self.u[r, keep_u], self.state0[3][r, keep_u]), f'u: replica {r} (H = {H}) written outside its {H + 1} slots'
        assert torch.equal(self.vv[r, keep_v], self.state0[4][r, keep_v]), f'v: replica {r} (H = {H}) written outside its {d + H} slots'
    for r in idle: assert (self.losses[r] == SENTINEL).all(), f'out_losses of replica {r}, outside the call, written'


def _view(flat, d, H):
  L = _layout(d, H)
  return [flat[L['w1']:L['w1'] + H * d].view(H, d), flat[L['b1']:L['b1'] + H], flat[L['w2']:L['w2'] + H].view(1, H), flat[L['b2']:L['b2'] + 1]]


def _ulp32(x):
  a = x.abs().float()
  return (torch.nextafter(a, torch.full_like(a, float('inf'))) - a).double()


def check_update(dv, active, tag=''):
  """Gradient, v, AdamW step, losses and u / v of every replica the call ran against float64."""
  p, inp, d = dv.p, dv.inp, dv.inp.d
  assert int(dv.step.item()) == 1, f'step counter {int(dv.step.item())} after one update'
  w1c, w2c = np.float32(1 - BETAS[0]), np.float32(1 - BETAS[1])
  names = ('dW1', 'db1', 'dw2', 'db2')
  for r in active:
    H = inp.Hs[r]
    what = f'{tag}replica {r} (H = {H})'
    m, v, prm = (_view(t[r].double().cpu(), d, H) for t in (dv.m, dv.v, dv.params))
    p0 = inp.params[r]
    g = [t / float(w1c) for t in m]
    f64, f32 = port_update(p, inp, r, torch.float64), port_update(p, inp, r, torch.float32)
    step_size, bc2 = LR / (1 - BETAS[0]), math.sqrt(1 - BETAS[1])
    for i, name in enumerate(names):
      _assert_vs_f64(g[i].numpy(), f64[0][i].numpy(), f32[0][i].numpy(), f'{name} {what}')
      # v = (1 - beta2) g^2 of the same fp32 gradient: a few roundings apart
      vg = v[i] / float(w2c)
      err = (vg - g[i] ** 2).abs()
      assert (err <= 1e-6 * g[i] ** 2).all(), f'{name} {what}: v / (1 - beta2) differs from g^2 by up to {float(err.max()):.3e}'
      term = step_size * m[i] / (v[i].sqrt() / bc2 + ADAM_EPS)
      ref = p0[i] * (1 - LR * WD) - term
      bound = 3 * _ulp32(ref) + 16 * U * term.abs()
      err = (prm[i] - ref).abs()
      assert (err <= bound).all(), f'{name} {what}: parameter off the AdamW step of its own m, v by {float((err / bound).max()):.2f}x the bound'
    got = dv.losses[r].double().cpu()
    _assert_vs_f64(got[0].item(), f64[1][0], f32[1][0], f'{p["loss"]} loss {what}')
    if p['gp'] > 0: _assert_vs_f64(got[1].item(), f64[1][1], f32[1][1], f'gradient-penalty loss {what}')
    else: assert got[1].item() == 0.0, f'gradient-penalty loss {got[1].item()} without a penalty ({what})'
    if p['sn']:
      for name, t, n, i in (('u', dv.u, H + 1, 0), ('v', dv.vv, d + H, 1)):
        _assert_vs_f64(t[r, :n].double().cpu().numpy(), f64[2][i].numpy(), f32[2][i].numpy(), f'spectral-norm {name} {what}')


def _prepare_update(p, inp, active):
  inp.clear_kinks(p, active)
  for r in active:
    for z, _, _ in inp.forwards(p, r): assert z.abs().min() >= KINK, 'a hidden pre-activation at the ReLU kink'
    if p['loss'].startswith('PUGAIL'):
      inner, margin = inp.pugail_inner(p, r), MARGIN[p['loss']]
      assert abs(inner + margin) > CLAMP_GAP, f'replica {r}: PUGAIL clamp {inner:.3e} within {CLAMP_GAP} of -margin: change the seed'
      if margin < float('inf'): assert inner < -margin, f'replica {r}: the clamp is not active ({inner:.3e}): change the seed'


def _seed(p): return p['S'] * 7919 + p['A'] * 131 + p['H'] * 17 + p['B'] + 3 * LOSSES.index(p.get('loss', 'BCE')) + int(p['sn'])


def _run(dv, call, expect_launches):
  import il_b200
  from il_b200 import _lib
  launches = []
  def fn():
    before = il_b200.launch_count()
    _lib.check(call())
    launches.append(il_b200.launch_count() - before)
  for _ in range(3):  # now and then a trace misses one of the call's kernels (the launch counter still shows it): take it again
    names = kernels_of(fn, attempts=3, setup=dv.reset)
    if len(names) >= expect_launches: break
  assert set(launches) == {expect_launches}, f'library launches per call: {launches}'
  return names


def _set_tiled(v):
  from il_b200 import _lib
  _lib.set_option('gail_tiled', v)


@pytest.mark.parametrize('p', ROUTES)
def test_gail_route(p):
  from il_b200 import _lib
  S, A, H, B = p['S'], p['A'], p['H'], p['B']
  NB, R = 3, 2
  active = [2, 0] if p['order'] else [0, 1]
  inp = Inputs(p, [H] * NB, seed=_seed(p))
  d = inp.d
  if p['kind'] == 'update': _prepare_update(p, inp, active)
  dv = Device(p, inp, _layout(d, H)['total'] + 12, H + 4, d + H + 3)
  order = torch.tensor(active, dtype=torch.int32, device=DEV) if p['order'] else None
  gail = dv.gail_struct(order, p.get('rf', 'AIRL'))
  try:
    _set_tiled(p['tiled'])
    if p['kind'] == 'update':
      a = dv.update_args(gail, R)
      names = _run(dv, lambda: _lib.lib().il_gail_update(_lib.handle(), C.byref(a), _lib.stream()), 2)
    else:
      ld = p['ld']
      rs = B * ld + 3  # padded replica stride of the reward output
      reward = torch.full((NB * rs + 1, ), SENTINEL, device=DEV)
      logits = torch.full((NB, B), SENTINEL, device=DEV)
      b = dv.batch_struct(dv.pol)
      base_reset = dv.reset
      def reset():
        base_reset()
        reward.fill_(SENTINEL)
        logits.fill_(SENTINEL)
      dv.reset = reset
      names = _run(dv, lambda: _lib.lib().il_gail_reward(_lib.handle(), C.byref(gail), R, C.byref(b), reward.data_ptr(), rs, ld, logits.data_ptr(), _lib.stream()), 1)
  finally:
    _set_tiled(1)
  expect = [TICK, p['kernel']] if p['kind'] == 'update' else [p['kernel']]
  assert names == expect, f'expected {expect}, the call ran {names}'
  if p['kind'] == 'update':
    check_update(dv, active)
    dv.check_untouched(active)
    return
  # reward rows: eval-mode forward; parameters, u / v and the batch are read only
  for name, t, t0 in zip(('params', 'u', 'v'), (dv.params, dv.u, dv.vv), (dv.state0[0], dv.state0[3], dv.state0[4])):
    if t is not None: assert torch.equal(t, t0), f'il_gail_reward wrote {name}'
  dv.check_untouched(active)
  written = torch.zeros_like(reward, dtype=torch.bool)
  for r in active:
    idx = r * rs + torch.arange(B, device=DEV) * p['ld']
    written[idx] = True
    f64, f32 = port_reward(p, inp, r, torch.float64), port_reward(p, inp, r, torch.float32)
    _assert_vs_f64(logits[r].double().cpu().numpy(), f64[0].numpy(), f32[0].numpy(), f'logits replica {r}')
    _assert_vs_f64(reward[idx].double().cpu().numpy(), f64[1].numpy(), f32[1].numpy(), f'{p["rf"]} reward replica {r}')
  assert (reward[~written] == SENTINEL).all(), f'{int((reward[~written] != SENTINEL).sum())} reward floats outside the B x ld x R output written'
  for r in range(NB):
    if r not in active: assert (logits[r] == SENTINEL).all(), f'logits of replica {r}, outside the call, written'


def test_gail_width_classes():
  """A GAILDiscriminator with per-replica widths (128, 32, 48) on halfcheetah (d = 24): one call runs gail_update_tiled_kernel<1> (32),
  gail_update_kernel<16> (48) and gail_update_tiled_kernel<4> (128) over replica_order [1, 2, 0]; each replica against its own float64 update,
  the rest of each replica's block (the widest stride) untouched."""
  import il_b200
  from il_b200 import _lib
  from il_b200.config import Config, load_config
  S, A, B, widths = 18, 6, 256, [128, 32, 48]
  p = dict(kind='update', S=S, A=A, H=max(widths), B=B, loss='BCE', gp=1.0, ent=0.05, sn=True, state_only=False)
  inp = Inputs(p, widths, seed=2024)
  active = [0, 1, 2]
  _prepare_update(p, inp, active)
  icfg = Config(dict(load_config(['algorithm=GAIL']).imitation, spectral_norm=True))
  disc = il_b200.GAILDiscriminator(S, A, icfg, 0.97, replicas=3, hidden_size=widths, device=DEV)
  assert disc.hidden_size_r == widths and disc._replica_order.tolist() == [1, 2, 0]
  dv = Device(p, inp, disc.mlp.flat.size(1), disc.u.size(1), disc.v.size(1), params=disc.mlp.flat, u=disc.u, v=disc.v)
  a = dv.update_args(disc.c_struct(), 3)
  names = _run(dv, lambda: _lib.lib().il_gail_update(_lib.handle(), C.byref(a), _lib.stream()), 4)
  assert names == [TICK, tiled(1), untiled(16), tiled(4)], names
  check_update(dv, active)
  dv.check_untouched(active)


@pytest.mark.parametrize('what,env,H,state_only,loss,gp,eps_mix,text', [
  ('hidden_times_input', 'ant', 256, False, 'BCE', 1.0, True, 'exceeds the kernel limit 16384'),
  ('hidden_size', 'hopper', 260, False, 'BCE', 1.0, True, 'hidden size 260 exceeds the kernel limit 256'),
  ('state_only_grad_penalty', 'hopper', 64, True, 'BCE', 1.0, True, 'grad_penalty with a state-only discriminator'),
  ('mixup_without_eps_mix', 'hopper', 64, False, 'Mixup', 0.0, False, 'Mixup needs eps_mix'),
])
def test_gail_update_refused(what, env, H, state_only, loss, gp, eps_mix, text):
  import il_b200
  from il_b200 import _lib
  S, A = ENV[env]
  p = dict(kind='update', S=S, A=A, H=H, B=64, loss=loss, gp=gp, ent=0.0, sn=True, state_only=state_only)
  inp = Inputs(p, [H] * 2, seed=7)
  dv = Device(p, inp, _layout(inp.d, H)['total'], H + 1, inp.d + H)
  a = dv.update_args(dv.gail_struct(), 2, eps_mix=eps_mix)
  before = il_b200.launch_count()
  rc = _lib.lib().il_gail_update(_lib.handle(), C.byref(a), _lib.stream())
  torch.cuda.synchronize()
  assert rc != 0, 'the call was accepted'
  assert text in _lib.last_error(), _lib.last_error()
  assert il_b200.launch_count() == before, 'a refused call launched a kernel'
  for t, t0 in zip((dv.params, dv.m, dv.v, dv.u, dv.vv, dv.step, dv.losses), dv.state0):
    assert torch.equal(t, t0), 'a refused call wrote its state'
