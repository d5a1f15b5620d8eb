"""Sweeps over the GAIL discriminator's choices as replicas of one program: the fused update / reward kernels with per-replica loss function,
reward function, spectral norm, prior and margin against uniform calls (bitwise, slice by slice), the device Beta sampler, sweep Trainers
against the uniform runs of their jobs, a 3-replica group against the oracle loop, Mixup with alpha != 1 under CUDA graphs, and the multirun
command line."""
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LOSSES = ['BCE', 'Mixup', 'PUGAIL', 'Mixup', 'PUGAIL', 'BCE', 'PUGAIL']
SNS = [True, False, True, True, False, False, True]
PRIORS = [0.7, 0.5, 0.3, 0.9, 0.7, 0.2, 0.8]
MARGINS = [float('inf'), 0.0, 0.0, 1.0, float('inf'), 0.5, 0.3]  # margin 0 gates the PUGAIL policy term off for some batches
REWARDS = ['AIRL', 'GAIL', 'FAIRL', 'GAIL', 'AIRL', 'FAIRL', 'AIRL']


# ---- 1. kernels -------------------------------------------------------------------------------------------------------------------
def _icfg(H, **kw):
  from il_b200.config import Config, load_config
  c = load_config(['algorithm=GAIL', f'imitation.discriminator.hidden_size={H}']).imitation
  return Config(dict(c, **kw))


def _batch(R, B, S, A, seed):
  from il_b200 import TransitionBatch
  from il_b200._lib import py_row_layout
  off, row = py_row_layout(S, A)
  g = torch.Generator(device='cuda').manual_seed(seed)
  rows = torch.randn(R, B, row, device='cuda', generator=g)
  rows[..., off['weights']] = torch.rand(R, B, device='cuda', generator=g) + 0.5
  return TransitionBatch(rows.contiguous(), S, A, False)


def _disc_pair(R, S, A, H, r, seed=0):
  """The per-replica discriminator and the uniform one with replica r's choices for every replica, holding the same parameters / u / v."""
  from il_b200 import GAILDiscriminator
  torch.manual_seed(seed)
  sweep = GAILDiscriminator(S, A, _icfg(H), 0.97, replicas=R, spectral_norm=SNS[:R], reward_function=REWARDS[:R], device='cuda')
  uni = GAILDiscriminator(S, A, _icfg(H), 0.97, replicas=R, spectral_norm=SNS[r], reward_function=REWARDS[r], device='cuda')
  uni.mlp.flat.copy_(sweep.mlp.flat)
  if SNS[r]: uni.u.copy_(sweep.u); uni.v.copy_(sweep.v)
  return sweep, uni


def _update_matches_uniform_calls(S, A, H, tiled, training, gp, R=7, B=32, steps=2):
  import il_b200
  from il_b200 import _lib
  pol, exp = _batch(R, B, S, A, 1), _batch(R, B, S, A, 2)
  eps_gp, eps_mix = torch.rand(R, B, device='cuda'), torch.rand(R, B, device='cuda')
  f = lambda x: torch.tensor(x, dtype=torch.float32, device='cuda')
  _lib.set_option('gail_tiled', tiled)
  try:
    sweep, _ = _disc_pair(R, S, A, H, 0)
    sweep.train(training)
    opt = il_b200.AdamW(sweep.parameters(), lr=3e-3, weight_decay=0.1)
    cfg = _icfg(H, loss_function=LOSSES[:R], pos_class_prior=f(PRIORS[:R]), nonnegative_margin=f(MARGINS[:R]), grad_penalty=gp, entropy_bonus=0.05)
    losses = torch.zeros(R, 2, device='cuda')
    for _ in range(steps): il_b200.adversarial_imitation_update(None, sweep, pol, exp, opt, cfg, eps_gp=eps_gp, eps_mix=eps_mix, out_losses=losses)
    for r in range(R):
      _, uni = _disc_pair(R, S, A, H, r)
      uni.train(training)
      uopt = il_b200.AdamW(uni.parameters(), lr=3e-3, weight_decay=0.1)
      ucfg = _icfg(H, loss_function=LOSSES[r], pos_class_prior=PRIORS[r], nonnegative_margin=MARGINS[r], grad_penalty=gp, entropy_bonus=0.05)
      ul = torch.zeros(R, 2, device='cuda')
      for _ in range(steps): il_b200.adversarial_imitation_update(None, uni, pol, exp, uopt, ucfg, eps_gp=eps_gp, eps_mix=eps_mix, out_losses=ul)
      torch.cuda.synchronize()
      for name, a, b in (('params', sweep.mlp.flat, uni.mlp.flat), ('m', opt.exp_avg, uopt.exp_avg), ('v', opt.exp_avg_sq, uopt.exp_avg_sq), ('losses', losses, ul)):
        a, b = a.reshape(R, -1)[r], b.reshape(R, -1)[r]
        assert torch.equal(a, b), f'replica {r} ({LOSSES[r]}, sn={SNS[r]}): {name} differs by {float((a - b).abs().max())}'
      if SNS[r]: assert torch.equal(sweep.u[r], uni.u[r]) and torch.equal(sweep.v[r], uni.v[r]), f'replica {r}: u / v'
      else: assert torch.equal(sweep.u[r], torch.zeros_like(sweep.u[r])) and torch.equal(sweep.v[r], torch.zeros_like(sweep.v[r])), f'replica {r} touched its u / v'
  finally:
    _lib.set_option('gail_tiled', 1)


@pytest.mark.parametrize('H', [32, 64, 128])  # d = 23: gail_update_tiled_kernel<1>, <2>, <4>
@pytest.mark.parametrize('training', [1, 0])
@pytest.mark.parametrize('gp', [0.0, 1.0])
def test_tiled_update_per_replica_equals_uniform_calls(H, training, gp):
  _update_matches_uniform_calls(17, 6, H, 1, training, gp)


# gail_tiled off (gail_update_kernel<4>, <16>), and ant-sized inputs (d = 35 > 32: the tiled kernel does not take them; <16>, <32>)
@pytest.mark.parametrize('S,A,H,tiled', [(17, 6, 32, 0), (17, 6, 64, 0), (27, 8, 64, 1), (27, 8, 128, 1)])
@pytest.mark.parametrize('training', [1, 0])
@pytest.mark.parametrize('gp', [0.0, 1.0])
def test_untiled_update_per_replica_equals_uniform_calls(S, A, H, tiled, training, gp):
  _update_matches_uniform_calls(S, A, H, tiled, training, gp)


@pytest.mark.parametrize('tiled', [1, 0])
def test_reward_per_replica_equals_uniform_calls(tiled):
  from il_b200 import _lib
  R, B, S, A, H = 7, 48, 17, 6, 64
  batch = _batch(R, B, S, A, 3)
  _lib.set_option('gail_tiled', tiled)
  try:
    sweep, _ = _disc_pair(R, S, A, H, 0)
    sweep.u.normal_()  # stored vectors as after training, so that sigma != 1
    sweep.v.normal_()
    sweep.eval()
    out = sweep._run(batch, want_logits=True)
    for r in range(R):
      _, uni = _disc_pair(R, S, A, H, r)
      if SNS[r]: uni.u.copy_(sweep.u); uni.v.copy_(sweep.v)
      uni.eval()
      ref = uni._run(batch, want_logits=True)
      torch.cuda.synchronize()
      for k in ('reward', 'logits'): assert torch.equal(out[k][r], ref[k][r]), f'replica {r} ({REWARDS[r]}, sn={SNS[r]}): {k}'
  finally:
    _lib.set_option('gail_tiled', 1)


# ---- 2. the Beta sampler ----------------------------------------------------------------------------------------------------------
def _beta(alphas, n, seed=7, stream_id=8, counter=5):
  from il_b200.models import _RNG
  rng = _RNG(seed)
  rng.counter = torch.full((1, ), counter, dtype=torch.int64, device='cuda')
  a = torch.tensor(alphas, dtype=torch.float32, device='cuda')
  out = rng.beta((len(alphas), n), a, 'cuda', stream_id=stream_id)
  torch.cuda.synchronize()
  return out, int(rng.counter)


def test_beta_at_alpha_one_is_the_uniform_fill():
  from il_b200.models import _RNG
  n = 1001  # replica boundaries fall inside Philox groups of 4
  out, ctr = _beta([1.0, 0.4, 1.0, 3.0], n)
  rng = _RNG(7)
  rng.counter = torch.full((1, ), 5, dtype=torch.int64, device='cuda')
  uni = rng.uniform((4, n), 'cuda', stream_id=8)
  assert int(rng.counter) == ctr == 5 + (4 * n + 3) // 4
  assert torch.equal(out[0], uni[0]) and torch.equal(out[2], uni[2])
  assert not torch.equal(out[1], uni[1])


def test_beta_slice_depends_only_on_its_own_alpha():
  a, _ = _beta([0.4, 2.0, 8.0, 1.0, 0.1], 999)
  b, _ = _beta([0.4, 8.0, 1.0, 0.1, 2.0], 999)
  assert torch.equal(a[0], b[0])
  assert not torch.equal(a[1], b[4])  # the same alpha at another position: other elements, other draws


def test_beta_graph_replay_equals_eager():
  from il_b200.models import _RNG
  alphas = torch.tensor([0.1, 0.4, 1.0, 2.0, 8.0], dtype=torch.float32, device='cuda')
  rng = _RNG(11)
  rng.counter = torch.zeros(1, dtype=torch.int64, device='cuda')
  out = torch.empty(5, 4000, device='cuda')
  eager = [rng.beta(None, alphas, 'cuda', out=out).clone() for _ in range(2)]
  rng.counter.zero_()
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(s):
    rng.beta(None, alphas, 'cuda', out=out)  # warm-up outside the capture
  torch.cuda.current_stream().wait_stream(s)
  rng.counter.zero_()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    rng.beta(None, alphas, 'cuda', out=out)
  rng.counter.zero_()
  for e in eager:
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, e)


def test_beta_distribution():
  from scipy import stats
  alphas, n = [0.1, 0.4, 2.0, 8.0], 1 << 20
  out, _ = _beta(alphas, n, seed=2024, stream_id=3, counter=0)
  x = out.cpu().numpy()
  assert np.isfinite(x).all() and (x >= 0).all() and (x <= 1).all()
  rs = np.random.RandomState(0)
  for i, a in enumerate(alphas):
    d = stats.beta(a, a)
    xi = x[i].astype(np.float64)
    # At alpha 0.1 about 9 % of the mass lies within 3e-8 of 1 (float32 rounds it to 1) and 1 % within 1e-16 (float64 cannot hold it apart
    # from 1), so the test runs on the folded distance z = min(x, 1 - x) ~ 2 F on [0, 1/2] by the symmetry of Beta(a, a) (1 - x is exact for a
    # float32 x >= 1/2), and places each draw inside its float32 rounding interval by the distribution itself (inverse CDF of a uniform
    # between the CDFs of the interval ends) before scipy.stats.kstest; the two halves must be balanced.
    lo = np.clip((xi + np.nextafter(x[i], np.float32(-1)).astype(np.float64)) / 2, 0, 1)
    hi = np.clip((xi + np.nextafter(x[i], np.float32(2)).astype(np.float64)) / 2, 0, 1)
    upper = xi >= 0.5
    zlo, zhi = np.clip(np.where(upper, 1 - hi, lo), 0, 0.5), np.clip(np.where(upper, 1 - lo, hi), 0, 0.5)
    G = lambda z: 2 * d.cdf(z)
    z = d.ppf((G(zlo) + rs.uniform(size=n) * (G(zhi) - G(zlo))) / 2)
    p = stats.kstest(z, G).pvalue
    assert p > 1e-4, f'alpha {a}: KS p = {p}'
    assert abs(upper.mean() - 0.5) < 5 * 0.5 / np.sqrt(n), f'alpha {a}: {upper.mean()} of the draws above 1/2'
    m, v, k = (float(t) for t in d.stats(moments='mvk'))
    assert abs(xi.mean() - m) < 5 * np.sqrt(v / n), f'alpha {a}: mean {xi.mean()}'
    assert abs(xi.var() - v) < 5 * v * np.sqrt((k + 2) / n), f'alpha {a}: variance {xi.var()} vs {v}'


# ---- 3. loops: a group's job blocks equal the uniform runs of their jobs ---------------------------------------------------------
def _buffers(tr):
  out = dict(actor=tr.actor.mlp.flat, critic=tr.critic.mlp.flat, target=tr.target_critic.mlp.flat, log_alpha=tr.log_alpha, rewards=tr.batch.rows, gail_losses=tr.gail_losses,
             disc=tr.discriminator.parameters()[0], disc_m=tr.discriminator_optimiser.exp_avg, disc_v=tr.discriminator_optimiser.exp_avg_sq, **tr.sac_out)
  for n in ('u', 'v'):
    if getattr(tr.discriminator, n, None) is not None: out['sn_' + n] = getattr(tr.discriminator, n)
  return {k: v.detach().reshape(tr.R, -1).clone() for k, v in out.items()}


def _make(base, R, per_replica=None, values=None):
  from il_b200.config import load_config
  from il_b200.train import Trainer
  cfg = load_config(base + [f'replicas={R}'] + [f'{k}={v!r}' for k, v in (values or {}).items()])
  return Trainer(cfg, replicas=R, per_replica=per_replica)


def _drive(tr, steps):
  for _ in range(steps): tr.train_step()
  torch.cuda.synchronize()


def _sweep_matches_uniform_runs(base, per_job, R=1, steps=40):
  J = len(next(iter(per_job.values())))
  Rt = J * R
  sweep = _make(base, Rt, per_replica={k: [v for v in vals for _ in range(R)] for k, vals in per_job.items()})
  gp_on, mix_on = sweep._grad_penalty_on, sweep._mixup_on
  assert mix_on
  _drive(sweep, steps)
  got = _buffers(sweep)
  sn = sweep.discriminator.spectral_norm_r
  del sweep
  for j in range(J):
    uni = _make(base, Rt, values={k: vals[j] for k, vals in per_job.items()})
    # the group draws the Mixup (and gradient-penalty) noise for all its replicas from one device noise stream: the uniform run of a job
    # without Mixup draws it too, so both see the same noise afterwards
    uni._grad_penalty_on, uni._mixup_on = gp_on, mix_on
    _drive(uni, steps)
    ref = _buffers(uni)
    blk = slice(j * R, (j + 1) * R)
    for k, v in ref.items():
      assert torch.equal(got[k][blk], v[blk]), f'job {j} ({ {k_: vals[j] for k_, vals in per_job.items()} }): {k} differs (max |diff| {float((got[k][blk] - v[blk]).abs().max())})'
    if sn is not None and not sn[j * R]: assert not got['sn_u'][blk].any() and not got['sn_v'][blk].any(), f'job {j} touched its u / v'
    del uni


SMALL = ['algorithm=GAIL', 'env=hopper', 'steps=40', 'training.start=20', 'training.batch_size=32', 'imitation.trajectories=2', 'reinforcement.actor.hidden_size=64',
         'reinforcement.critic.hidden_size=64', 'cuda_graphs=true', 'device_rng=true', 'seed=5', 'evaluation.episodes=1', 'imitation.mixup_alpha=0.4']


def _grid():
  jobs = [(l, rf, sn) for l in ('BCE', 'Mixup', 'PUGAIL') for rf in ('GAIL', 'AIRL', 'FAIRL') for sn in (True, False)]
  return {'imitation.loss_function': [j[0] for j in jobs], 'imitation.discriminator.reward_function': [j[1] for j in jobs], 'imitation.spectral_norm': [j[2] for j in jobs]}


def test_choice_grid_blocks_equal_uniform_runs():
  _sweep_matches_uniform_runs(SMALL, _grid())


def test_choice_group_blocks_equal_uniform_runs_at_the_benchmarked_configuration():
  base = ['algorithm=GAIL', 'env=hopper', 'training.start=20', 'training.batch_size=256', 'imitation.trajectories=2', 'gemm_mode=tf32x3', 'cuda_graphs=true', 'seed=5']
  _sweep_matches_uniform_runs(base, {'imitation.loss_function': ['BCE', 'Mixup', 'PUGAIL', 'Mixup'], 'imitation.discriminator.reward_function': ['AIRL', 'GAIL', 'FAIRL', 'AIRL'],
                                     'imitation.spectral_norm': [True, False, True, False], 'imitation.mixup_alpha': [0.4, 0.4, 0.4, 1.0],
                                     'imitation.pos_class_prior': [0.7, 0.7, 0.4, 0.7], 'imitation.nonnegative_margin': [float('inf'), float('inf'), 0.3, float('inf')]})


# ---- 4. semantics: each replica of a group against the oracle loop built with its values --------------------------------------------
class _Injected:
  def __init__(self, seq): self.seq = seq
  def _pop(self, k): return self.seq[k].pop(0)
  def reset_u(self): return self._pop('reset_u')
  def act_eps(self, A): return self._pop('act_eps')
  def policy_indices(self, mem, n): return self._pop('idx_pol')
  def expert_indices(self, mem, n): return self._pop('idx_exp')
  def gp_eps(self, B): return self._pop('eps_gp')
  def mixup_eps(self, B, alpha): return self._pop('eps_mix')
  def sac_eps(self, B, A): return self._pop('eps_next'), self._pop('eps_new')


def test_choice_group_replicas_match_the_oracle_with_their_values():
  from il_b200.config import load_config
  from il_b200.train import Trainer
  from oracle import loop as oloop
  R, B, H, steps, start = 3, 32, 64, 60, 30
  vals = {'imitation.loss_function': ['BCE', 'Mixup', 'PUGAIL'], 'imitation.discriminator.reward_function': ['AIRL', 'GAIL', 'FAIRL'], 'imitation.spectral_norm': [True, False, True],
          'imitation.mixup_alpha': [1.0, 0.4, 1.0], 'imitation.nonnegative_margin': [float('inf'), float('inf'), 0.3]}
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=2',
                     f'reinforcement.actor.hidden_size={H}', f'reinforcement.critic.hidden_size={H}', 'cuda_graphs=false', 'gemm_mode=fp32', f'replicas={R}', 'seed=3'])
  tr = Trainer(cfg, replicas=R, per_replica=vals)
  tr.inject = True
  rs = np.random.RandomState(123)
  S, A, obs = tr.S, tr.A, tr.env.obs
  expert_raw = tr.env.synthesize_raw_dataset(5)
  loops = []
  for r in range(R):
    d, Hd, sn = S + A, tr.discriminator.mlp.dims[1], vals['imitation.spectral_norm'][r]
    init = dict(actor=tr.actor.mlp.export_params(r, 0), twin=[tr.critic.mlp.export_params(r, 0), tr.critic.mlp.export_params(r, 1)], g=tr.discriminator.mlp.export_params(r, 0))
    if sn: init['sn'] = [(tr.discriminator.u[r, :Hd].cpu().clone(), tr.discriminator.v[r, :d].cpu().clone()), (tr.discriminator.u[r, Hd:Hd + 1].cpu().clone(), tr.discriminator.v[r, d:d + Hd].cpu().clone())]
    im = dict(loss_function=vals['imitation.loss_function'][r], reward_function=vals['imitation.discriminator.reward_function'][r], spectral_norm=sn,
              mixup_alpha=vals['imitation.mixup_alpha'][r], nonnegative_margin=vals['imitation.nonnegative_margin'][r])
    loops.append(oloop.OracleLoop('GAIL', 'hopper', seed=3 + r, batch_size=B, start=start, memory_size=tr.cfg.memory.size, hidden_size=H, trajectories=2, expert_raw=expert_raw, init=init,
                                  mix_expert_data=cfg.imitation.mix_expert_data, imitation=im))
  Ne = tr.expert_memory.size
  u0 = rs.uniform(size=(R, obs)).astype(np.float32)
  tr.env.batch.reset(torch.from_numpy(u0).cuda(), tr.state)
  for r, lp in enumerate(loops): lp.state, lp.t = lp.env.reset(torch.from_numpy(u0[r])), 0
  err, per = {}, {}

  def e(k, r, x):
    err[k], per[(k, r)] = max(err.get(k, 0), x), max(per.get((k, r), 0), x)

  for step in range(1, steps + 1):
    noise = dict(act_eps=rs.standard_normal((R, A)).astype(np.float32), reset_u=rs.uniform(size=(R, obs)).astype(np.float32), eps_gp=rs.uniform(size=(R, B)).astype(np.float32),
                 eps_mix=rs.beta(0.4, 0.4, size=(R, B)).astype(np.float32), eps_next=rs.standard_normal((R, B, A)).astype(np.float32),
                 eps_new=rs.standard_normal((R, B, A)).astype(np.float32))
    upd = step >= start
    if upd:
      noise['idx_pol'] = np.stack([rs.randint(0, max(lp.memory.idx - 1, 1), size=B) for lp in loops]).astype(np.int32)
      noise['idx_exp'] = rs.randint(0, Ne - 1, size=(R, B)).astype(np.int32)
    tr.eps_act.copy_(torch.from_numpy(noise['act_eps']))
    tr.u_reset.copy_(torch.from_numpy(noise['reset_u']))
    if upd:
      for k, t in (('idx_pol', tr.idx_pol), ('idx_exp', tr.idx_exp), ('eps_gp', tr.eps_gp), ('eps_mix', tr.eps_mix), ('eps_next', tr.eps_next), ('eps_new', tr.eps_new)):
        t.copy_(torch.from_numpy(noise[k]))
    tr.train_step()
    for r, lp in enumerate(loops):
      seq = {k: [torch.from_numpy(np.asarray(x[r]))] for k, x in noise.items()}
      seq['act_eps'] = [torch.from_numpy(noise['act_eps'][r:r + 1])]
      lp.noise = _Injected(seq)
      lp.run_step()
      e('state', r, float((tr.state[r].cpu() - lp.state[0]).abs().max()))
      if upd:
        e('q', r, float((tr.sac_out['q_values'][r].cpu() - lp.last['sac']['q_values']).abs().max()))
        e('reward', r, float((tr.batch['rewards'][r].cpu() - lp.last['rewards']).abs().max()))
  for r, lp in enumerate(loops):
    for i, p in enumerate(lp.agent.actor):
      e('actor', r, float((tr.actor.mlp.layer_views()[0][i][r].cpu() - p.detach()).abs().max()))
  print('choice group vs oracle', err, per)
  assert err['state'] < 2e-3, per
  assert err['q'] < 5e-3, per
  assert err['reward'] < 5e-3, per
  assert err['actor'] < 5e-4, per


# ---- 5. Mixup with alpha != 1 in a single (non-sweep) Trainer under CUDA graphs -------------------------------------------------------
def test_mixup_alpha_trainer_graph_equals_eager():
  runs = {}
  for graphs in (True, False):
    tr = _make(SMALL[:-1] + ['imitation.loss_function=Mixup', 'imitation.mixup_alpha=0.4', f'cuda_graphs={str(graphs).lower()}'], 2)
    _drive(tr, 40)
    if graphs: assert 'step+update' in tr.graphs
    runs[graphs] = _buffers(tr)
    runs[(graphs, 'eps')] = tr.eps_mix.clone()
    del tr
  for k, v in runs[True].items(): assert torch.equal(v, runs[False][k]), k
  e = runs[(True, 'eps')]
  assert torch.equal(e, runs[(False, 'eps')]) and not torch.equal(e, e.clamp(0.25, 0.75))  # Beta(0.4, 0.4) puts mass near 0 and 1


# ---- 6. the multirun command line -------------------------------------------------------------------------------------------------
def _fcnn(sizes, sn):
  from torch import nn
  layers = []
  for i in range(len(sizes) - 1):
    lin = nn.Linear(sizes[i], sizes[i + 1])
    layers.append(nn.utils.parametrizations.spectral_norm(lin) if sn else lin)
    if i < len(sizes) - 2: layers.append(nn.ReLU())
  return nn.Sequential(*layers)


def test_multirun_over_the_choice_grid_is_one_group(tmp_path):
  import subprocess
  import sys
  import yaml
  S, A, H = 12, 3, 64
  cli = ['algorithm=GAIL', 'env=hopper', 'steps=60', 'training.start=30', 'evaluation.interval=60', 'evaluation.episodes=1', 'imitation.trajectories=2', 'memory.size=100',
         'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'training.batch_size=32', 'imitation.mixup_alpha=0.4', 'seed=9']
  swept = ['imitation.loss_function=BCE,Mixup,PUGAIL', 'imitation.discriminator.reward_function=GAIL,AIRL,FAIRL', 'imitation.spectral_norm=true,false']
  res = subprocess.run([sys.executable, 'train.py', '-m', *cli, *swept, f'output_dir={tmp_path}'], cwd=ROOT, capture_output=True, text=True, timeout=900)
  assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
  assert 'in 1 group(s)' in res.stdout
  (out, ) = glob.glob(os.path.join(str(tmp_path), '*_sweeper', '*'))
  assert sorted(os.listdir(out), key=int) == [str(j) for j in range(18)]
  grid = _grid()
  from il_b200.config import load_config
  from il_b200.train import Trainer
  for j in range(18):
    d = os.path.join(out, str(j))
    ov = yaml.safe_load(open(os.path.join(d, 'overrides.yaml')))
    sn = grid['imitation.spectral_norm'][j]
    assert ov[-2] == f'imitation.spectral_norm={"true" if sn else "false"}'
    sd = torch.load(os.path.join(d, 'discriminator.pth'))
    m = torch.nn.Module()
    m.g = _fcnn([S + A, H, 1], sn)
    m.load_state_dict(sd, strict=True)  # a single run's keys and shapes for this job's spectral_norm
  uni = {}
  for j in (1, 2, 9):  # BCE/GAIL/no SN, BCE/AIRL/SN, Mixup/AIRL/no SN: one uniform 18-replica run each, the job's block compared
    values = {k: v[j] for k, v in grid.items()}
    cfg = load_config(cli + [f'{k}={str(v).lower() if isinstance(v, bool) else v}' for k, v in values.items()] + ['replicas=18', f'output_dir={tmp_path}/u'])
    tr = Trainer(cfg, replicas=18)
    tr._grad_penalty_on, tr._mixup_on = True, True
    for _ in range(cfg.steps): tr.train_step()
    torch.cuda.synchronize()
    ref = tr.discriminator.state_dict()
    sd = torch.load(os.path.join(out, str(j), 'discriminator.pth'))
    assert set(sd) == set(ref)
    for k, v in sd.items(): assert torch.equal(v.cpu(), ref[k][j].cpu()), f'job {j}: {k}'
    del tr
