"""Sweeps over the fused GAIL discriminator's hidden size as replicas of one program: the update / reward kernels with per-replica widths (one launch
per width class) against uniform discriminators of each width (bitwise, padding untouched), per-replica initialisation, sweep Trainers against
the uniform runs of their jobs, a 3-replica group against the oracle loop, and the multirun command line."""
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
W = 'imitation.discriminator.hidden_size'

WIDTHS = [64, 128, 32, 64, 128, 32, 64]
LOSSES = ['BCE', 'Mixup', 'PUGAIL', 'Mixup', 'PUGAIL', 'BCE', 'PUGAIL']
SNS = [True, False, True, True, False, False, True]
PRIORS = [0.7, 0.5, 0.3, 0.9, 0.7, 0.2, 0.8]
MARGINS = [float('inf'), 0.0, 0.0, 1.0, float('inf'), 0.5, 0.3]
REWARDS = ['AIRL', 'GAIL', 'FAIRL', 'GAIL', 'AIRL', 'FAIRL', 'AIRL']


def _icfg(**kw):
  from il_b200.config import Config, load_config
  return Config(dict(load_config(['algorithm=GAIL']).imitation, **kw))


def _batch(R, B, S, A, seed):
  from il_b200 import TransitionBatch
  from il_b200._lib import py_row_layout
  off, row = py_row_layout(S, A)
  g = torch.Generator(device='cuda').manual_seed(seed)
  rows = torch.randn(R, B, row, device='cuda', generator=g)
  rows[..., off['weights']] = torch.rand(R, B, device='cuda', generator=g) + 0.5
  return TransitionBatch(rows.contiguous(), S, A, False)


def _stride(d, H):
  from il_b200._lib import py_mlp_offsets
  return py_mlp_offsets([d, H, 1])[2]


def _sweep_disc(R, S, A, widths, seed=0):
  from il_b200 import GAILDiscriminator
  torch.manual_seed(seed)
  return GAILDiscriminator(S, A, _icfg(), 0.97, replicas=R, spectral_norm=SNS[:R], reward_function=REWARDS[:R], hidden_size=widths, device='cuda')


def _uniform_like(sweep, S, A, r):
  """A uniform discriminator of replica r's width with replica r's choices for every replica, replica r holding the sweep's parameters / u / v."""
  from il_b200 import GAILDiscriminator
  H, d = sweep.hidden_size_r[r], sweep.mlp.dims[0]
  uni = GAILDiscriminator(S, A, _icfg(), 0.97, replicas=sweep.replicas, spectral_norm=SNS[r], reward_function=REWARDS[r], hidden_size=H, device='cuda')
  assert uni.hidden_size_r is None and uni.mlp.dims[1] == H
  uni.mlp.flat[r].copy_(sweep.mlp.flat[r, :_stride(d, H)])
  if SNS[r]: uni.u[r].copy_(sweep.u[r, :H + 1]); uni.v[r].copy_(sweep.v[r, :d + H])
  return uni


def _assert_padding_zero(sweep, opt, r):
  H, d = sweep.hidden_size_r[r], sweep.mlp.dims[0]
  n = _stride(d, H)
  for name, t in (('params', sweep.mlp.flat), ('m', opt.exp_avg), ('v', opt.exp_avg_sq)):
    assert not t.reshape(sweep.replicas, -1)[r, n:].any(), f'replica {r} (width {H}): {name} padding written'
  if sweep.u is not None:
    rows = (sweep.u[r, H + 1:], sweep.v[r, d + H:]) if SNS[r] else (sweep.u[r], sweep.v[r])
    assert not rows[0].any() and not rows[1].any(), f'replica {r} (width {H}): u / v padding written'


def _update_matches_uniform(S, A, widths, tiled, training, gp, B=32, steps=2):
  import il_b200
  from il_b200 import _lib
  R = len(widths)
  pol, exp = _batch(R, B, S, A, 1), _batch(R, B, S, A, 2)
  eps_gp, eps_mix = torch.rand(R, B, device='cuda'), torch.rand(R, B, device='cuda')
  f = lambda x: torch.tensor(x, dtype=torch.float32, device='cuda')
  _lib.set_option('gail_tiled', tiled)
  try:
    sweep = _sweep_disc(R, S, A, widths)
    assert sweep.hidden_size_r == list(widths) and sweep.mlp.dims[1] == max(widths)
    sweep.train(training)
    opt = il_b200.AdamW(sweep.parameters(), lr=3e-3, weight_decay=0.1)
    cfg = _icfg(loss_function=LOSSES[:R], pos_class_prior=f(PRIORS[:R]), nonnegative_margin=f(MARGINS[:R]), grad_penalty=gp, entropy_bonus=0.05)
    losses = torch.zeros(R, 2, device='cuda')
    starts = {r: _uniform_like(sweep, S, A, r) for r in range(R)}  # the starting values, before the sweep trains
    for _ in range(steps): il_b200.adversarial_imitation_update(None, sweep, pol, exp, opt, cfg, eps_gp=eps_gp, eps_mix=eps_mix, out_losses=losses)
    assert int(opt.step_count) == steps  # one optimiser step per call, not per width class
    for r in range(R):
      H, d = widths[r], S + A
      uni = starts[r]
      uni.train(training)
      uopt = il_b200.AdamW(uni.parameters(), lr=3e-3, weight_decay=0.1)
      ucfg = _icfg(loss_function=LOSSES[r], pos_class_prior=PRIORS[r], nonnegative_margin=MARGINS[r], grad_penalty=gp, entropy_bonus=0.05)
      ul = torch.zeros(R, 2, device='cuda')
      for _ in range(steps): il_b200.adversarial_imitation_update(None, uni, pol, exp, uopt, ucfg, eps_gp=eps_gp, eps_mix=eps_mix, out_losses=ul)
      torch.cuda.synchronize()
      n = _stride(d, H)
      for name, a, b in (('params', sweep.mlp.flat, uni.mlp.flat), ('m', opt.exp_avg, uopt.exp_avg), ('v', opt.exp_avg_sq, uopt.exp_avg_sq)):
        a, b = a.reshape(R, -1)[r, :n], b.reshape(R, -1)[r]
        assert torch.equal(a, b), f'replica {r} (width {H}, {LOSSES[r]}, sn={SNS[r]}): {name} differs by {float((a - b).abs().max())}'
      assert torch.equal(losses[r], ul[r]), f'replica {r} (width {H}): losses {losses[r].tolist()} vs {ul[r].tolist()}'
      if SNS[r]: assert torch.equal(sweep.u[r, :H + 1], uni.u[r]) and torch.equal(sweep.v[r, :d + H], uni.v[r]), f'replica {r}: u / v'
      _assert_padding_zero(sweep, opt, r)
  finally:
    _lib.set_option('gail_tiled', 1)


@pytest.mark.parametrize('training', [1, 0])
@pytest.mark.parametrize('gp', [0.0, 1.0])
def test_tiled_update_per_width_equals_uniform(training, gp):  # d = 23: gail_update_tiled_kernel<1>, <2>, <4> in one call
  _update_matches_uniform(17, 6, WIDTHS, 1, training, gp)


# gail_tiled off (gail_update_kernel<4>, <16>); ant-sized inputs (d = 35: <16>, <32>); a width outside {32, 64, 128} (48: <16>) beside the tiled 64
@pytest.mark.parametrize('S,A,widths,tiled', [(17, 6, WIDTHS, 0), (27, 8, WIDTHS, 1), (17, 6, [48, 64, 64, 48, 48, 64, 48], 1)])
@pytest.mark.parametrize('training', [1, 0])
@pytest.mark.parametrize('gp', [0.0, 1.0])
def test_untiled_update_per_width_equals_uniform(S, A, widths, tiled, training, gp):
  _update_matches_uniform(S, A, widths, tiled, training, gp)


@pytest.mark.parametrize('tiled', [1, 0])
def test_reward_per_width_equals_uniform(tiled):
  from il_b200 import _lib
  R, B, S, A = 7, 48, 17, 6
  batch = _batch(R, B, S, A, 3)
  _lib.set_option('gail_tiled', tiled)
  try:
    sweep = _sweep_disc(R, S, A, WIDTHS)
    sweep.u.normal_()  # stored vectors as after training, so that sigma != 1
    sweep.v.normal_()
    sweep.eval()
    out = sweep._run(batch, want_logits=True)
    for r in range(R):
      uni = _uniform_like(sweep, S, A, r)
      uni.eval()
      ref = uni._run(batch, want_logits=True)
      torch.cuda.synchronize()
      for k in ('reward', 'logits'): assert torch.equal(out[k][r], ref[k][r]), f'replica {r} (width {WIDTHS[r]}, {REWARDS[r]}, sn={SNS[r]}): {k}'
  finally:
    _lib.set_option('gail_tiled', 1)


def test_width_table_is_validated():
  from il_b200 import _lib
  import ctypes as C
  R, B, S, A = 7, 32, 17, 6
  batch = _batch(R, B, S, A, 3)
  sweep = _sweep_disc(R, S, A, WIDTHS)
  sweep.eval()
  out = torch.empty(R, B, device='cuda')
  bad = []
  g = sweep.c_struct(); g.width_class_H[2] = 256; bad.append((g, 'outside'))  # wider than the widest replica
  g = sweep.c_struct(); g.width_class_begin[2] = g.width_class_begin[1]; bad.append((g, 'increase'))
  g = sweep.c_struct(); g.width_class_begin[2] = R; bad.append((g, 'increase'))
  g = sweep.c_struct(); g.n_width_classes = _lib.MAX_WIDTH_CLASSES + 1; bad.append((g, 'at most'))
  for g, msg in bad:
    rc = _lib.lib().il_gail_reward(_lib.handle(), C.byref(g), R, C.byref(batch.c_struct()), out.data_ptr(), out.stride(0), out.stride(1), None, _lib.stream())
    assert rc != 0 and msg in _lib.last_error(), _lib.last_error()


# ---- initialisation ---------------------------------------------------------------------------------------------------------------
def test_replica_init_equals_a_single_run_of_its_width():
  from il_b200 import GAILDiscriminator
  from il_b200.net import ReplicaRNG
  R, S, A, seed = 7, 17, 6, 11
  sweep = GAILDiscriminator(S, A, _icfg(), 0.97, replicas=R, rng=ReplicaRNG(seed, R), spectral_norm=SNS, hidden_size=WIDTHS, device='cuda')
  opt_like = type('O', (), dict(exp_avg=torch.zeros_like(sweep.mlp.flat), exp_avg_sq=torch.zeros_like(sweep.mlp.flat)))
  for r in range(R):
    H, d = WIDTHS[r], S + A
    one = GAILDiscriminator(S, A, _icfg(), 0.97, replicas=1, rng=ReplicaRNG(seed + r, 1), spectral_norm=SNS[r], hidden_size=H, device='cuda')
    assert torch.equal(sweep.mlp.flat[r, :_stride(d, H)], one.mlp.flat[0]), f'replica {r} (width {H})'
    if SNS[r]: assert torch.equal(sweep.u[r, :H + 1], one.u[0]) and torch.equal(sweep.v[r, :d + H], one.v[0])
    _assert_padding_zero(sweep, opt_like, r)
    sd, ref = sweep.state_dict(spectral_norm=SNS[r], hidden_size=H), one.state_dict()
    assert set(sd) == set(ref) and all(torch.equal(sd[k][r], ref[k]) for k in ref), f'replica {r}: state_dict'
  with pytest.raises(ValueError, match='hidden_size'):
    sweep.state_dict()
  # load_state_dict with a width writes the replicas of that width only
  one = GAILDiscriminator(S, A, _icfg(), 0.97, replicas=1, rng=ReplicaRNG(99, 1), spectral_norm=True, hidden_size=32, device='cuda')
  before = sweep.mlp.flat.clone()
  sweep.load_state_dict(one.state_dict(), spectral_norm=True, hidden_size=32)
  for r in range(R):
    if WIDTHS[r] == 32: assert torch.equal(sweep.mlp.flat[r, :_stride(S + A, 32)], one.mlp.flat[0])
    else: assert torch.equal(sweep.mlp.flat[r], before[r])


def _trainer(base, R, fast_init=False, per_replica=None, values=None):
  from il_b200.config import load_config
  from il_b200.train import Trainer
  cfg = load_config(base + [f'replicas={R}'] + [f'{k}={v!r}' for k, v in (values or {}).items()])
  return Trainer(cfg, replicas=R, fast_init=fast_init, per_replica=per_replica)


SMALL = ['algorithm=GAIL', 'env=hopper', 'steps=40', 'training.start=20', 'training.batch_size=32', 'imitation.trajectories=2', 'reinforcement.actor.hidden_size=64',
         'reinforcement.critic.hidden_size=64', 'cuda_graphs=true', 'device_rng=true', 'seed=5', 'evaluation.episodes=1']


def test_fast_init_width_classes_start_like_fast_init_runs_of_their_width():
  widths = [128, 32, 64, 32, 128, 64]
  sweep = _trainer(SMALL, 6, fast_init=True, per_replica={W: widths})
  state_after = torch.get_rng_state()
  d, disc = sweep.S + sweep.A, sweep.discriminator
  assert disc.hidden_size_r == widths
  for H in (32, 64, 128):
    uni = _trainer(SMALL, 6, fast_init=True, values={W: H})
    if H == widths[0]: assert torch.equal(torch.get_rng_state(), state_after)  # the global stream goes on as after replica 0's width
    for r in (r for r in range(6) if widths[r] == H):
      assert torch.equal(disc.mlp.flat[r, :_stride(d, H)], uni.discriminator.mlp.flat[0]), f'replica {r} (width {H})'
      assert torch.equal(disc.u[r, :H + 1], uni.discriminator.u[0]) and torch.equal(disc.v[r, :d + H], uni.discriminator.v[0])
      assert not disc.mlp.flat[r, _stride(d, H):].any()
    assert torch.equal(sweep.actor.mlp.flat, uni.actor.mlp.flat)
    del uni


# ---- loops: a group's job blocks equal the uniform runs of their jobs ---------------------------------------------------------------
def _buffers(tr, H=None):
  """Per-replica buffers; with a width, the discriminator's blocks at that width's single-run layout."""
  d_in = tr.S + tr.A
  disc, opt = tr.discriminator, tr.discriminator_optimiser
  n = _stride(d_in, H) if H is not None else disc.mlp.flat.size(1)
  out = dict(actor=tr.actor.mlp.flat, critic=tr.critic.mlp.flat, target=tr.target_critic.mlp.flat, log_alpha=tr.log_alpha, rewards=tr.batch.rows, gail_losses=tr.gail_losses,
             disc=disc.mlp.flat[:, :n], disc_m=opt.exp_avg.reshape(tr.R, -1)[:, :n], disc_v=opt.exp_avg_sq.reshape(tr.R, -1)[:, :n], **tr.sac_out)
  if disc.u is not None:
    Hu = disc.mlp.dims[1] if H is None else H
    out['sn_u'], out['sn_v'] = disc.u[:, :Hu + 1], disc.v[:, :d_in + Hu]
  return {k: v.detach().reshape(tr.R, -1).clone() for k, v in out.items()}


def test_width_by_loss_grid_blocks_equal_uniform_runs():
  jobs = [(H, l) for H in (32, 64, 128) for l in ('BCE', 'Mixup', 'PUGAIL')]
  per_job = {W: [j[0] for j in jobs], 'imitation.loss_function': [j[1] for j in jobs]}
  J = len(jobs)
  sweep = _trainer(SMALL, J, per_replica=per_job)
  gp_on, mix_on = sweep._grad_penalty_on, sweep._mixup_on
  assert mix_on and sweep.use_graphs
  for _ in range(40): sweep.train_step()
  torch.cuda.synchronize()
  assert 'step+update' in sweep.graphs and sweep.updates > 2
  got = {H: _buffers(sweep, H) for H in (32, 64, 128)}
  full = _buffers(sweep)
  for j, (H, l) in enumerate(jobs):  # padding of the job's block stays zero
    n = _stride(sweep.S + sweep.A, H)
    assert not full['disc'][j, n:].any() and not full['disc_m'][j, n:].any() and not full['disc_v'][j, n:].any(), f'job {j}'
  del sweep
  for j, (H, l) in enumerate(jobs):
    uni = _trainer(SMALL, J, values={W: H, 'imitation.loss_function': l})
    uni._grad_penalty_on, uni._mixup_on = gp_on, mix_on
    for _ in range(40): uni.train_step()
    torch.cuda.synchronize()
    ref = _buffers(uni)
    for k, v in ref.items():
      assert torch.equal(got[H][k][j], v[j]), f'job {j} (width {H}, {l}): {k} differs (max |diff| {float((got[H][k][j] - v[j]).abs().max())})'
    del uni


# ---- semantics: each replica of a width group against the oracle loop built with its width --------------------------------------------
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


def test_width_group_replicas_match_the_oracle_with_their_width():
  from il_b200.config import load_config
  from il_b200.train import Trainer
  from oracle import loop as oloop
  R, B, H, steps, start = 3, 32, 64, 60, 30
  vals = {W: [32, 64, 128], 'imitation.loss_function': ['BCE', 'Mixup', 'PUGAIL']}
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=2',
                     f'reinforcement.actor.hidden_size={H}', f'reinforcement.critic.hidden_size={H}', 'cuda_graphs=false', 'gemm_mode=fp32', f'replicas={R}', 'seed=3'])
  tr = Trainer(cfg, replicas=R, per_replica=vals)
  tr.inject = True
  rs = np.random.RandomState(123)
  S, A, obs = tr.S, tr.A, tr.env.obs
  expert_raw = tr.env.synthesize_raw_dataset(5)
  disc, loops = tr.discriminator, []
  for r in range(R):
    d, Hd = S + A, vals[W][r]
    init = dict(actor=tr.actor.mlp.export_params(r, 0), twin=[tr.critic.mlp.export_params(r, 0), tr.critic.mlp.export_params(r, 1)],
                g=[v[r].cpu().clone() for v in disc._width_views(Hd)],
                sn=[(disc.u[r, :Hd].cpu().clone(), disc.v[r, :d].cpu().clone()), (disc.u[r, Hd:Hd + 1].cpu().clone(), disc.v[r, d:d + Hd].cpu().clone())])
    im = dict(hidden_size=Hd, loss_function=vals['imitation.loss_function'][r])
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
                 eps_mix=rs.uniform(size=(R, B)).astype(np.float32), eps_next=rs.standard_normal((R, B, A)).astype(np.float32),
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
  print('width group vs oracle', err, per)
  assert err['state'] < 2e-3, per
  assert err['q'] < 5e-3, per
  assert err['reward'] < 5e-3, per
  assert err['actor'] < 5e-4, per


# ---- the multirun command line -------------------------------------------------------------------------------------------------------
def _fcnn(sizes, sn):
  from torch import nn
  layers = []
  for i in range(len(sizes) - 1):
    lin = nn.Linear(sizes[i], sizes[i + 1])
    layers.append(nn.utils.parametrizations.spectral_norm(lin) if sn else lin)
    if i < len(sizes) - 2: layers.append(nn.ReLU())
  return nn.Sequential(*layers)


def test_multirun_over_widths_is_one_group(tmp_path):
  import subprocess
  import sys
  import yaml
  S, A = 12, 3
  cli = ['algorithm=GAIL', 'env=hopper', 'steps=60', 'training.start=30', 'evaluation.interval=60', 'evaluation.episodes=1', 'imitation.trajectories=2', 'memory.size=100',
         'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'training.batch_size=32', 'seed=9']
  swept = [f'{W}=32,64,128', 'imitation.spectral_norm=true,false', 'imitation.loss_function=BCE,Mixup']
  res = subprocess.run([sys.executable, 'train.py', '-m', *cli, *swept, f'output_dir={tmp_path}'], cwd=ROOT, capture_output=True, text=True, timeout=900)
  assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
  assert 'in 1 group(s)' in res.stdout
  (out, ) = glob.glob(os.path.join(str(tmp_path), '*_sweeper', '*'))
  assert sorted(os.listdir(out), key=int) == [str(j) for j in range(12)]
  jobs = [(H, sn, l) for H in (32, 64, 128) for sn in (True, False) for l in ('BCE', 'Mixup')]
  for j, (H, sn, l) in enumerate(jobs):
    ov = yaml.safe_load(open(os.path.join(out, str(j), 'overrides.yaml')))
    assert ov[-4:-1] == [f'{W}={H}', f'imitation.spectral_norm={str(sn).lower()}', f'imitation.loss_function={l}']
    m = torch.nn.Module()
    m.g = _fcnn([S + A, H, 1], sn)
    m.load_state_dict(torch.load(os.path.join(out, str(j), 'discriminator.pth')), strict=True)  # a single run's keys and shapes for this job's width and flag
  from il_b200.config import load_config
  from il_b200.train import Trainer
  j = 3  # width 32, no spectral norm, Mixup: one uniform 12-replica run, the job's block compared
  H, sn, l = jobs[j]
  cfg = load_config(cli + [f'{W}={H}', f'imitation.spectral_norm={str(sn).lower()}', f'imitation.loss_function={l}', 'replicas=12', f'output_dir={tmp_path}/u'])
  tr = Trainer(cfg, replicas=12)
  tr._grad_penalty_on, tr._mixup_on = True, True
  for _ in range(cfg.steps): tr.train_step()
  torch.cuda.synchronize()
  ref = tr.discriminator.state_dict()
  sd = torch.load(os.path.join(out, str(j), 'discriminator.pth'))
  assert set(sd) == set(ref)
  for k, v in sd.items(): assert torch.equal(v.cpu(), ref[k][j].cpu()), f'job {j}: {k}'
