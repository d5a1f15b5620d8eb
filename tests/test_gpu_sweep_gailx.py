"""Sweeps over the general GAIL discriminator's choices as replicas of one program (csrc/gail_general.cu): il_gailx_update with per-replica loss
function, prior, margin, spectral norm, reward function and penalty pass against uniform calls at each replica's values (bitwise, replica by
replica), il_gailx_reward likewise, sweep Trainers against the uniform runs of their jobs, a 3-replica group against the oracle loop, the multirun
command line, and the refusal of a spectral-norm flag array without u / v buffers."""
import ctypes as C
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
# margin 0 at prior 0.3: with a freshly initialised discriminator the policy and expert terms are about equal, so prior * E - P < 0 and the clamp is active
MARGINS = [float('inf'), 0.0, 0.0, 1.0, float('inf'), 0.5, 0.3]
REWARDS = ['AIRL', 'GAIL', 'FAIRL', 'GAIL', 'AIRL', 'FAIRL', 'AIRL']
# penalty pass with spectral norm (0, 3, 6) and without (5); outside it with spectral norm (2) and without (1, 4)
GPS = [0.5, 0.0, 0.0, 0.5, 0.0, 0.5, 1.0]

# (S, A, overrides, gradient penalty on): depth-2 relu, depth-1 tanh, shaping with the log-policy term, state-only sigmoid (no penalty: undefined there)
CONFIGS = {'depth2-relu': (17, 6, ['imitation.discriminator.depth=2'], True),
           'depth1-tanh': (17, 6, ['imitation.discriminator.activation=tanh'], True),
           'shaping-logp': (17, 6, ['imitation.discriminator.reward_shaping=true', 'imitation.discriminator.subtract_log_policy=true', 'imitation.discriminator.activation=tanh'], True),
           'state_only-sigmoid': (17, 6, ['imitation.discriminator.depth=2', 'imitation.discriminator.activation=sigmoid', 'imitation.state_only=true'], False)}


# ---- 1. the C ABI: one call with per-replica values against uniform calls -----------------------------------------------------------
def _icfg(over, **kw):
  from il_b200.config import Config, load_config
  c = load_config(['algorithm=GAIL', 'imitation.discriminator.hidden_size=32', *over]).imitation
  return Config(dict(c, **kw))


def _batch(R, B, S, A, seed):
  from il_b200 import TransitionBatch
  from il_b200._lib import py_row_layout
  off, row = py_row_layout(S, A)
  g = torch.Generator(device='cuda').manual_seed(seed)
  rows = torch.randn(R, B, row, device='cuda', generator=g)
  rows[..., off['weights']] = torch.rand(R, B, device='cuda', generator=g) + 0.5
  rows[..., off['terminals']] = (torch.rand(R, B, device='cuda', generator=g) < 0.2).float()
  return TransitionBatch(rows.contiguous(), S, A, False)


def _uv(d):
  return [(n, getattr(d, n)) for n in ('g_u', 'g_v', 'h_u', 'h_v') if getattr(d, n, None) is not None]


def _disc_pair(over, R, S, A, r, seed=0):
  """The per-replica discriminator and the uniform one with replica r's choices for every replica, holding the same parameters / u / v."""
  from il_b200 import GAILDiscriminator
  torch.manual_seed(seed)
  sweep = GAILDiscriminator(S, A, _icfg(over), 0.97, replicas=R, spectral_norm=SNS[:R], reward_function=REWARDS[:R], device='cuda')
  uni = GAILDiscriminator(S, A, _icfg(over), 0.97, replicas=R, spectral_norm=SNS[r], reward_function=REWARDS[r], device='cuda')
  assert sweep.general and uni.general
  uni.flat.copy_(sweep.flat)
  if SNS[r]:
    for (n, a), (m, b) in zip(_uv(sweep), _uv(uni)): b.copy_(a)
  return sweep, uni


def _actor(S, A, R):
  from il_b200 import SoftActor
  from il_b200.config import load_config
  torch.manual_seed(11)
  return SoftActor(S, A, load_config(['algorithm=GAIL', 'reinforcement.actor.hidden_size=32']).reinforcement.actor, replicas=R, device='cuda')


@pytest.mark.parametrize('config', list(CONFIGS))
@pytest.mark.parametrize('training', [1, 0])
def test_update_per_replica_equals_uniform_calls(config, training, R=7, B=40, steps=2):
  import il_b200
  S, A, over, gp_on = CONFIGS[config]
  pol, exp = _batch(R, B, S, A, 1), _batch(R, B, S, A, 2)
  eps_gp, eps_mix = torch.rand(R, B, device='cuda'), torch.rand(R, B, device='cuda')
  f = lambda x: torch.tensor(x, dtype=torch.float32, device='cuda')
  actor = _actor(S, A, R)
  gps = GPS[:R] if gp_on else [0.0] * R
  sweep, _ = _disc_pair(over, R, S, A, 0)
  sweep.train(training)
  opt = il_b200.AdamW(sweep.parameters(), lr=3e-3, weight_decay=0.1)
  cfg = _icfg(over, loss_function=LOSSES[:R], pos_class_prior=f(PRIORS[:R]), nonnegative_margin=f(MARGINS[:R]), grad_penalty=f(gps) if gp_on else 0.0, entropy_bonus=0.05)
  penalty_pass = torch.tensor([int(x > 0) for x in gps], dtype=torch.int32, device='cuda') if gp_on else None
  losses = torch.zeros(R, 2, device='cuda')
  for _ in range(steps):
    il_b200.adversarial_imitation_update(actor, sweep, pol, exp, opt, cfg, eps_gp=eps_gp, eps_mix=eps_mix, out_losses=losses, penalty_pass=penalty_pass)
  for r in range(R):
    _, uni = _disc_pair(over, R, S, A, r)
    uni.train(training)
    uopt = il_b200.AdamW(uni.parameters(), lr=3e-3, weight_decay=0.1)
    ucfg = _icfg(over, loss_function=LOSSES[r], pos_class_prior=PRIORS[r], nonnegative_margin=MARGINS[r], grad_penalty=gps[r], entropy_bonus=0.05)
    ul = torch.zeros(R, 2, device='cuda')
    for _ in range(steps): il_b200.adversarial_imitation_update(actor, uni, pol, exp, uopt, ucfg, eps_gp=eps_gp, eps_mix=eps_mix, out_losses=ul)
    torch.cuda.synchronize()
    what = f'replica {r} ({LOSSES[r]}, sn={SNS[r]}, gp={gps[r]})'
    for name, a, b in (('params', sweep.flat, uni.flat), ('m', opt.exp_avg, uopt.exp_avg), ('v', opt.exp_avg_sq, uopt.exp_avg_sq), ('losses', losses, ul)):
      a, b = a.reshape(R, -1)[r], b.reshape(R, -1)[r]
      assert torch.equal(a, b), f'{what}: {name} differs by {float((a - b).abs().max())}'
    for (n, a), ub in zip(_uv(sweep), [b for _, b in _uv(uni)] if SNS[r] else [None] * 4):
      if SNS[r]: assert torch.equal(a[r], ub[r]), f'{what}: {n}'
      else: assert not a[r].any(), f'{what} touched its {n}'


def test_penalty_pass_null_keeps_every_replica_in_the_pass():
  """Without penalty_pass a replica at grad_penalty 0 takes the pass's power iterations (the public semantics of per-replica grad_penalty): its u / v
  then differ from a call that masks it out of the pass, while its zero penalty leaves the parameters as they are."""
  import il_b200
  S, A, over, _ = CONFIGS['depth2-relu']
  R, B = 3, 32
  pol, exp = _batch(R, B, S, A, 1), _batch(R, B, S, A, 2)
  eps_gp = torch.rand(R, B, device='cuda')
  runs = {}
  for key, pp in (('null', None), ('masked', torch.tensor([1, 0, 1], dtype=torch.int32, device='cuda'))):
    torch.manual_seed(0)
    d = il_b200.GAILDiscriminator(S, A, _icfg(over), 0.97, replicas=R, spectral_norm=True, device='cuda')
    d.train()
    opt = il_b200.AdamW(d.parameters(), lr=3e-3, weight_decay=0.1)
    cfg = _icfg(over, grad_penalty=torch.tensor([1.0, 0.0, 0.5], device='cuda'))
    il_b200.adversarial_imitation_update(None, d, pol, exp, opt, cfg, eps_gp=eps_gp, penalty_pass=pp)
    torch.cuda.synchronize()
    runs[key] = (d.flat.clone(), d.g_u.clone(), d.g_v.clone())
  assert torch.equal(runs['null'][0], runs['masked'][0])  # the loss passes come first: the parameters see the same gradient
  for r in (0, 2):
    for i in (1, 2): assert torch.equal(runs['null'][i][r], runs['masked'][i][r])
  for i in (1, 2): assert not torch.equal(runs['null'][i][1], runs['masked'][i][1])  # replica 1: one more power iteration without the mask


@pytest.mark.parametrize('config', ['depth2-relu', 'shaping-logp'])
def test_reward_per_replica_equals_uniform_calls(config):
  R, B = 7, 48
  S, A, over, _ = CONFIGS[config]
  batch = _batch(R, B, S, A, 3)
  actor = _actor(S, A, R)
  sweep, _ = _disc_pair(over, R, S, A, 0)
  for _, t in _uv(sweep): t.normal_()  # stored vectors as after training, so that sigma != 1
  sweep.eval()
  out = sweep.predict_reward_batch(batch, write_rewards=False, actor=actor)
  logits = sweep._run(batch, want_logits=True, log_policy=actor._run(batch.rows[..., :S], given=batch.rows[..., S:S + A], want=('log_prob', ))['log_prob'])['logits']
  for r in range(R):
    _, uni = _disc_pair(over, R, S, A, r)
    if SNS[r]:
      for (_, a), (_, b) in zip(_uv(sweep), _uv(uni)): b.copy_(a)
    uni.eval()
    ref = uni.predict_reward_batch(batch, write_rewards=False, actor=actor)
    ref_logits = uni._run(batch, want_logits=True, log_policy=actor._run(batch.rows[..., :S], given=batch.rows[..., S:S + A], want=('log_prob', ))['log_prob'])['logits']
    torch.cuda.synchronize()
    assert torch.equal(out[r], ref[r]), f'replica {r} ({REWARDS[r]}, sn={SNS[r]}): reward'
    assert torch.equal(logits[r], ref_logits[r]), f'replica {r}: logits'


def test_spectral_norm_flags_without_uv_are_refused_before_any_launch():
  import il_b200
  from il_b200 import _lib
  S, A, over, _ = CONFIGS['shaping-logp']
  R, B = 3, 16
  pol, exp = _batch(R, B, S, A, 1), _batch(R, B, S, A, 2)
  torch.manual_seed(0)
  d = il_b200.GAILDiscriminator(S, A, _icfg(over, spectral_norm=False, loss_function='BCE', grad_penalty=0.0), 0.97, replicas=R, device='cuda')
  d.train()
  flags = torch.tensor([1, 0, 1], dtype=torch.int32, device='cuda')
  opt = il_b200.AdamW(d.parameters(), lr=3e-3, weight_decay=0.1)
  lp = torch.zeros(R, B, device='cuda')
  a = _lib.GailxUpdateArgs()
  a.disc, a.opt, a.params_floats, a.policy, a.expert = d.cx_struct(), opt.c_struct(), d.flat.numel(), pol.c_struct(), exp.c_struct()
  a.disc.spectral_norm_r = flags.data_ptr()
  a.logp_policy = a.logp_expert = lp.data_ptr()
  a.R, a.loss_function, a.training = R, _lib.LOSS['BCE'], 1
  ws = torch.zeros(1 << 24, dtype=torch.uint8, device='cuda')
  a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
  before = (d.flat.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), ws.clone())
  torch.cuda.synchronize()
  n0 = il_b200.launch_count()
  lib = _lib.lib()
  assert lib.il_gailx_update(_lib.handle(), C.byref(a), _lib.stream()) != 0
  assert b'spectral_norm_r' in lib.il_last_error()
  out = torch.empty(R, B, device='cuda')
  assert lib.il_gailx_reward(_lib.handle(), C.byref(a.disc), R, C.byref(a.policy), lp.data_ptr(), out.data_ptr(), B, 1, None, ws.data_ptr(), ws.numel(), _lib.stream()) != 0
  torch.cuda.synchronize()
  assert il_b200.launch_count() == n0
  for x, y in zip(before, (d.flat, opt.exp_avg, opt.exp_avg_sq, ws)): assert torch.equal(x, y)


# ---- 2. loops: a group's job blocks equal the uniform runs of their jobs ---------------------------------------------------------
def _buffers(tr):
  d = tr.discriminator
  out = dict(actor=tr.actor.mlp.flat, critic=tr.critic.mlp.flat, target=tr.target_critic.mlp.flat, log_alpha=tr.log_alpha, rewards=tr.batch.rows, gail_losses=tr.gail_losses,
             disc=d.parameters()[0], disc_m=tr.discriminator_optimiser.exp_avg, disc_v=tr.discriminator_optimiser.exp_avg_sq, **tr.sac_out)
  out.update({'sn_' + n: t for n, t in _uv(d)})
  return {k: v.detach().reshape(tr.R, -1).clone() for k, v in out.items()}


def _make(base, R, per_replica=None, values=None):
  from il_b200.config import load_config
  from il_b200.train import Trainer
  cfg = load_config(base + [f'replicas={R}'] + [f'{k}={v!r}' for k, v in (values or {}).items()])
  return Trainer(cfg, replicas=R, per_replica=per_replica)


def _drive(tr, steps):
  for _ in range(steps): tr.train_step()
  torch.cuda.synchronize()


def _sweep_matches_uniform_runs(base, per_job, steps=40):
  J = len(next(iter(per_job.values())))
  sweep = _make(base, J, per_replica=per_job)
  assert sweep.discriminator.general
  gp_on, mix_on = sweep._grad_penalty_on, sweep._mixup_on
  _drive(sweep, steps)
  assert 'step+update' in sweep.graphs
  got = _buffers(sweep)
  sn = sweep.discriminator.spectral_norm_r
  del sweep
  for j in range(J):
    uni = _make(base, J, values={k: vals[j] for k, vals in per_job.items()})
    # the group draws the Mixup and penalty noise for all its replicas from one device stream when any job needs it: the uniform run of a job
    # that does not need it draws it too, so both see the same noise afterwards
    uni._grad_penalty_on, uni._mixup_on = gp_on, mix_on
    _drive(uni, steps)
    ref = _buffers(uni)
    vals = {k: v[j] for k, v in per_job.items()}
    for k, v in ref.items():
      assert k in got, f'job {j} ({vals}): {k} missing from the sweep'
      assert torch.equal(got[k][j], v[j]), f'job {j} ({vals}): {k} differs (max |diff| {float((got[k][j] - v[j]).abs().max())})'
    if sn is not None and not sn[j]:
      for k in got:
        if k.startswith('sn_'): assert not got[k][j].any(), f'job {j} touched its {k}'
    del uni


SMALL = ['algorithm=GAIL', 'env=hopper', 'steps=40', 'training.start=20', 'training.batch_size=32', 'imitation.trajectories=2', 'reinforcement.actor.hidden_size=64',
         'reinforcement.critic.hidden_size=64', 'imitation.discriminator.hidden_size=32', 'cuda_graphs=true', 'device_rng=true', 'seed=5', 'evaluation.episodes=1']
GENERAL = {'depth2-tanh': ['imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh'],
           'shaping-logp': ['imitation.discriminator.reward_shaping=true', 'imitation.discriminator.subtract_log_policy=true']}


def _grid():
  jobs = [(l, rf, sn) for l in ('BCE', 'Mixup', 'PUGAIL') for rf in ('GAIL', 'AIRL', 'FAIRL') for sn in (True, False)]
  return {'imitation.loss_function': [j[0] for j in jobs], 'imitation.discriminator.reward_function': [j[1] for j in jobs], 'imitation.spectral_norm': [j[2] for j in jobs]}


@pytest.mark.parametrize('general', list(GENERAL))
def test_choice_grid_blocks_equal_uniform_runs(general):
  _sweep_matches_uniform_runs(SMALL + GENERAL[general], _grid())


@pytest.mark.parametrize('general', list(GENERAL))
def test_penalty_by_spectral_norm_blocks_equal_uniform_runs(general):
  _sweep_matches_uniform_runs(SMALL + GENERAL[general] + ['imitation.loss_function=PUGAIL', 'imitation.nonnegative_margin=0.1'],
                              {'imitation.grad_penalty': [0.0, 0.5, 0.0, 0.5], 'imitation.spectral_norm': [True, True, False, False]})


# ---- 3. semantics: each replica of a group against the oracle loop built with its values --------------------------------------------
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
  R, B, H, Hd, steps, start = 3, 32, 64, 32, 50, 30
  vals = {'imitation.loss_function': ['BCE', 'Mixup', 'PUGAIL'], 'imitation.discriminator.reward_function': ['AIRL', 'GAIL', 'FAIRL'], 'imitation.spectral_norm': [True, False, True],
          'imitation.grad_penalty': [1.0, 0.0, 0.5], 'imitation.nonnegative_margin': [float('inf'), float('inf'), 0.3]}
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=2',
                     f'reinforcement.actor.hidden_size={H}', f'reinforcement.critic.hidden_size={H}', 'cuda_graphs=false', 'gemm_mode=fp32', f'replicas={R}', 'seed=3',
                     'imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh', f'imitation.discriminator.hidden_size={Hd}'])
  tr = Trainer(cfg, replicas=R, per_replica=vals)
  assert tr.discriminator.general
  tr.inject = True
  rs = np.random.RandomState(123)
  S, A, obs = tr.S, tr.A, tr.env.obs
  expert_raw = tr.env.synthesize_raw_dataset(5)
  loops, dd = [], tr.discriminator
  for r in range(R):
    sn = vals['imitation.spectral_norm'][r]
    init = dict(actor=tr.actor.mlp.export_params(r, 0), twin=[tr.critic.mlp.export_params(r, 0), tr.critic.mlp.export_params(r, 1)])
    im = dict(depth=2, activation='tanh', hidden_size=Hd, loss_function=vals['imitation.loss_function'][r], reward_function=vals['imitation.discriminator.reward_function'][r],
              spectral_norm=sn, grad_penalty=vals['imitation.grad_penalty'][r], nonnegative_margin=vals['imitation.nonnegative_margin'][r])
    lp = oloop.OracleLoop('GAIL', 'hopper', seed=3 + r, batch_size=B, start=start, memory_size=tr.cfg.memory.size, hidden_size=H, trajectories=2, expert_raw=expert_raw, init=init,
                          mix_expert_data=cfg.imitation.mix_expert_data, imitation=im)
    for P_, src in zip(lp.disc.g, dd.g_mlp.export_params(r, 0)): P_.data.copy_(src)
    if sn:
      uo, vo = 0, 0
      for l in range(dd.g_mlp.n_layers):
        od, idim = dd.g_mlp.dims[l + 1], dd.g_mlp.dims[l]
        lp.disc.g_sn[l] = (dd.g_u[r, uo:uo + od].cpu().clone(), dd.g_v[r, vo:vo + idim].cpu().clone())
        uo, vo = uo + od, vo + idim
    loops.append(lp)
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
  print('general choice group vs oracle', err, per)
  assert err['state'] < 2e-3, per
  assert err['q'] < 5e-3, per
  assert err['reward'] < 5e-3, per
  assert err['actor'] < 5e-4, per


# ---- 4. the multirun command line -------------------------------------------------------------------------------------------------
def _fcnn(sizes, sn):
  from torch import nn
  layers = []
  for i in range(len(sizes) - 1):
    lin = nn.Linear(sizes[i], sizes[i + 1])
    layers.append(nn.utils.parametrizations.spectral_norm(lin) if sn else lin)
    if i < len(sizes) - 2: layers.append(nn.ReLU())
  return nn.Sequential(*layers)


def test_multirun_over_the_general_choice_grid_is_one_group(tmp_path):
  import subprocess
  import sys
  import yaml
  S, A, H = 12, 3, 64
  cli = ['algorithm=GAIL', 'env=hopper', 'steps=60', 'training.start=30', 'evaluation.interval=60', 'evaluation.episodes=1', 'imitation.trajectories=2', 'memory.size=100',
         'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'training.batch_size=32', 'seed=9', 'imitation.discriminator.depth=2']
  swept = ['imitation.loss_function=BCE,Mixup,PUGAIL', 'imitation.discriminator.reward_function=GAIL,AIRL,FAIRL', 'imitation.spectral_norm=true,false']
  res = subprocess.run([sys.executable, 'train.py', '-m', *cli, *swept, f'output_dir={tmp_path}'], cwd=ROOT, capture_output=True, text=True, timeout=900)
  assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
  assert 'in 1 group(s)' in res.stdout
  (out, ) = glob.glob(os.path.join(str(tmp_path), '*_sweeper', '*'))
  assert sorted(os.listdir(out), key=int) == [str(j) for j in range(18)]
  grid = _grid()
  for j in range(18):
    d = os.path.join(out, str(j))
    ov = yaml.safe_load(open(os.path.join(d, 'overrides.yaml')))
    sn = grid['imitation.spectral_norm'][j]
    assert ov[-2] == f'imitation.spectral_norm={"true" if sn else "false"}'
    sd = torch.load(os.path.join(d, 'discriminator.pth'))
    m = torch.nn.Module()
    m.g = _fcnn([S + A, H, H, 1], sn)
    m.load_state_dict(sd, strict=True)  # a single run's keys and shapes for this job's spectral_norm
