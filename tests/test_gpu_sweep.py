"""Hyper-parameter sweeps as replicas of one program (Trainer(per_replica=...), `train.py -m`): the per-replica AdamW / polyak kernels against one
scalar call per replica slice, sweep Trainers against the uniform runs of their jobs (bitwise), a 2-replica sweep against the oracle loop built with
each replica's values, and the multirun command line."""
import ctypes as C
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- 1. AdamW kernels ---------------------------------------------------------------------------------------------------------
def _adam_sweep_vs_slices(rf, R, polyak, tma, lrs, wds, taus):
  import il_b200
  from il_b200 import _lib
  lib, h = _lib.lib(), _lib.handle()
  n = rf * R
  torch.manual_seed(1)
  p0, g = torch.randn(n, device='cuda'), torch.randn(n, device='cuda') * 0.1
  m0, v0 = torch.sin(p0), torch.cos(p0) ** 2
  tau_t = torch.tensor(taus, dtype=torch.float32, device='cuda')
  _lib.set_option('adam_tma', tma)
  try:
    p, tgt = p0.clone(), p0.clone() * 0.5
    opt = il_b200.AdamW([p], lr=lrs, weight_decay=wds)
    assert opt.replica_floats == rf
    opt.exp_avg.copy_(m0); opt.exp_avg_sq.copy_(v0)
    for _ in range(2):
      a = opt.c_struct()
      if polyak: _lib.check(lib.il_adam_step_polyak_r(h, p.data_ptr(), g.data_ptr(), C.byref(a), n, tgt.data_ptr(), tau_t.data_ptr(), _lib.stream()))
      else: _lib.check(lib.il_adam_step(h, p.data_ptr(), g.data_ptr(), C.byref(a), n, _lib.stream()))
    ref = []
    for r in range(R):
      sl = slice(r * rf, (r + 1) * rf)
      pr, tr = p0[sl].clone(), p0[sl].clone() * 0.5
      o = il_b200.AdamW([pr], lr=lrs[r], weight_decay=wds[r])
      o.exp_avg.copy_(m0[sl]); o.exp_avg_sq.copy_(v0[sl])
      for _ in range(2):
        a = o.c_struct()
        if polyak: _lib.check(lib.il_adam_step_polyak(h, pr.data_ptr(), g[sl].contiguous().data_ptr(), C.byref(a), rf, tr.data_ptr(), float(tau_t[r]), _lib.stream()))
        else: _lib.check(lib.il_adam_step(h, pr.data_ptr(), g[sl].contiguous().data_ptr(), C.byref(a), rf, _lib.stream()))
      ref.append((pr, o.exp_avg, o.exp_avg_sq, tr))
    torch.cuda.synchronize()
  finally:
    _lib.set_option('adam_tma', 1)
  for r, (pr, mr, vr, tr) in enumerate(ref):
    sl = slice(r * rf, (r + 1) * rf)
    assert torch.equal(p[sl], pr) and torch.equal(opt.exp_avg[sl], mr) and torch.equal(opt.exp_avg_sq[sl], vr), f'replica {r}'
    if polyak: assert torch.equal(tgt[sl], tr), f'target of replica {r}'


def _grid(R):
  lrs = [1e-4 * (1 + 0.37 * r) for r in range(R)]
  wds = [0.0 if r == 1 else 0.01 * (r + 1) for r in range(R)]  # one replica without weight decay
  taus = [0.99 - 0.003 * r for r in range(R)]
  return lrs, wds, taus


@pytest.mark.parametrize('polyak', [False, True])
def test_plain_adam_kernel_per_replica_equals_scalar_calls(polyak):
  R = 5
  _adam_sweep_vs_slices(1000, R, polyak, 0, *_grid(R))


@pytest.mark.parametrize('tma', range(8))
@pytest.mark.parametrize('polyak', [False, True])
def test_tma_adam_kernel_per_replica_equals_scalar_calls(polyak, tma):
  """16 replicas of 70012 floats (a multiple of 4, not of any tile: tiles straddle replica boundaries) — above the TMA switch-over size, so
  the per-replica call runs the TMA-staged kernel of every ring geometry; and 16 hopper actors (256-wide) as laid out by the Trainer."""
  from il_b200 import _lib
  R = 16
  _adam_sweep_vs_slices(70012, R, polyak, tma, *_grid(R))
  if tma == 1: _adam_sweep_vs_slices(_lib.py_mlp_offsets([12, 256, 256, 6])[2], R, polyak, tma, *_grid(R))


# ---- 2. loops: a sweep block equals the uniform run of its job -------------------------------------------------------------------
def _buffers(tr):
  """Every per-replica buffer the loop updates, each as [replicas, -1]."""
  Rt = tr.R
  out = dict(actor=tr.actor.mlp.flat, critic=tr.critic.mlp.flat, target=tr.target_critic.mlp.flat, log_alpha=tr.log_alpha,
             actor_m=tr.actor_optimiser.exp_avg, actor_v=tr.actor_optimiser.exp_avg_sq, critic_m=tr.critic_optimiser.exp_avg, critic_v=tr.critic_optimiser.exp_avg_sq,
             alpha_m=tr.temperature_optimiser.exp_avg, alpha_v=tr.temperature_optimiser.exp_avg_sq, rewards=tr.batch.rows, gail_losses=tr.gail_losses, **tr.sac_out)
  d = tr.discriminator
  if getattr(tr, 'discriminator_optimiser', None) is not None:
    out.update(disc=d.parameters()[0], disc_m=tr.discriminator_optimiser.exp_avg, disc_v=tr.discriminator_optimiser.exp_avg_sq)
  for n in ('u', 'v', 'g_u', 'g_v', 'h_u', 'h_v'):
    if getattr(d, n, None) is not None: out['disc_' + n] = getattr(d, n)
  return {k: v.detach().reshape(Rt, -1).clone() for k, v in out.items()}


def _make(base, R, per_replica=None, values=None):
  from il_b200.config import load_config
  from il_b200.train import Trainer
  cfg = load_config(base + [f'replicas={R}'] + [f'{k}={v!r}' for k, v in (values or {}).items()])
  return Trainer(cfg, replicas=R, per_replica=per_replica)


def _drive(tr, steps, pre):
  if pre == 'bc': tr.bc_pretrain(8)
  elif pre == 'disc': tr.pretrain_discriminator()
  for _ in range(steps): tr.train_step()
  torch.cuda.synchronize()


def _sweep_matches_uniform_runs(base, per_job, R, steps=40, pre=None):
  J = len(next(iter(per_job.values())))
  Rt = J * R
  sweep = _make(base, Rt, per_replica={k: [v for v in vals for _ in range(R)] for k, vals in per_job.items()})
  gp_on = sweep._grad_penalty_on
  _drive(sweep, steps, pre)
  got = _buffers(sweep)
  del sweep
  for j in range(J):
    uni = _make(base, Rt, values={k: vals[j] for k, vals in per_job.items()})
    # the group draws the gradient-penalty noise for all its replicas (one device noise stream): the uniform run of a job at
    # grad_penalty 0 consumes that draw too, so both see the same noise afterwards
    uni._grad_penalty_on = gp_on
    _drive(uni, steps, pre)
    ref = _buffers(uni)
    for k, v in ref.items():
      blk = slice(j * R, (j + 1) * R)
      assert torch.equal(got[k][blk], v[blk]), f'job {j}: {k} differs (max |diff| {float((got[k][blk] - v[blk]).abs().max())})'
    del uni


SMALL = ['env=hopper', 'steps=40', 'training.start=20', 'training.batch_size=32', 'imitation.trajectories=2', 'reinforcement.actor.hidden_size=64',
         'reinforcement.critic.hidden_size=64', 'cuda_graphs=true', 'device_rng=true', 'seed=5', 'evaluation.episodes=1']


def test_gail_sweep_blocks_equal_uniform_runs():
  """Tiled discriminator; grad_penalty (one job at 0: that replica skips the penalty pass) and entropy_bonus vary, with both learning rates."""
  _sweep_matches_uniform_runs(['algorithm=GAIL'] + SMALL, {'imitation.grad_penalty': [1.0, 0.0, 5.0, 1.0], 'imitation.entropy_bonus': [0.0, 0.1, 0.0, 0.02],
                                                        'training.learning_rate': [3e-4, 1e-4, 3e-4, 6e-4], 'imitation.learning_rate': [3e-5, 3e-5, 1e-4, 1e-5]}, R=1)


def test_gail_sweep_blocks_equal_uniform_runs_at_the_benchmarked_configuration():
  base = ['algorithm=GAIL', 'env=hopper', 'training.start=20', 'training.batch_size=256', 'imitation.trajectories=2', 'gemm_mode=tf32x3', 'cuda_graphs=true', 'seed=5']
  _sweep_matches_uniform_runs(base, {'training.learning_rate': [3e-4, 1e-4, 3e-4, 6e-4], 'reinforcement.discount': [0.97, 0.97, 0.99, 0.9],
                                     'imitation.grad_penalty': [1.0, 0.0, 1.0, 2.0]}, R=1)


def test_general_gail_shaping_discount_sweep_blocks_equal_uniform_runs():
  _sweep_matches_uniform_runs(['algorithm=GAIL', 'imitation.discriminator.reward_shaping=true'] + SMALL, {'reinforcement.discount': [0.97, 0.9, 0.99, 0.95]}, R=2)


def test_sac_sweep_blocks_equal_uniform_runs():
  _sweep_matches_uniform_runs(['algorithm=SAC'] + SMALL, {'training.learning_rate': [3e-4, 1e-3, 1e-4, 3e-4], 'training.weight_decay': [0.0, 0.0, 0.01, 0.1],
                                                       'reinforcement.polyak_factor': [0.995, 0.99, 0.995, 0.9], 'reinforcement.target_temperature': [-1.0, -0.5, -2.0, -1.0]}, R=2)


@pytest.mark.parametrize('algorithm', ['RED', 'DRIL'])
def test_pretrained_discriminator_sweep_blocks_equal_uniform_runs(algorithm):
  base = [f'algorithm={algorithm}', 'imitation.pretraining.iterations=5'] + SMALL
  _sweep_matches_uniform_runs(base, {'imitation.learning_rate': [1e-3, 3e-4, 1e-4, 1e-3], 'imitation.weight_decay': [0.0, 0.1, 1.0, 10.0]}, R=1, pre='disc')


def test_bc_pretraining_sweep_blocks_equal_uniform_runs():
  _sweep_matches_uniform_runs(['algorithm=SAC', 'bc_pretraining.iterations=8'] + SMALL, {'bc_pretraining.learning_rate': [1e-3, 3e-4, 1e-4, 3e-3],
                                                                                    'bc_pretraining.weight_decay': [0.0, 0.1, 1.0, 0.0]}, R=2, steps=0, pre='bc')


# ---- 3. semantics: each replica of a sweep against the oracle loop built with that replica's values ------------------------------
class _Injected:
  def __init__(self, seq): self.seq = seq
  def _pop(self, k): return self.seq[k].pop(0)
  def reset_u(self): return self._pop('reset_u')
  def act_eps(self, A): return self._pop('act_eps')
  def policy_indices(self, mem, n): return self._pop('idx_pol')
  def expert_indices(self, mem, n): return self._pop('idx_exp')
  def gp_eps(self, B): return self._pop('eps_gp')
  def sac_eps(self, B, A): return self._pop('eps_next'), self._pop('eps_new')


def test_gail_sweep_replicas_match_the_oracle_with_their_values():
  # values near the defaults: the loop amplifies fp32 rounding differences (test_gpu_loop), the more the larger the steps
  _oracle_case({'training.learning_rate': [3e-4, 2e-4], 'training.weight_decay': [0.0, 1e-3], 'reinforcement.discount': [0.97, 0.95],
                'reinforcement.polyak_factor': [0.99, 0.98], 'reinforcement.target_temperature': [-0.5, -1.0], 'imitation.learning_rate': [3e-5, 1e-5],
                'imitation.weight_decay': [10.0, 5.0], 'imitation.grad_penalty': [1.0, 0.0]})


def _oracle_case(vals):
  from il_b200.config import get_key, load_config
  from il_b200.train import Trainer
  from oracle import loop as oloop
  R, B, H, steps, start = 2, 32, 64, 60, 30
  cfg = load_config(['algorithm=GAIL', 'env=hopper', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=2',
                     f'reinforcement.actor.hidden_size={H}', f'reinforcement.critic.hidden_size={H}', 'cuda_graphs=false', 'gemm_mode=fp32', f'replicas={R}', 'seed=3'])
  tr = Trainer(cfg, replicas=R, per_replica=vals)
  keys = ('training.learning_rate', 'training.weight_decay', 'reinforcement.discount', 'reinforcement.polyak_factor', 'reinforcement.target_temperature',
          'imitation.learning_rate', 'imitation.weight_decay', 'imitation.grad_penalty')
  vals = {k: vals.get(k, [get_key(cfg, k)] * R) for k in keys}  # the oracle is built with every value explicitly
  tr.inject = True
  rs = np.random.RandomState(123)
  S, A, obs = tr.S, tr.A, tr.env.obs
  expert_raw = tr.env.synthesize_raw_dataset(5)
  loops = []
  for r in range(R):
    d, Hd = S + A, tr.discriminator.mlp.dims[1]
    init = dict(actor=tr.actor.mlp.export_params(r, 0), twin=[tr.critic.mlp.export_params(r, 0), tr.critic.mlp.export_params(r, 1)], g=tr.discriminator.mlp.export_params(r, 0),
                sn=[(tr.discriminator.u[r, :Hd].cpu().clone(), tr.discriminator.v[r, :d].cpu().clone()), (tr.discriminator.u[r, Hd:Hd + 1].cpu().clone(), tr.discriminator.v[r, d:d + Hd].cpu().clone())])
    v = {k: x[r] for k, x in vals.items()}
    loops.append(oloop.OracleLoop('GAIL', 'hopper', seed=3 + r, batch_size=B, start=start, memory_size=tr.cfg.memory.size, hidden_size=H, trajectories=2, expert_raw=expert_raw, init=init,
                                  mix_expert_data=cfg.imitation.mix_expert_data, lr=v['training.learning_rate'], weight_decay=v['training.weight_decay'],
                                  discount=v['reinforcement.discount'], polyak=v['reinforcement.polyak_factor'], target_temperature=v['reinforcement.target_temperature'],
                                  imitation=dict(learning_rate=v['imitation.learning_rate'], weight_decay=v['imitation.weight_decay'], grad_penalty=v['imitation.grad_penalty'])))
  Ne = tr.expert_memory.size
  u0 = rs.uniform(size=(R, obs)).astype(np.float32)
  tr.env.batch.reset(torch.from_numpy(u0).cuda(), tr.state)
  for r, lp in enumerate(loops): lp.state, lp.t = lp.env.reset(torch.from_numpy(u0[r])), 0
  err, per = {}, {}  # max error overall / per (quantity, replica)

  def e(k, r, x):
    err[k], per[(k, r)] = max(err.get(k, 0), x), max(per.get((k, r), 0), x)

  for step in range(1, steps + 1):
    noise = dict(act_eps=rs.standard_normal((R, A)).astype(np.float32), reset_u=rs.uniform(size=(R, obs)).astype(np.float32), eps_gp=rs.uniform(size=(R, B)).astype(np.float32),
                 eps_next=rs.standard_normal((R, B, A)).astype(np.float32), eps_new=rs.standard_normal((R, B, A)).astype(np.float32))
    upd = step >= start
    if upd:
      noise['idx_pol'] = np.stack([rs.randint(0, max(lp.memory.idx - 1, 1), size=B) for lp in loops]).astype(np.int32)
      noise['idx_exp'] = rs.randint(0, Ne - 1, size=(R, B)).astype(np.int32)
    tr.eps_act.copy_(torch.from_numpy(noise['act_eps']))
    tr.u_reset.copy_(torch.from_numpy(noise['reset_u']))
    if upd:
      for k, t in (('idx_pol', tr.idx_pol), ('idx_exp', tr.idx_exp), ('eps_gp', tr.eps_gp), ('eps_next', tr.eps_next), ('eps_new', tr.eps_new)): t.copy_(torch.from_numpy(noise[k]))
    tr.train_step()
    for r, lp in enumerate(loops):
      seq = {k: [torch.from_numpy(np.asarray(x[r]))] for k, x in noise.items()}
      seq['act_eps'] = [torch.from_numpy(noise['act_eps'][r:r + 1])]
      if vals['imitation.grad_penalty'][r] == 0: seq.pop('eps_gp')  # the oracle of a replica without a penalty draws no penalty noise
      lp.noise = _Injected(seq)
      lp.run_step()
      e('state', r, float((tr.state[r].cpu() - lp.state[0]).abs().max()))
      if upd:
        e('q', r, float((tr.sac_out['q_values'][r].cpu() - lp.last['sac']['q_values']).abs().max()))
        e('reward', r, float((tr.batch['rewards'][r].cpu() - lp.last['rewards']).abs().max()))
  for r, lp in enumerate(loops):
    for i, p in enumerate(lp.agent.actor):
      e('actor', r, float((tr.actor.mlp.layer_views()[0][i][r].cpu() - p.detach()).abs().max()))
  print('sweep vs oracle', err, per)
  assert err['state'] < 2e-3, per
  assert err['q'] < 5e-3, per
  assert err['reward'] < 5e-3, per
  assert err['actor'] < 5e-4, per


# ---- 4. the multirun command line ------------------------------------------------------------------------------------------------
def _fcnn(sizes):
  from torch import nn
  layers = []
  for i in range(len(sizes) - 2): layers += [nn.Linear(sizes[i], sizes[i + 1]), nn.ReLU()]
  return nn.Sequential(*layers, nn.Linear(sizes[-2], sizes[-1]))


def _multirun(tmp_path, *args):
  cmd = [sys.executable, 'train.py', '-m', *args, f'output_dir={tmp_path}']
  res = subprocess.run(cmd, cwd=ROOT, capture_output=True, text=True, timeout=900)
  assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
  runs = glob.glob(os.path.join(str(tmp_path), '*_sweeper', '*'))
  assert len(runs) == 1, runs
  return runs[0], res.stdout


SMALL_CLI = ['algorithm=GAIL', 'env=hopper', 'steps=60', 'training.start=30', 'evaluation.interval=60', 'evaluation.episodes=1', 'logging.interval=30', 'imitation.trajectories=2',
             'memory.size=100', 'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32']


def test_multirun_writes_one_directory_per_job(tmp_path):
  import yaml
  S, A, H = 12, 3, 32
  out, stdout = _multirun(tmp_path, *SMALL_CLI, 'training.batch_size=32', 'training.learning_rate=1e-4,3e-4', 'reinforcement.discount=0.97,0.99')
  assert os.path.basename(os.path.dirname(out)) == 'GAIL_hopper_sweeper'
  assert 'in 1 group(s)' in stdout
  assert sorted(os.listdir(out)) == ['0', '1', '2', '3']
  for j in range(4):
    d = os.path.join(out, str(j))
    assert sorted(os.listdir(d)) == ['agent.pth', 'discriminator.pth', 'metrics.pth', 'overrides.yaml']
    ov = yaml.safe_load(open(os.path.join(d, 'overrides.yaml')))
    assert ov[:len(SMALL_CLI)] == SMALL_CLI and ov[len(SMALL_CLI):-1] == ['training.batch_size=32', f'training.learning_rate={"1e-4" if j < 2 else "3e-4"}',
                                                                         f'reinforcement.discount={"0.97" if j % 2 == 0 else "0.99"}']
    assert f'job {j}: step 60: test return' in stdout
    agent = torch.load(os.path.join(d, 'agent.pth'))
    actor = torch.nn.Module()
    actor.actor = _fcnn([S, H, H, 2 * A])
    actor.load_state_dict(agent['actor'])  # strict: a single run's keys and shapes
    critic = torch.nn.Module()
    critic.critic_1, critic.critic_2 = torch.nn.Module(), torch.nn.Module()
    critic.critic_1.critic, critic.critic_2.critic = _fcnn([S + A, H, H, 1]), _fcnn([S + A, H, H, 1])
    critic.load_state_dict(agent['critic'])
    assert agent['log_alpha'].shape == (1, )
    m = torch.load(os.path.join(d, 'metrics.pth'), weights_only=False)
    assert m['test_steps'] == [60] and len(m['test_returns'][0]) == 1 and m['predicted_rewards'][0].shape == (32, ) and m['alphas'][0].shape == (1, )
    assert len(m['train_returns']) == 1
  assert stdout.count(': score ') == 4


def test_multirun_over_a_shape_key_runs_two_groups(tmp_path):
  out, stdout = _multirun(tmp_path, *SMALL_CLI, 'training.batch_size=32,64')
  assert 'in 2 group(s)' in stdout and sorted(os.listdir(out)) == ['0', '1']
