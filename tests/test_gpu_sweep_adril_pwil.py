"""Sweeps over AdRIL's update frequency and balanced sampling, PWIL's reward scales and DRIL's quantile cutoff as replicas of one program: the
relabel and PWIL reward kernels with per-replica values against uniform calls (bitwise, slice by slice, eager and graph-replayed), the DRIL
threshold against the uniform threshold of each cutoff, sweep Trainers against the uniform runs of their jobs, 3-replica groups against the
oracle loop, and the multirun command line."""
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- 1. the relabel kernel ----------------------------------------------------------------------------------------------------------
UF = [0, 10, 1250, 7, 0, 25]  # 0: SQIL labels; 1250: a frequency above every step of the test
BAL = [True, True, False, False, False, True]
NEXP = 3


def _relabel_inputs(R, B, S, A, calls):
  """Per call: policy rows, expert rows, step [R] and trajectory counters [R] (0 and 1 included: max(nt, 1))."""
  from il_b200._lib import py_row_layout
  off, row = py_row_layout(S, A)
  g = torch.Generator(device='cuda').manual_seed(11)
  out = []
  for i in range(calls):
    pol, exp = torch.randn(R, B, row, device='cuda', generator=g), torch.randn(R, B, row, device='cuda', generator=g)
    pol[..., off['step']] = torch.randint(1, 60, (R, B), device='cuda', generator=g).float()
    step = torch.tensor([30.0 + 9 * i + 3 * r for r in range(R)], device='cuda')
    nt = torch.tensor([(i + r) % 4 for r in range(R)], dtype=torch.int32, device='cuda')
    out.append((pol, exp, step, nt))
  return out


def test_relabel_per_replica_equals_uniform_calls_eager_and_graph():
  from il_b200 import RewardRelabeller, TransitionBatch
  R, B, S, A, calls = len(UF), 24, 11, 3, 5
  inputs = _relabel_inputs(R, B, S, A, calls)
  tb = lambda rows: TransitionBatch(rows, S, A, False)
  sweep = RewardRelabeller(UF, BAL)
  assert sweep.update_freq == 1250 and sweep.balanced is True
  got, flags = [], []
  for pol, exp, step, nt in inputs:
    b = tb(pol.clone())
    sweep.resample_and_relabel(b, tb(exp), step, nt, NEXP, step_offset=-1.0)
    got.append(b.rows)
    flags.append(int(sweep._flag))
  assert flags == [0, 1, 0, 1, 0]
  for r in range(R):
    uni = RewardRelabeller(UF[r], BAL[r])
    for i, (pol, exp, step, nt) in enumerate(inputs):
      b = tb(pol[r:r + 1].clone())
      uni.resample_and_relabel(b, tb(exp[r:r + 1].clone()), step[r:r + 1], nt[r:r + 1], NEXP, step_offset=-1.0)
      assert torch.equal(got[i][r], b.rows[0]), f'call {i}, replica {r} (update_freq {UF[r]}, balanced {BAL[r]}): rows differ'
      if BAL[r]: assert int(uni._flag) == flags[i], f'call {i}: flag sequence'
    if not BAL[r]: assert int(uni._flag) == 1  # an unbalanced run never toggles the flag
  # the same calls replayed from one captured graph
  pol_s, exp_s, step_s, nt_s = (torch.empty_like(x) for x in inputs[0])
  rel = RewardRelabeller(UF, BAL)
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    rel.resample_and_relabel(tb(pol_s), tb(exp_s), step_s, nt_s, NEXP, step_offset=-1.0)
  rel._flag.fill_(1)
  for i, (pol, exp, step, nt) in enumerate(inputs):
    for dst, src in zip((pol_s, exp_s, step_s, nt_s), (pol, exp, step, nt)): dst.copy_(src)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(pol_s, got[i]), f'graph replay {i}: rows differ'
    assert int(rel._flag) == flags[i], f'graph replay {i}: flag'


def test_relabel_rewards_follow_each_replicas_rule():
  """The labels themselves: SQIL replicas 1 / 0, AdRIL replicas 1 / N_expert and -1[round > row round] / max(nt, 1), per replica."""
  from il_b200 import RewardRelabeller, TransitionBatch
  from il_b200._lib import py_row_layout
  R, B, S, A = len(UF), 24, 11, 3
  off, _ = py_row_layout(S, A)
  (pol, exp, step, nt), = _relabel_inputs(R, B, S, A, 1)
  b = TransitionBatch(pol.clone(), S, A, False)
  RewardRelabeller(UF, BAL).resample_and_relabel(b, TransitionBatch(exp, S, A, False), step, nt, NEXP, step_offset=-1.0)
  rew, rows = b.rows[..., off['rewards']].cpu().numpy(), pol.cpu().numpy()
  for r in range(R):
    expert = np.ones(B, bool) if BAL[r] else np.arange(B) < B // 2  # the flag starts at 1: balanced replicas take the expert batch
    for i in range(B):
      if expert[i]: want = np.float32(1.0) / np.float32(NEXP) if UF[r] else 1.0
      elif UF[r] == 0: want = 0.0
      else:
        rnd = np.ceil(np.float32(float(step[r]) - 1.0) / np.float32(UF[r]))
        want = -np.float32(rnd > np.ceil(rows[r, i, off['step']] / np.float32(UF[r]))) / np.float32(max(int(nt[r]), 1))
      assert rew[r, i] == np.float32(want), (r, i, rew[r, i], want)


# ---- 2. the PWIL reward kernel -------------------------------------------------------------------------------------------------------
SCALES, BWS = [1.0, 5.0, 10.0, 5.0, 1.0], [10.0, 1.0, 5.0, 5.0, 1.0]


def _pwil(R, scales, bws, N=160, S=11, A=3, T=40):
  from il_b200 import PWILDiscriminator
  from il_b200.config import Config
  g = torch.Generator().manual_seed(3)
  mem = dict(states=torch.randn(N, S, generator=g), actions=torch.randn(N, A, generator=g))
  cfg = Config(state_only=False, reward_scale=5, reward_bandwidth_scale=5)
  return PWILDiscriminator(S, A, cfg, mem, T, replicas=R, device='cuda', reward_scale=scales, reward_bandwidth_scale=bws)


def test_pwil_reward_per_replica_equals_uniform_calls():
  R, S, A, steps = len(SCALES), 11, 3, 12
  g = torch.Generator(device='cuda').manual_seed(5)
  inputs = [(torch.randn(R, S, device='cuda', generator=g), torch.randn(R, A, device='cuda', generator=g),
             (torch.rand(R, device='cuda', generator=g) > 0.25).int(), (torch.rand(R, device='cuda', generator=g) > 0.7).int()) for _ in range(steps)]

  def run(d):
    outs, weights = [], []
    for s, a, active, done in inputs:
      out = torch.full((R, ), -7.0, device='cuda')  # inactive replicas leave it alone
      d.compute_reward_batch(s, a, out=out, active=active)
      outs.append(out)
      weights.append(d.expert_weights.clone())
      d.reset(mask=done)
    torch.cuda.synchronize()
    return outs, weights

  sweep = _pwil(R, SCALES, BWS)
  assert sweep.reward_scale_r is not None and sweep.reward_bandwidth_r is not None
  got_r, got_w = run(sweep)
  for r in range(R):
    uni = _pwil(R, SCALES[r], BWS[r])
    assert uni.reward_scale_r is None and uni.reward_bandwidth_r is None
    ref_r, ref_w = run(uni)
    for i in range(steps):
      assert torch.equal(got_r[i][r], ref_r[i][r]), f'step {i}, replica {r} (scale {SCALES[r]}, bandwidth scale {BWS[r]}): reward'
      assert torch.equal(got_w[i][r], ref_w[i][r]), f'step {i}, replica {r}: atom weights'
  assert any(float(o[r]) == -7.0 for o in got_r for r in range(R))  # the mask held some replica back


# ---- 3. the DRIL threshold -----------------------------------------------------------------------------------------------------------
def test_dril_threshold_per_replica_equals_uniform_thresholds():
  from il_b200 import SoftActor
  from il_b200.config import load_config
  R, S, A, N = 5, 11, 3, 301
  cutoffs = [0.8, 0.98, 0.9, 0.8, 0.5]
  torch.manual_seed(0)
  actor = SoftActor(S, A, load_config(['algorithm=DRIL']).imitation.discriminator, replicas=R, device='cuda')
  es, ea = torch.randn(N, S, device='cuda'), torch.randn(N, A, device='cuda')
  masks = actor.draw_masks(N * SoftActor.ENSEMBLE)
  actor.set_uncertainty_threshold(es, ea, cutoffs, masks=masks)
  got = actor._q.clone()
  assert len(set(got.tolist())) > 1
  for c in sorted(set(cutoffs)):
    actor.set_uncertainty_threshold(es, ea, c, masks=masks)
    for r in range(R):
      if cutoffs[r] == c: assert torch.equal(got[r], actor._q[r]), f'replica {r}: cutoff {c}'
  actor.set_uncertainty_threshold(es, ea, [0.9] * R, masks=masks)  # equal values: the scalar call
  ref = actor._q.clone()
  actor.set_uncertainty_threshold(es, ea, 0.9, masks=masks)
  assert torch.equal(ref, actor._q)


# ---- 4. loops: a group's job blocks equal the uniform runs of their jobs ---------------------------------------------------------
def _buffers(tr):
  """Every per-replica buffer the loop updates, each as [replicas, -1]."""
  out = dict(actor=tr.actor.mlp.flat, critic=tr.critic.mlp.flat, target=tr.target_critic.mlp.flat, log_alpha=tr.log_alpha, actor_m=tr.actor_optimiser.exp_avg,
             actor_v=tr.actor_optimiser.exp_avg_sq, critic_m=tr.critic_optimiser.exp_avg, critic_v=tr.critic_optimiser.exp_avg_sq, alpha_m=tr.temperature_optimiser.exp_avg,
             alpha_v=tr.temperature_optimiser.exp_avg_sq, rows=tr.batch.rows, rewards=tr.batch.rows[..., tr.batch.off['rewards']], store_reward=tr.store_reward,
             return_sum=tr.return_sum, last_return=tr.last_return, episodes=tr.episodes, state=tr.state, **tr.sac_out)
  d = tr.discriminator
  if getattr(tr, 'discriminator_optimiser', None) is not None:
    out.update(disc=d.parameters()[0], disc_m=tr.discriminator_optimiser.exp_avg, disc_v=tr.discriminator_optimiser.exp_avg_sq)
  if getattr(d, '_q', None) is not None: out['dril_q'] = d._q
  if getattr(d, 'expert_weights', None) is not None: out['pwil_weights'] = d.expert_weights
  return {k: v.detach().reshape(tr.R, -1).clone() for k, v in out.items()}


def _make(base, R, per_replica=None, values=None):
  from il_b200.config import load_config
  from il_b200.train import Trainer
  cfg = load_config(base + [f'replicas={R}'] + [f'{k}={str(v).lower() if isinstance(v, bool) else v}' for k, v in (values or {}).items()])
  return Trainer(cfg, replicas=R, per_replica=per_replica)


def _drive(tr, steps, pre):
  if pre: tr.pretrain_discriminator()
  for _ in range(steps): tr.train_step()
  torch.cuda.synchronize()


def _sweep_matches_uniform_runs(base, per_job, R=2, steps=40, pre=False):
  """A group of J jobs x R replicas against, for each job, the uniform program of the same J x R replicas at that job's values: one device
  noise stream and one seed for both, so job j's block must be bitwise the same."""
  J = len(next(iter(per_job.values())))
  Rt = J * R
  sweep = _make(base, Rt, per_replica={k: [v for v in vals for _ in range(R)] for k, vals in per_job.items()})
  _drive(sweep, steps, pre)
  assert 'step+update' in sweep.graphs
  got = _buffers(sweep)
  del sweep
  for j in range(J):
    uni = _make(base, Rt, values={k: vals[j] for k, vals in per_job.items()})
    assert not uni.per_replica
    _drive(uni, steps, pre)
    ref = _buffers(uni)
    blk = slice(j * R, (j + 1) * R)
    for k, v in ref.items():
      assert torch.equal(got[k][blk], v[blk]), f'job {j} ({ {k_: vals[j] for k_, vals in per_job.items()} }): {k} differs'
    del uni


SMALL = ['env=hopper', 'steps=40', 'training.start=20', 'training.batch_size=32', 'imitation.trajectories=2', 'reinforcement.actor.hidden_size=64',
         'reinforcement.critic.hidden_size=64', 'cuda_graphs=true', 'device_rng=true', 'seed=5', 'evaluation.episodes=1']


def test_adril_grid_blocks_equal_uniform_runs():
  """SQIL, balanced and unbalanced AdRIL, with a frequency small enough that the rounds turn over during the run and one above every step."""
  _sweep_matches_uniform_runs(['algorithm=AdRIL'] + SMALL, {'imitation.update_freq': [0, 8, 1250, 8, 0, 25], 'imitation.balanced': [True, True, False, False, False, True]})


def test_pwil_scale_grid_blocks_equal_uniform_runs():
  _sweep_matches_uniform_runs(['algorithm=PWIL'] + SMALL, {'imitation.reward_scale': [1, 5, 10, 5], 'imitation.reward_bandwidth_scale': [1, 10, 5, 5]})


def test_dril_cutoff_blocks_equal_uniform_runs():
  _sweep_matches_uniform_runs(['algorithm=DRIL', 'imitation.pretraining.iterations=5'] + SMALL, {'imitation.quantile_cutoff': [0.8, 0.98, 0.9]}, pre=True)


# ---- 5. semantics: each replica of a group against the oracle loop built with its own values --------------------------------------
class _Injected:
  def __init__(self, seq): self.seq = seq
  def _pop(self, k): return self.seq[k].pop(0)
  def reset_u(self): return self._pop('reset_u')
  def act_eps(self, A): return self._pop('act_eps')
  def policy_indices(self, mem, n): return self._pop('idx_pol')
  def expert_indices(self, mem, n): return self._pop('idx_exp')
  def gp_eps(self, B): return self._pop('eps_gp')
  def sac_eps(self, B, A): return self._pop('eps_next'), self._pop('eps_new')


def _oracle_case(algorithm, vals, steps, start=30, B=32, H=64):
  """The loop of tests/test_gpu_loop.py with R = 3 replicas of one group, replica r's oracle loop built with replica r's values."""
  from il_b200.config import load_config
  from il_b200.train import Trainer
  from oracle import loop as oloop
  R = len(next(iter(vals.values())))
  cfg = load_config([f'algorithm={algorithm}', 'env=hopper', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=2',
                     f'reinforcement.actor.hidden_size={H}', f'reinforcement.critic.hidden_size={H}', 'cuda_graphs=false', 'gemm_mode=fp32', f'replicas={R}', 'seed=3'])
  tr = Trainer(cfg, replicas=R, per_replica=vals)
  assert set(tr.per_replica) == set(vals)
  tr.inject = True
  rs = np.random.RandomState(123)
  S, A, obs = tr.S, tr.A, tr.env.obs
  expert_raw = tr.env.synthesize_raw_dataset(5)
  loops = []
  for r in range(R):
    init = dict(actor=tr.actor.mlp.export_params(r, 0), twin=[tr.critic.mlp.export_params(r, 0), tr.critic.mlp.export_params(r, 1)])
    im = {k.split('.')[-1]: v[r] for k, v in vals.items()}
    loops.append(oloop.OracleLoop(algorithm, 'hopper', seed=3 + r, batch_size=B, start=start, memory_size=tr.cfg.memory.size, hidden_size=H, trajectories=2, expert_raw=expert_raw,
                                  init=init, mix_expert_data=cfg.imitation.mix_expert_data, imitation=im))
  Ne = tr.expert_memory.size
  u0 = rs.uniform(size=(R, obs)).astype(np.float32)
  tr.env.batch.reset(torch.from_numpy(u0).cuda(), tr.state)
  for r, lp in enumerate(loops): lp.state, lp.t = lp.env.reset(torch.from_numpy(u0[r])), 0
  err, per = {}, {}

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
      lp.noise = _Injected(seq)
      lp.run_step()
      e('state', r, float((tr.state[r].cpu() - lp.state[0]).abs().max()))
      assert int(tr.memory._idx[r]) == lp.memory.idx, f'step {step} replica {r}: ring index'
      if upd:
        e('q', r, float((tr.sac_out['q_values'][r].cpu() - lp.last['sac']['q_values']).abs().max()))
        e('reward', r, float((tr.batch['rewards'][r].cpu() - lp.last['rewards']).abs().max()))
  for r, lp in enumerate(loops):
    for i, p in enumerate(lp.agent.actor):
      e('actor', r, float((tr.actor.mlp.layer_views()[0][i][r].cpu() - p.detach()).abs().max()))
  print(algorithm, 'group vs oracle', err, per)
  return err, per


def test_adril_group_replicas_match_the_oracle_with_their_values():
  """SQIL, balanced AdRIL and unbalanced AdRIL in one program: the shared alternation flag toggles on every update, the unbalanced replica
  never reads it."""
  err, per = _oracle_case('AdRIL', {'imitation.update_freq': [0, 20, 15], 'imitation.balanced': [True, True, False]}, steps=70)
  assert err['state'] < 2e-3, per
  assert err['q'] < 5e-3, per
  assert err['reward'] < 1e-6, per  # the labels are exact on both sides
  assert err['actor'] < 5e-4, per


def test_pwil_group_replicas_match_the_oracle_with_their_values():
  err, per = _oracle_case('PWIL', {'imitation.reward_scale': [1.0, 5.0, 10.0], 'imitation.reward_bandwidth_scale': [5.0, 1.0, 10.0]}, steps=60)
  assert err['state'] < 2e-3, per
  assert err['q'] < 5e-3, per
  assert err['reward'] < 5e-3, per
  assert err['actor'] < 5e-4, per


# ---- 6. the multirun command line -------------------------------------------------------------------------------------------------
CLI = ['env=hopper', 'steps=60', 'training.start=30', 'evaluation.interval=60', 'evaluation.episodes=1', 'logging.interval=30', 'imitation.trajectories=2', 'memory.size=100',
       'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'training.batch_size=32', 'seed=9']


def _schema(x):
  """Keys, list lengths, array shapes and leaf types of a metrics dict."""
  if isinstance(x, dict): return {k: _schema(v) for k, v in x.items()}
  if isinstance(x, (list, tuple)): return [_schema(v) for v in x]
  if isinstance(x, np.ndarray): return ('array', x.shape, str(x.dtype))
  if torch.is_tensor(x): return ('tensor', tuple(x.shape), str(x.dtype))
  return type(x).__name__


def test_multirun_over_the_adril_grid_is_one_group(tmp_path):
  import yaml
  swept = ['imitation.balanced=true,false', 'imitation.update_freq=0,1250']
  res = subprocess.run([sys.executable, 'train.py', '-m', 'algorithm=AdRIL', *CLI, *swept, f'output_dir={tmp_path}/sweep'], cwd=ROOT, capture_output=True, text=True, timeout=900)
  assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
  assert 'sweep: 4 job(s) in 1 group(s)' in res.stdout
  assert "per-replica ['imitation.balanced', 'imitation.update_freq']" in res.stdout
  (out, ) = glob.glob(os.path.join(str(tmp_path), 'sweep', 'AdRIL_hopper_sweeper', '*'))
  assert sorted(os.listdir(out)) == ['0', '1', '2', '3']
  single = subprocess.run([sys.executable, 'train.py', 'algorithm=AdRIL', *CLI, f'output_dir={tmp_path}/single'], cwd=ROOT, capture_output=True, text=True, timeout=900)
  assert single.returncode == 0, single.stdout[-2000:] + single.stderr[-4000:]
  (one, ) = glob.glob(os.path.join(str(tmp_path), 'single', 'AdRIL_hopper', '*'))
  ref = _schema(torch.load(os.path.join(one, 'metrics.pth'), weights_only=False))
  for j, (bal, uf) in enumerate([(b, u) for b in ('true', 'false') for u in ('0', '1250')]):
    d = os.path.join(out, str(j))
    assert sorted(os.listdir(d)) == ['agent.pth', 'metrics.pth', 'overrides.yaml']
    assert yaml.safe_load(open(os.path.join(d, 'overrides.yaml'))) == ['algorithm=AdRIL', *CLI, f'imitation.balanced={bal}', f'imitation.update_freq={uf}',
                                                                              f'output_dir={tmp_path}/sweep']
    m = torch.load(os.path.join(d, 'metrics.pth'), weights_only=False)
    assert _schema(m) == ref, f'job {j}: metrics.pth schema'
    assert m['test_steps'] == [60] and m['predicted_rewards'][0].shape == (32, )
    assert f'job {j}: step 60: test return' in res.stdout
