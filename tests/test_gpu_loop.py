"""k-step loop parity (SURVEY §4 "integration"): the replica-batched Trainer (rollout + replay + discriminator
update + relabel + SAC update, train.py:149-203) against independent oracle loops, every noise draw and replay
index injected identically on both sides, identical initial weights. fp32 rounding differences amplify through the
loop (SURVEY §7 "chaotic divergence"), so the tolerance is looser than for single calls."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


class _Injected:
  """Noise source for the oracle loop that replays pre-drawn arrays (one per call, in order)."""

  def __init__(self, seq): self.seq = seq
  def _pop(self, k): return self.seq[k].pop(0)
  def reset_u(self): return self._pop('reset_u')
  def act_eps(self, A): return self._pop('act_eps')
  def policy_indices(self, mem, n): return self._pop('idx_pol')
  def expert_indices(self, mem, n): return self._pop('idx_exp')
  def gp_eps(self, B): return self._pop('eps_gp')
  def sac_eps(self, B, A): return self._pop('eps_next'), self._pop('eps_new')


def _run(algorithm, env_name, steps, start, B, H, extra=(), graphs=False, gemm_mode='fp32', imitation=None):
  import il_b200
  from il_b200.config import load_config
  from il_b200.train import Trainer
  from oracle import loop as oloop, port
  R = 2
  cfg = load_config([f'algorithm={algorithm}', f'env={env_name}', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=2',
                     f'reinforcement.actor.hidden_size={H}', f'reinforcement.critic.hidden_size={H}', f'cuda_graphs={str(graphs).lower()}', f'gemm_mode={gemm_mode}', f'replicas={R}', 'seed=3', *extra])
  tr = Trainer(cfg, replicas=R)
  tr.inject = True
  rs = np.random.RandomState(123)
  S, A, obs = tr.S, tr.A, tr.env.obs
  expert_raw = tr.env.synthesize_raw_dataset(5) if algorithm != 'SAC' else None
  loops = []
  for r in range(R):
    init = dict(actor=tr.actor.mlp.export_params(r, 0), twin=[tr.critic.mlp.export_params(r, 0), tr.critic.mlp.export_params(r, 1)])
    if algorithm == 'GAIL' and not tr.discriminator.general:
      d, Hd = S + A, tr.discriminator.mlp.dims[1]
      init['g'] = tr.discriminator.mlp.export_params(r, 0)
      init['sn'] = [(tr.discriminator.u[r, :Hd].cpu().clone(), tr.discriminator.v[r, :d].cpu().clone()), (tr.discriminator.u[r, Hd:Hd + 1].cpu().clone(), tr.discriminator.v[r, d:d + Hd].cpu().clone())]
    lp = oloop.OracleLoop(algorithm, env_name, seed=3 + r, batch_size=B, start=start, memory_size=cfg.memory.size, hidden_size=H, trajectories=2, expert_raw=expert_raw, init=init,
                          mix_expert_data=cfg.imitation.mix_expert_data, imitation=imitation)
    if algorithm == 'GAIL' and tr.discriminator.general:  # general discriminator (g / h nets): start the oracle from the product's initial weights and spectral-norm vectors
      dd = tr.discriminator
      for name, mlp, u, v in (('g', dd.g_mlp, dd.g_u, dd.g_v), ('h', dd.h_mlp, dd.h_u, dd.h_v)):
        if mlp is None: continue
        for P_, src in zip(getattr(lp.disc, name), mlp.export_params(r, 0)): P_.data.copy_(src)
        if dd.spectral_norm:
          sn, uo, vo = getattr(lp.disc, name + '_sn'), 0, 0
          for l in range(mlp.n_layers):
            od, idim = mlp.dims[l + 1], mlp.dims[l]
            sn[l] = (u[r, uo:uo + od].cpu().clone(), v[r, vo:vo + idim].cpu().clone())
            uo, vo = uo + od, vo + idim
    loops.append(lp)
  if algorithm != 'SAC':  # same expert buffer on both sides
    np.testing.assert_allclose(tr.expert_memory.states.cpu().numpy(), loops[0].expert_memory.data['states'].numpy(), rtol=1e-4, atol=1e-5)
    Ne = tr.expert_memory.size
  # identical initial env state
  u0 = rs.uniform(size=(R, obs)).astype(np.float32)
  tr.env.batch.reset(torch.from_numpy(u0).cuda(), tr.state)
  for r, lp in enumerate(loops): lp.state, lp.t = lp.env.reset(torch.from_numpy(u0[r])), 0
  max_err = {}
  for step in range(1, steps + 1):
    noise = dict(act_eps=rs.standard_normal((R, A)).astype(np.float32), reset_u=rs.uniform(size=(R, obs)).astype(np.float32), eps_gp=rs.uniform(size=(R, B)).astype(np.float32),
                 eps_next=rs.standard_normal((R, B, A)).astype(np.float32), eps_new=rs.standard_normal((R, B, A)).astype(np.float32))
    upd = step >= start
    if upd:
      # indices valid on both sides: below (idx before this step's append) - 1, a subset of the reference's range
      noise['idx_pol'] = np.stack([rs.randint(0, max(lp.memory.idx - 1, 1), size=B) for lp in loops]).astype(np.int32)
      if algorithm != 'SAC': noise['idx_exp'] = rs.randint(0, Ne - 1, size=(R, B)).astype(np.int32)
    tr.eps_act.copy_(torch.from_numpy(noise['act_eps']))
    tr.u_reset.copy_(torch.from_numpy(noise['reset_u']))
    if upd:
      tr.idx_pol.copy_(torch.from_numpy(noise['idx_pol']))
      if algorithm != 'SAC': tr.idx_exp.copy_(torch.from_numpy(noise['idx_exp']))
      tr.eps_gp.copy_(torch.from_numpy(noise['eps_gp']))
      tr.eps_next.copy_(torch.from_numpy(noise['eps_next']))
      tr.eps_new.copy_(torch.from_numpy(noise['eps_new']))
    tr.train_step()
    for r, lp in enumerate(loops):
      seq = {k: [torch.from_numpy(np.asarray(v[r]))] for k, v in noise.items()}
      seq['act_eps'] = [torch.from_numpy(noise['act_eps'][r:r + 1])]
      lp.noise = _Injected(seq)
      lp.run_step()
    # compare state trajectories and (after updates) losses / parameters
    for r, lp in enumerate(loops):
      err = float((tr.state[r].cpu() - lp.state[0]).abs().max())
      max_err['state'] = max(max_err.get('state', 0), err)
      assert int(tr.memory._idx[r]) == lp.memory.idx, f'step {step} replica {r}: ring index {int(tr.memory._idx[r])} vs {lp.memory.idx}'
      if upd:
        e = float((tr.sac_out['q_values'][r].cpu() - lp.last['sac']['q_values']).abs().max())
        max_err['q'] = max(max_err.get('q', 0), e)
        e = float((tr.batch['rewards'][r].cpu() - lp.last['rewards']).abs().max())
        max_err['reward'] = max(max_err.get('reward', 0), e)
  for r, lp in enumerate(loops):
    for i, p in enumerate(lp.agent.actor):
      e = float((tr.actor.mlp.layer_views()[0][i][r].cpu() - p.detach()).abs().max())
      max_err['actor'] = max(max_err.get('actor', 0), e)
  return max_err


@pytest.mark.parametrize('algorithm,env_name,extra', [('GAIL', 'hopper', ()), ('SAC', 'hopper', ()), ('GMMIL', 'halfcheetah', ()), ('PWIL', 'hopper', ()),
                                                      ('GAIL', 'walker2d', ('imitation.mix_expert_data=mixed_batch', )),
                                                      # train.py:133,136-143: expert rows pre-filled into every replica's ring (the ring of 60 rows wraps during the
                                                      # transfer), PWIL's greedy relabelling of the expert's own transitions
                                                      ('GMMIL', 'halfcheetah', ('imitation.mix_expert_data=prefill_memory', )),
                                                      ('PWIL', 'hopper', ('imitation.mix_expert_data=prefill_memory', )),
                                                      ('PWIL', 'hopper', ('imitation.mix_expert_data=mixed_batch', ))])
def test_loop_matches_oracle(algorithm, env_name, extra):
  err = _run(algorithm, env_name, steps=60, start=30, B=32, H=64, extra=extra)
  print(algorithm, env_name, err)
  assert err['state'] < 2e-3, err
  assert err.get('q', 0) < 5e-3, err
  assert err.get('reward', 0) < 5e-3, err
  assert err['actor'] < 5e-4, err


def test_loop_matches_oracle_at_the_benchmarked_configuration():
  """The configuration bench.py times (VERDICT r1 weak #1): 256-wide actor / critic, batch 256, dense layers on the 3xTF32 wgmma
  engine (incl. the first layer fused into its producers), the whole iteration replayed as a CUDA graph — 62 steps, 32 of them
  updates, 2 replicas, every noise draw and index injected on both sides."""
  err = _run('GAIL', 'hopper', steps=62, start=30, B=256, H=256, graphs=True, gemm_mode='tf32x3')
  print('bench config', err)
  assert err['state'] < 2e-3, err
  assert err.get('q', 0) < 5e-3, err
  assert err.get('reward', 0) < 5e-3, err
  assert err['actor'] < 5e-4, err


@pytest.mark.parametrize('extra,imitation', [
    (('imitation.discriminator.reward_shaping=true', 'imitation.discriminator.subtract_log_policy=true'), dict(reward_shaping=True, subtract_log_policy=True)),
    (('imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh', 'imitation.discriminator.hidden_size=32'), dict(depth=2, activation='tanh', hidden_size=32))])
def test_loop_with_general_discriminator_matches_oracle(extra, imitation):
  """SURVEY §8f row 3 inside the loop: reward shaping + subtract_log_policy (linear g, MLP h, log-policy from the live actor) and a depth-2
  tanh discriminator (second-order terms of the gradient penalty), csrc/gail_general.cu vs the oracle loop (pinned to the reference's train())."""
  err = _run('GAIL', 'hopper', steps=50, start=30, B=32, H=64, extra=extra, imitation=imitation)
  print('general discriminator', imitation, err)
  assert err['state'] < 2e-3, err
  assert err.get('q', 0) < 5e-3, err
  assert err.get('reward', 0) < 5e-3, err
  assert err['actor'] < 5e-4, err


@pytest.mark.parametrize('extra,imitation', [(('imitation.update_freq=20', ), dict(update_freq=20, balanced=True)),
                                             (('imitation.update_freq=15', 'imitation.balanced=false'), dict(update_freq=15, balanced=False)),
                                             (('imitation.update_freq=0', ), dict(update_freq=0, balanced=True))])
def test_loop_adril_sqil_matches_oracle(extra, imitation):
  """SURVEY §8f row 4: RewardRelabeller (models.py:293-318) inside the loop — balanced alternation with the flag on the device, AdRIL round
  arithmetic on the stored `step` column and the per-replica trajectory counters, SQIL labels."""
  err = _run('AdRIL', 'hopper', steps=70, start=30, B=32, H=64, extra=extra, imitation=imitation)
  print('AdRIL', imitation, err)
  assert err['state'] < 2e-3, err
  assert err.get('q', 0) < 5e-3, err
  assert err.get('reward', 0) < 1e-6, err
  assert err['actor'] < 5e-4, err


def _mask(rs, shape, p): return ((rs.uniform(size=shape) >= p) / (1.0 - p)).astype(np.float32)


@pytest.mark.parametrize('algorithm', ['DRIL', 'RED'])
def test_dropout_discriminator_loops_match_oracle(algorithm):
  """SURVEY §8f row 4 inside the loop (train.py:117-133 pre-training, :190-191 / :196-197 relabelling): DRIL's dropout policy ensemble and RED's predictor are
  pre-trained on injected expert minibatches with injected dropout masks, the threshold / bandwidth is fixed, then 40 loop steps (10 updates) with the reward of
  every sampled batch coming from the pre-trained network — all on csrc/dropout_nets.cu, against the oracle loop (pinned to the reference's train())."""
  from il_b200.config import load_config
  from il_b200.train import Trainer
  from oracle import cases, loop as oloop
  R, B, H, steps, start, iters = 2, 32, 64, 40, 30, 6
  p_in, p_h = (0.1, 0.1) if algorithm == 'DRIL' else (0.2, 0.3)
  dH = 32
  extra = [f'imitation.discriminator.hidden_size={dH}', f'imitation.discriminator.input_dropout={p_in}', f'imitation.discriminator.dropout={p_h}', f'imitation.pretraining.iterations={iters}',
           'imitation.learning_rate=0.001']
  cfg = load_config([f'algorithm={algorithm}', 'env=hopper', f'steps={steps}', f'training.start={start}', f'training.batch_size={B}', 'imitation.trajectories=2',
                     f'reinforcement.actor.hidden_size={H}', f'reinforcement.critic.hidden_size={H}', 'cuda_graphs=false', 'gemm_mode=fp32', f'replicas={R}', 'seed=3', *extra])
  tr = Trainer(cfg, replicas=R)
  tr.inject = True
  rs = np.random.RandomState(321)
  S, A, obs = tr.S, tr.A, tr.env.obs
  din = S if algorithm == 'DRIL' else S + A
  expert_raw = tr.env.synthesize_raw_dataset(5)
  im = dict(hidden_size=dH, input_dropout=p_in, dropout=p_h, pretraining_iterations=iters, learning_rate=1e-3, weight_decay=cfg.imitation.weight_decay,
            depth=cfg.imitation.discriminator.depth, activation=cfg.imitation.discriminator.activation)
  if algorithm == 'DRIL': im['quantile_cutoff'] = cfg.imitation.quantile_cutoff
  loops = []
  for r in range(R):
    init = dict(actor=tr.actor.mlp.export_params(r, 0), twin=[tr.critic.mlp.export_params(r, 0), tr.critic.mlp.export_params(r, 1)])
    lp = oloop.OracleLoop(algorithm, 'hopper', seed=3 + r, batch_size=B, start=start, memory_size=cfg.memory.size, hidden_size=H, trajectories=2, expert_raw=expert_raw, init=init,
                          mix_expert_data=cfg.imitation.mix_expert_data, imitation=im, bc_aux_loss=bool(cfg.imitation.bc_aux_loss))  # DRIL.yaml: bc_aux_loss true
    d = tr.discriminator
    if algorithm == 'DRIL':
      for P_, src in zip(lp.disc, d.mlp.export_params(r, 0)): P_.data.copy_(src)
    else:
      for P_, src in zip(lp.disc.predictor, d.predictor.export_params(r, 0)): P_.data.copy_(src)
      for P_, src in zip(lp.disc.target, d.target.export_params(r, 0)): P_.data.copy_(src)
    loops.append(lp)
  Ne = tr.expert_memory.size
  depth = im['depth']
  def draw(n): return [_mask(rs, (R, n, din), p_in)] + [_mask(rs, (R, n, dH), p_h) for _ in range(depth)]
  # ---- pre-training: same minibatches, same masks -------------------------------------------------------------------------------
  batches = rs.randint(0, Ne, size=(iters, R, B)).astype(np.int32)
  masks = [draw(B) for _ in range(iters)]
  thr = draw(Ne * 5) if algorithm == 'DRIL' else draw(B)
  tr.pretrain_discriminator(iters, batches=[torch.from_numpy(batches[i]) for i in range(iters)], masks=[[torch.from_numpy(m).cuda() for m in ms] for ms in masks],
                            threshold_masks=[torch.from_numpy(m).cuda() for m in thr])
  for r, lp in enumerate(loops):
    seq = [torch.from_numpy(m[r]) for ms in masks for m in ms] + [torch.from_numpy(m[r]) for m in thr]
    with cases.injected_dropout(seq):
      lp.pretrain_discriminator(batches=[batches[i, r].tolist() for i in range(iters)])
    assert not seq, 'the oracle consumed a different number of dropout draws'
    if algorithm == 'DRIL': np.testing.assert_allclose(float(tr.discriminator._q[r]), lp.dril_q, rtol=2e-3, atol=1e-9)
    else: np.testing.assert_allclose(float(tr.discriminator.sigma[r]), lp.disc.sigma_1, rtol=1e-4)
  u0 = rs.uniform(size=(R, obs)).astype(np.float32)
  tr.env.batch.reset(torch.from_numpy(u0).cuda(), tr.state)
  for r, lp in enumerate(loops): lp.state, lp.t = lp.env.reset(torch.from_numpy(u0[r])), 0
  err = {}
  for step in range(1, steps + 1):
    noise = dict(act_eps=rs.standard_normal((R, A)).astype(np.float32), reset_u=rs.uniform(size=(R, obs)).astype(np.float32),
                 eps_next=rs.standard_normal((R, B, A)).astype(np.float32), eps_new=rs.standard_normal((R, B, A)).astype(np.float32))
    upd = step >= start
    rew_masks = None
    if upd:
      noise['idx_pol'] = np.stack([rs.randint(0, max(lp.memory.idx - 1, 1), size=B) for lp in loops]).astype(np.int32)
      noise['idx_exp'] = rs.randint(0, Ne - 1, size=(R, B)).astype(np.int32)
      if algorithm == 'DRIL': rew_masks = draw(B * 5)
    tr.eps_act.copy_(torch.from_numpy(noise['act_eps']))
    tr.u_reset.copy_(torch.from_numpy(noise['reset_u']))
    if upd:
      tr.idx_pol.copy_(torch.from_numpy(noise['idx_pol']))
      tr.idx_exp.copy_(torch.from_numpy(noise['idx_exp']))
      tr.eps_next.copy_(torch.from_numpy(noise['eps_next']))
      tr.eps_new.copy_(torch.from_numpy(noise['eps_new']))
      tr.dril_masks = None if rew_masks is None else [torch.from_numpy(m).cuda() for m in rew_masks]
    tr.train_step()
    for r, lp in enumerate(loops):
      seq = {k: [torch.from_numpy(np.asarray(v[r]))] for k, v in noise.items()}
      seq['act_eps'] = [torch.from_numpy(noise['act_eps'][r:r + 1])]
      lp.noise = _Injected(seq)
      with cases.injected_dropout([] if rew_masks is None else [torch.from_numpy(m[r]) for m in rew_masks]):
        lp.run_step()
      err['state'] = max(err.get('state', 0), float((tr.state[r].cpu() - lp.state[0]).abs().max()))
      if upd:
        err['q'] = max(err.get('q', 0), float((tr.sac_out['q_values'][r].cpu() - lp.last['sac']['q_values']).abs().max()))
        err['reward'] = max(err.get('reward', 0), float((tr.batch['rewards'][r].cpu() - lp.last['rewards']).abs().max()))
  for r, lp in enumerate(loops):
    for i, p in enumerate(lp.agent.actor):
      err['actor'] = max(err.get('actor', 0), float((tr.actor.mlp.layer_views()[0][i][r].cpu() - p.detach()).abs().max()))
  print(algorithm, err)
  assert err['state'] < 2e-3, err
  assert err.get('q', 0) < 5e-3, err
  assert err.get('reward', 0) < 5e-3, err
  assert err['actor'] < 5e-4, err
