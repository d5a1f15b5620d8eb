"""GPU tests of the reference-facing surface: environment / evaluation parity with the CPU twin, initialisation
stream, state-dict keys, drop-in (R = 1) call shapes, CUDA-graph vs eager equivalence, device index sampling."""
import ctypes as C

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


class Cfg(dict):
  def __getattr__(self, k):
    v = self[k]
    return Cfg(v) if isinstance(v, dict) and not isinstance(v, Cfg) else v

  def get(self, k, d=None): return dict.get(self, k, d)


MODEL = Cfg(hidden_size=32, depth=2, activation='relu')


def test_env_step_matches_cpu_twin():
  import il_b200
  from il_b200.environments import D4RLEnv
  from oracle import port
  R = 3
  for name in ('hopper', 'halfcheetah', 'ant'):
    env = D4RLEnv(name, True, replicas=R)
    twins = [port.SyntheticEnv(name, True) for _ in range(R)]
    rs = np.random.RandomState(5)
    u = rs.uniform(size=(R, env.obs)).astype(np.float32)
    s = env.reset(torch.from_numpy(u))
    for r in range(R): np.testing.assert_allclose(s[r].cpu().numpy(), twins[r].reset(torch.from_numpy(u[r]))[0].numpy(), atol=1e-7)
    alive = [True] * R
    for t in range(40):
      a = np.tanh(rs.standard_normal((R, env.act)) * 2).astype(np.float32) * 1.3  # exercises the clamp (environments.py:36)
      ns, rew, done = env.step(torch.from_numpy(a))
      for r in range(R):
        if not alive[r]: continue
        tns, trew, tdone = twins[r].step(torch.from_numpy(a[r:r + 1]))
        np.testing.assert_allclose(ns[r].cpu().numpy(), tns[0].numpy(), rtol=1e-4, atol=2e-5)
        assert abs(float(rew[r]) - trew) < 1e-4
        assert bool(done[r]) == tdone
        if tdone: alive[r] = False


def test_evaluate_agent_matches_oracle():
  import il_b200
  from il_b200.environments import D4RLEnv
  from il_b200.evaluation import evaluate_agent
  from oracle import port
  R, E = 2, 3
  env = D4RLEnv('hopper', True, replicas=R, max_episode_steps=80)
  actor = il_b200.SoftActor(12, 3, MODEL, replicas=R)
  rs = np.random.RandomState(3)
  u = rs.uniform(size=(R * E, env.obs)).astype(np.float32)
  stats = {}
  got, traj = evaluate_agent(actor, env, E, return_trajectories=True, reset_noise=torch.from_numpy(u), out_stats=stats)
  total_steps = 0
  for r in range(R):
    twin = port.SyntheticEnv('hopper', True, max_episode_steps=80)
    ref = port.evaluate_agent(actor.mlp.export_params(r, 0), twin, E, [torch.from_numpy(u[r * E + e]) for e in range(E)])
    np.testing.assert_allclose(got[r].cpu().numpy(), np.float32(ref), rtol=2e-3, atol=2e-3)
    for e in range(E):  # evaluation.py:30-33: per-episode states / actions / rewards / terminals; the rewards add up to the return
      t = traj[r][e]
      L = t['rewards'].numel()
      total_steps += L
      assert t['states'].shape == (L, 12) and t['actions'].shape == (L, 3) and t['terminals'].shape == (L, )
      assert float(t['terminals'].sum()) == 1.0 and float(t['terminals'][-1]) == 1.0
      np.testing.assert_allclose(float(t['rewards'].sum()), float(got[r, e]), rtol=1e-4, atol=1e-4)
      np.testing.assert_allclose(t['states'][0, :11].numpy(), (u[r * E + e] * 2 - 1) * 0.1, rtol=1e-6, atol=1e-7)  # environments.py:29-33 reset state
  # the device loop ran exactly as long as the longest episode and counted every environment step
  assert stats['env_steps'] == total_steps and stats['iterations'] == max(t['rewards'].numel() for tr in traj for t in tr)
  # second evaluation on the same buffers (cached device graph) without trajectories gives the same returns
  again = evaluate_agent(actor, env, E, reset_noise=torch.from_numpy(u))
  np.testing.assert_array_equal(again.cpu().numpy(), got.cpu().numpy())
  # R == 1 returns a list of floats like the reference (evaluation.py:35)
  env1 = D4RLEnv('hopper', True, replicas=1, max_episode_steps=20)
  actor1 = il_b200.SoftActor(12, 3, MODEL, replicas=1)
  out = evaluate_agent(actor1, env1, 2)
  assert isinstance(out, list) and len(out) == 2 and all(isinstance(x, float) for x in out)


def test_initialisation_follows_the_reference_rng_stream():
  """Same seed, same construction order (train.py:64,76) -> bit-identical initial weights as the CPU restatement of
  models.py:52-66 (+ spectral-norm buffers), and replica r of a batched build == a single build with seed + r."""
  import il_b200
  from oracle import port
  icfg = Cfg(state_only=False, spectral_norm=True, discriminator=Cfg(hidden_size=16, depth=1, activation='relu', reward_shaping=False, subtract_log_policy=False, reward_function='AIRL'))
  torch.manual_seed(7)
  actor, critic = il_b200.SoftActor(12, 3, MODEL), il_b200.TwinCritic(12, 3, MODEL)
  disc = il_b200.GAILDiscriminator(12, 3, icfg, 0.97)
  torch.manual_seed(7)
  ref_actor = port.init_mlp([12, 32, 32, 6])
  ref_c1, ref_c2 = port.init_mlp([15, 32, 32, 1]), port.init_mlp([15, 32, 32, 1])
  g0 = port.init_mlp([15, 16], final_gain=2 ** 0.5)
  u0, v0 = port.spectral_norm_init(g0[0])
  for got, ref in ((actor.mlp.export_params(0, 0), ref_actor), (critic.mlp.export_params(0, 0), ref_c1), (critic.mlp.export_params(0, 1), ref_c2)):
    for a, b in zip(got, ref): assert torch.equal(a, b)
  assert torch.equal(disc.mlp.export_params(0, 0)[0], g0[0])
  np.testing.assert_allclose(disc.u[0, :16].cpu().numpy(), u0.numpy(), atol=1e-7)
  rng = il_b200.ReplicaRNG(7, 3)
  batched = il_b200.SoftActor(12, 3, MODEL, replicas=3, rng=rng)
  torch.manual_seed(9)
  single = il_b200.SoftActor(12, 3, MODEL)
  for a, b in zip(batched.mlp.export_params(2, 0), single.mlp.export_params(0, 0)): assert torch.equal(a, b)


def test_state_dict_uses_reference_keys():
  import il_b200
  icfg = Cfg(state_only=False, spectral_norm=True, discriminator=Cfg(hidden_size=16, depth=1, activation='relu', reward_shaping=False, subtract_log_policy=False, reward_function='AIRL'))
  actor, critic, disc = il_b200.SoftActor(12, 3, MODEL), il_b200.TwinCritic(12, 3, MODEL), il_b200.GAILDiscriminator(12, 3, icfg, 0.97)
  assert list(actor.state_dict()) == [f'actor.{l}.{n}' for l in (0, 2, 4) for n in ('weight', 'bias')]
  assert list(critic.state_dict()) == [f'critic_{t}.critic.{l}.{n}' for t in (1, 2) for l in (0, 2, 4) for n in ('weight', 'bias')]
  assert set(disc.state_dict()) == {f'g.{l}.{k}' for l in (0, 2) for k in ('bias', 'parametrizations.weight.original', 'parametrizations.weight.0._u', 'parametrizations.weight.0._v')}
  assert actor.state_dict()['actor.0.weight'].shape == (32, 12) and disc.state_dict()['g.2.parametrizations.weight.original'].shape == (1, 16)
  sd = actor.state_dict()
  sd['actor.4.bias'] = sd['actor.4.bias'] + 1
  actor.load_state_dict(sd)
  assert torch.allclose(actor.state_dict()['actor.4.bias'], sd['actor.4.bias'])


def test_drop_in_calls_with_reference_shapes():
  """The R = 1 call sequence of train.py:152-203 with the reference's argument / return shapes."""
  import il_b200
  from il_b200.environments import D4RLEnv
  torch.manual_seed(0)
  np.random.seed(0)
  env = D4RLEnv('hopper', True, load_data=True)
  env.seed(0)
  S, A = env.observation_space.shape[0], env.action_space.shape[0]
  assert (S, A) == (12, 3)
  actor, critic, log_alpha = il_b200.SoftActor(S, A, MODEL), il_b200.TwinCritic(S, A, MODEL), torch.zeros(1, device='cuda')
  target = il_b200.create_target_network(critic)
  oa, oc, ot = il_b200.AdamW(actor.parameters(), lr=3e-4, weight_decay=0), il_b200.AdamW(critic.parameters(), lr=3e-4, weight_decay=0), il_b200.Adam([log_alpha], lr=3e-4)
  memory = il_b200.ReplayMemory(500, S, A, True)
  state, t = env.reset(), 0
  assert state.shape == (1, S)
  for step in range(1, 81):
    policy = actor(state)
    action = policy.sample()
    assert action.shape == (1, A) and policy.log_prob(action).shape == (1, )
    next_state, reward, terminal = env.step(action)
    assert isinstance(reward, float) and isinstance(terminal, bool)
    t += 1
    memory.append(step, state, action, reward, next_state, terminal and t != env.max_episode_steps, t == env.max_episode_steps)
    state = next_state
    if terminal:
      if t != env.max_episode_steps: memory.wrap_for_absorbing_states()
      state, t = env.reset(), 0
  assert memory.idx >= 80 and not memory.full
  tr = memory.sample(16)
  assert tr['states'].shape == (16, S) and tr['absorbing'].shape == (16, ) and set(tr.keys()) >= {'step', 'states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights', 'absorbing'}
  tr['rewards'] = torch.ones(16, device='cuda')  # in-place relabelling like train.py:194
  assert float(tr.rows[0, :, tr.off['rewards']].sum()) == 16.0
  before = actor.state_dict()['actor.0.weight'].clone()
  log_probs, q = il_b200.sac_update(actor, critic, log_alpha, target, tr, oa, oc, ot, 0.99, -3.0, 0.995)
  assert log_probs.shape == (16, ) and q.shape == (16, )
  assert not torch.equal(before, actor.state_dict()['actor.0.weight'])
  # plain dicts of tensors (the reference's transitions type) are accepted too
  d = {k: tr[k].clone() for k in tr.keys()}
  il_b200.sac_update(actor, critic, log_alpha, target, d, oa, oc, ot, 0.99, -3.0, 0.995)
  assert actor.get_greedy_action(state).shape == (1, A) and actor.log_prob(state, action).shape == (1, )
  q1, q2 = critic(state, action)
  assert q1.shape == (1, ) and q2.shape == (1, )
  expert = env.get_dataset(trajectories=2, subsample=5)
  assert expert.num_trajectories == 2 and expert['states'].shape[1] == S


def test_cuda_graph_replay_equals_eager():
  import il_b200
  from il_b200.config import load_config
  from il_b200.train import Trainer
  outs = []
  for graphs in ('true', 'false'):
    cfg = load_config(['algorithm=GAIL', 'env=hopper', 'steps=40', 'training.start=6', 'training.batch_size=16', 'imitation.trajectories=2', 'reinforcement.actor.hidden_size=32',
                       'reinforcement.critic.hidden_size=32', f'cuda_graphs={graphs}', 'replicas=3', 'seed=1'])
    tr = Trainer(cfg)
    for _ in range(14): tr.train_step()
    torch.cuda.synchronize()
    outs.append((tr.actor.mlp.flat.clone(), tr.critic.mlp.flat.clone(), tr.discriminator.mlp.flat.clone(), tr.state.clone(), tr.memory._idx.clone()))
    assert tr.total_launches() > 0
    if graphs == 'true': assert 'step+update' in tr.graphs
  for a, b in zip(*outs): assert torch.equal(a, b)


def test_device_index_sampling_respects_memory_py_rules():
  import il_b200
  mem = il_b200.ReplayMemory(10, 12, 3, True, replicas=2)
  z = lambda *s: torch.zeros(*s, device='cuda')
  for i in range(7): mem.append(float(i + 1), z(2, 12), z(2, 3), 0.0, z(2, 12), 0.0, 0.0)
  idx = mem.sample_indices_device(4096)
  assert int(idx.min()) == 0 and int(idx.max()) == 5  # not full: randint(0, idx - 1) (memory.py:54)
  for i in range(8): mem.append(float(i + 8), z(2, 12), z(2, 3), 0.0, z(2, 12), 0.0, 0.0)
  assert bool(mem._full.all()) and int(mem._idx[0]) == 5
  idx = mem.sample_indices_device(8192)
  counts = torch.bincount(idx.flatten().long(), minlength=10)
  assert int(counts[4]) == 0 and int((counts > 0).sum()) == 9  # full: never the newest row (memory.py:55)
  u = torch.rand(2, 64, device='cuda')
  idx_u = mem.sample_indices_device(64, uniform=u)
  assert int(idx_u.max()) <= 9 and not bool((idx_u == 4).any())


def test_bc_pretraining_reduces_the_cloning_loss():
  """BASELINE.json configs[0] (BC hopper, 5 expert trajectories) on the accelerated path: the maximum-likelihood loss of
  training.py:62 must go down over pretraining, for every replica."""
  import il_b200
  from il_b200.config import load_config
  from il_b200.train import Trainer
  cfg = load_config(['algorithm=BC', 'env=hopper', 'steps=10', 'bc_pretraining.iterations=150', 'training.batch_size=64', 'imitation.trajectories=5', 'reinforcement.actor.hidden_size=64',
                     'reinforcement.critic.hidden_size=64', 'replicas=3', 'seed=2', 'bc_pretraining.learning_rate=0.001'])
  tr = Trainer(cfg)
  first = tr.bc_pretrain(1).clone()
  last = tr.bc_pretrain(150)
  assert bool((last < first).all()), (first, last)
  assert bool(torch.isfinite(last).all())


def test_twin_critic_forward_and_target_update_match_oracle():
  """models.py:123-141 and models.py:72-81 through il_critic_forward / il_polyak, 3 replicas."""
  import il_b200
  from oracle import port
  R, n, S, A = 3, 40, 12, 3
  torch.manual_seed(4)
  critic = il_b200.TwinCritic(S, A, MODEL, replicas=R, rng=il_b200.ReplicaRNG(4, R))
  s, a = torch.randn(R, n, S, device='cuda'), torch.tanh(torch.randn(R, n, A, device='cuda'))
  q1, q2 = critic(s, a)
  for r in range(R):
    ref1, ref2 = port.twin_critic_forward([critic.mlp.export_params(r, 0), critic.mlp.export_params(r, 1)], s[r].cpu(), a[r].cpu())
    np.testing.assert_allclose(q1[r].cpu().numpy(), ref1.numpy(), rtol=1e-4, atol=1e-5)
    np.testing.assert_allclose(q2[r].cpu().numpy(), ref2.numpy(), rtol=1e-4, atol=1e-5)
  target = il_b200.create_target_network(critic)
  assert target.mlp.flat.data_ptr() != critic.mlp.flat.data_ptr() and torch.equal(target.mlp.flat, critic.mlp.flat)
  critic.mlp.flat.add_(0.5)
  before = target.mlp.flat.clone()
  il_b200.update_target_network(critic, target, 0.99)
  np.testing.assert_allclose(target.mlp.flat.cpu().numpy(), (before * 0.99 + (1 - 0.99) * critic.mlp.flat).cpu().numpy(), rtol=1e-6, atol=1e-7)


def test_separate_wrap_call_equals_fused_wrap_and_transfer():
  """memory.py:65-68 as its own call (the reference's call pattern, train.py:157,162) == the fused append+wrap the
  trainer uses; transfer_transitions (memory.py:46-48) copies every row with weight 1."""
  import il_b200
  rs = np.random.RandomState(0)
  S, A, n = 12, 3, 20
  a, b = il_b200.ReplayMemory(50, S, A, True), il_b200.ReplayMemory(50, S, A, True)
  f = lambda *s: torch.from_numpy(rs.standard_normal(s).astype(np.float32)).cuda()
  for i in range(n):
    st, ac, ns, rw, term = f(1, S), f(1, A), f(1, S), float(rs.standard_normal()), bool(i % 6 == 5)
    a.append(i + 1, st, ac, rw, ns, term, False)
    if term: a.wrap_for_absorbing_states()
    b.append(float(i + 1), st, ac, rw, ns, float(term), 0.0, wrap=True)
  assert torch.equal(a.rows, b.rows) and a.idx == b.idx == n + 3 and a.num_trajectories == b.num_trajectories == 3
  c = il_b200.ReplayMemory(50, S, A, True)
  src = il_b200.ReplayMemory(a.idx, S, A, True, transitions=dict(states=a.states[:a.idx], actions=a.actions[:a.idx], rewards=a.rewards[:a.idx], next_states=a.next_states[:a.idx],
                                                                terminals=a.terminals[:a.idx], timeouts=a.timeouts[:a.idx], weights=a.weights[:a.idx] * 0.5, num_trajectories=3))
  c.transfer_transitions(src)
  assert c.idx == a.idx and torch.equal(c.states[:a.idx], a.states[:a.idx]) and bool((c.weights[:a.idx] == 1).all())


def test_evaluate_agent_many_episodes_uses_the_general_mlp_path():
  """More than 32 episodes per replica: the loop body runs the per-layer MLP program instead of the fused small-batch kernel."""
  import il_b200
  from il_b200.environments import D4RLEnv
  from il_b200.evaluation import evaluate_agent
  R, E = 2, 40
  env = D4RLEnv('halfcheetah', True, replicas=R, max_episode_steps=25)
  actor = il_b200.SoftActor(18, 6, MODEL, replicas=R)
  u = np.random.RandomState(5).uniform(size=(R * E, env.obs)).astype(np.float32)
  big = evaluate_agent(actor, env, E, reset_noise=torch.from_numpy(u))
  env2 = D4RLEnv('halfcheetah', True, replicas=R, max_episode_steps=25)
  small = torch.stack([evaluate_agent(actor, env2, 20, reset_noise=torch.from_numpy(u.reshape(R, E, -1)[:, h * 20:(h + 1) * 20].reshape(R * 20, -1).copy())) for h in range(2)], dim=1).reshape(R, E)
  np.testing.assert_allclose(big.cpu().numpy(), small.cpu().numpy(), rtol=1e-4, atol=1e-4)


def test_evaluate_agent_on_the_tensor_core_engine_pads_rows_and_matches_fp32():
  """30 episodes per replica with 256-wide nets and gemm_mode tf32x3 (train.py:213 at the benchmarked configuration): the greedy forward pads every
  replica's rows to the 128-row wgmma tile (zero rows, ignored) — same returns as the fp32 FFMA engine, which runs the 30 rows unpadded."""
  import il_b200
  from il_b200 import _lib
  from il_b200.environments import D4RLEnv
  from il_b200.evaluation import evaluate_agent
  R, E = 3, 30
  cfg = type(MODEL)(hidden_size=256, depth=2, activation='relu')
  actor = il_b200.SoftActor(12, 3, cfg, replicas=R)
  u = np.random.RandomState(11).uniform(size=(R * E, 11)).astype(np.float32)
  lib, h = _lib.lib(), _lib.handle()
  out = {}
  for mode in ('fp32', 'tf32x3'):
    _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE[mode]))
    try:
      env = D4RLEnv('hopper', True, replicas=R, max_episode_steps=60)
      stats = {}
      out[mode] = (evaluate_agent(actor, env, E, reset_noise=torch.from_numpy(u), out_stats=stats).cpu().numpy(), dict(stats))
    finally:
      _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE['fp32']))
  np.testing.assert_allclose(out['tf32x3'][0], out['fp32'][0], rtol=2e-3, atol=2e-3)
  assert out['tf32x3'][1] == out['fp32'][1]  # same loop length and environment-step count: the padded rows are not episodes


def test_return_allreduce_single_process_matches_torch():
  from il_b200 import distributed
  r = torch.randn(7, 30, device='cuda') * 10
  s = distributed.return_stats_device(r).cpu()
  np.testing.assert_allclose(s.numpy(), [float(r.sum()), float((r * r).sum()), 210.0], rtol=1e-5)
  mean, std, n = distributed.return_statistics(r)
  assert n == 210 and abs(mean - float(r.mean())) < 1e-3 and abs(std - float(r.std(unbiased=False))) < 1e-2


@pytest.mark.parametrize('polyak', [False, True])
def test_adam_tma_staged_kernel_is_bitwise_the_plain_kernel(polyak):
  """AdamW (+ fused polyak) with TMA staging (cp.async.bulk tiles through shared memory, mbarrier complete_tx, a copy thread feeding 256 compute
  threads) against the plain 128-bit streaming kernel: same arithmetic, so bit-identical parameters / moments / target for every tile / ring
  geometry, including a ragged last tile and CTAs with different tile counts."""
  import il_b200
  from il_b200 import _lib
  n = 4096 * 148 * 2 * 3 + 2048 * 3 + 12  # > the switch-over size, several tiles per CTA, not a multiple of any tile
  torch.manual_seed(0)
  p0, g = torch.randn(n, device='cuda'), torch.randn(n, device='cuda') * 0.1
  outs = []
  lib, h = _lib.lib(), _lib.handle()
  for tma in range(8):
    _lib.set_option('adam_tma', tma)
    try:
      p, tgt = p0.clone(), p0.clone() * 0.5
      opt = il_b200.AdamW([p], lr=1e-3, weight_decay=0.01)
      opt.exp_avg.copy_(torch.sin(p0)); opt.exp_avg_sq.copy_(torch.cos(p0) ** 2)
      a = opt.c_struct()
      for _ in range(2):
        if polyak: _lib.check(lib.il_adam_step_polyak(h, p.data_ptr(), g.data_ptr(), C.byref(a), n, tgt.data_ptr(), 0.995, _lib.stream()))
        else: _lib.check(lib.il_adam_step(h, p.data_ptr(), g.data_ptr(), C.byref(a), n, _lib.stream()))
      torch.cuda.synchronize()
      outs.append((p.clone(), opt.exp_avg.clone(), opt.exp_avg_sq.clone(), tgt.clone()))
    finally:
      _lib.set_option('adam_tma', 1)
  for variant, o in enumerate(outs[1:], 1):
    for x, y in zip(outs[0], o): assert torch.equal(x, y), f'adam_tma={variant}'
