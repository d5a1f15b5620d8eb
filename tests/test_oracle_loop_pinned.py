"""Pins oracle/loop.py — the restated step schedule of train.py:146-227 that the GPU loop tests and the CPU baseline are
built on — against the reference's REAL `train.train(cfg)`: the unmodified train.py / environments.py / memory.py /
models.py / training.py / evaluation.py run end to end (oracle/ref_train.py stubs only hydra, plotting and `gym.make`,
which returns the synthetic-environment twin) and the oracle loop, fed by the same global torch / numpy RNG streams,
must arrive at the same parameters after the same number of steps. What the reference's train() wrote is stored in
tests/golden/reference.npz (python -m oracle.ref_golden regenerates it next to the reference tree)."""
import numpy as np
import pytest
import torch

from il_b200 import config
from oracle import loop, ref_golden

STEPS, MAX_EPISODE_STEPS, B, H, START = 60, 25, 16, 32, 8
ATOL = 2e-6  # fp32, same torch CPU ops on both sides; observed 3e-8 after 60 steps


def _cfg(algorithm, env, seed, extra=()):
  cfg = config.load_config([f'algorithm={algorithm}', f'env={env}', f'steps={STEPS}', f'training.start={START}', f'training.batch_size={B}', f'reinforcement.actor.hidden_size={H}',
                            f'reinforcement.critic.hidden_size={H}', 'imitation.trajectories=3', f'evaluation.interval={STEPS}', 'evaluation.episodes=2', 'logging.interval=10',
                            'memory.size=1000', f'seed={seed}', *extra])
  for k in ('replicas', 'device_rng', 'cuda_graphs', 'gemm_mode', 'output_dir'): cfg.pop(k, None)  # keys this build adds
  return cfg


def _close(name, ref, mine, atol=ATOL):
  ref, mine = torch.as_tensor(ref).detach().float(), torch.as_tensor(mine).detach().float()
  assert ref.shape == mine.shape, (name, ref.shape, mine.shape)
  err = float((ref - mine).abs().max())
  assert err <= atol * max(1.0, float(ref.abs().max())), f'{name}: max abs err {err:.3e}'


CONFIGS = [
  # (algorithm, env, reference-side overrides, oracle-loop kwargs)
  ('GAIL', 'hopper', (), {}),
  ('GAIL', 'walker2d', ('imitation.mix_expert_data=mixed_batch', ), dict(mix_expert_data='mixed_batch')),
  ('GAIL', 'hopper', ('imitation.loss_function=Mixup', 'imitation.entropy_bonus=0.1', 'imitation.grad_penalty=0.5'), dict(imitation=dict(loss_function='Mixup', entropy_bonus=0.1, grad_penalty=0.5))),
  ('GAIL', 'hopper', ('imitation.loss_function=PUGAIL', 'imitation.nonnegative_margin=0.3', 'imitation.grad_penalty=0', 'imitation.spectral_norm=false',
                      'imitation.discriminator.reward_function=FAIRL'),
   dict(imitation=dict(loss_function='PUGAIL', nonnegative_margin=0.3, grad_penalty=0.0, spectral_norm=False, reward_function='FAIRL'))),
  ('GAIL', 'hopper', ('imitation.bc_aux_loss=true', ), dict(bc_aux_loss=True)),
  ('GAIL', 'hopper', ('imitation.discriminator.reward_shaping=true', 'imitation.discriminator.subtract_log_policy=true', 'imitation.discriminator.hidden_size=16'),
   dict(imitation=dict(reward_shaping=True, subtract_log_policy=True, hidden_size=16))),
  ('GAIL', 'halfcheetah', ('imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh', 'imitation.discriminator.hidden_size=16', 'imitation.discriminator.reward_function=GAIL'),
   dict(imitation=dict(depth=2, activation='tanh', hidden_size=16, reward_function='GAIL'))),
  ('GAIL', 'hopper', ('imitation.state_only=true', 'imitation.grad_penalty=0', 'imitation.discriminator.activation=sigmoid', 'imitation.discriminator.reward_shaping=true'),
   dict(imitation=dict(state_only=True, grad_penalty=0.0, activation='sigmoid', reward_shaping=True))),
  # AdRIL (balanced alternation, rounds of 20 steps so several round boundaries fall inside the run), unbalanced AdRIL, SQIL (update_freq 0)
  ('AdRIL', 'hopper', ('imitation.update_freq=20', ), dict(mix_expert_data='mixed_batch', imitation=dict(update_freq=20, balanced=True))),
  ('AdRIL', 'walker2d', ('imitation.update_freq=15', 'imitation.balanced=false'), dict(mix_expert_data='mixed_batch', imitation=dict(update_freq=15, balanced=False))),
  ('AdRIL', 'hopper', ('imitation.update_freq=0', ), dict(mix_expert_data='mixed_batch', imitation=dict(update_freq=0, balanced=True))),
  # DRIL (dropout policy ensemble, BC pretraining, quantile threshold, MC-dropout reward; bc_aux_loss from DRIL.yaml) and RED (predictor / target
  # embeddings, regression pretraining, median-heuristic bandwidth, with and without dropout / prefill)
  ('DRIL', 'hopper', ('imitation.pretraining.iterations=9', 'imitation.discriminator.hidden_size=16'),
   dict(bc_aux_loss=True, imitation=dict(hidden_size=16, activation='tanh', input_dropout=0.1, dropout=0.1, pretraining_iterations=9, learning_rate=3e-5, weight_decay=0.0))),
  ('DRIL', 'walker2d', ('imitation.pretraining.iterations=5', 'imitation.discriminator.hidden_size=16', 'imitation.discriminator.depth=2', 'imitation.discriminator.dropout=0.4',
                        'imitation.mix_expert_data=mixed_batch', 'imitation.quantile_cutoff=0.9', 'imitation.bc_aux_loss=false'),
   dict(mix_expert_data='mixed_batch', imitation=dict(hidden_size=16, depth=2, activation='tanh', input_dropout=0.1, dropout=0.4, pretraining_iterations=5, quantile_cutoff=0.9,
                                                      learning_rate=3e-5, weight_decay=0.0))),
  ('RED', 'hopper', ('imitation.pretraining.iterations=11', ), dict(imitation=dict(hidden_size=32, pretraining_iterations=11, learning_rate=3e-5, weight_decay=0.0))),
  ('RED', 'halfcheetah', ('imitation.pretraining.iterations=6', 'imitation.discriminator.input_dropout=0.2', 'imitation.discriminator.dropout=0.3', 'imitation.discriminator.depth=2',
                          'imitation.mix_expert_data=prefill_memory', 'imitation.weight_decay=0.5'),
   dict(mix_expert_data='prefill_memory', imitation=dict(hidden_size=32, depth=2, input_dropout=0.2, dropout=0.3, pretraining_iterations=6, learning_rate=3e-5, weight_decay=0.5))),
  ('SAC', 'hopper', (), {}),
  ('SAC', 'ant', ('training.weight_decay=0.01', ), dict(weight_decay=0.01)),
  ('GMMIL', 'halfcheetah', (), {}),
  ('GMMIL', 'hopper', ('imitation.mix_expert_data=mixed_batch', ), dict(mix_expert_data='mixed_batch')),
  ('GMMIL', 'hopper', ('imitation.mix_expert_data=prefill_memory', ), dict(mix_expert_data='prefill_memory')),
  ('PWIL', 'hopper', (), {}),
  ('PWIL', 'hopper', ('imitation.mix_expert_data=mixed_batch', ), dict(mix_expert_data='mixed_batch')),
  ('PWIL', 'walker2d', ('imitation.mix_expert_data=prefill_memory', ), dict(mix_expert_data='prefill_memory')),
]


CONFIG_IDS = [f'{a}-{e}-{i}' for i, (a, e, _, _) in enumerate(CONFIGS)]
LOOP_SEED = 3


@pytest.mark.parametrize('case_id,algorithm,env,extra,kwargs', [(i, *c) for i, c in zip(CONFIG_IDS, CONFIGS)], ids=CONFIG_IDS)
def test_restated_loop_equals_the_reference_train_function(case_id, algorithm, env, extra, kwargs):
  seed = LOOP_SEED
  raw = loop.synthesize_raw_dataset(env, True, 5, MAX_EPISODE_STEPS)
  ref = ref_golden.load_train_result(case_id)  # the reference's train(_cfg(algorithm, env, seed, extra)) on the same raw dataset

  threads = torch.get_num_threads()
  torch.set_num_threads(1)
  try:
    ol = loop.OracleLoop(algorithm, env, seed=seed, batch_size=B, start=START, memory_size=STEPS, hidden_size=H, trajectories=3, max_episode_steps=MAX_EPISODE_STEPS,
                         expert_raw=raw, **kwargs)
    if algorithm in ('DRIL', 'RED'): ol.pretrain_discriminator()
    for _ in range(STEPS): ol.run_step()
  finally:
    torch.set_num_threads(threads)

  for i, (k, v) in enumerate(ref['agent']['actor'].items()): _close(f'actor.{k}', v, ol.agent.actor[i])
  critic = list(ref['agent']['critic'].items())
  assert len(critic) == 12
  for t in range(2):
    for i in range(6): _close(f'critic.{critic[6 * t + i][0]}', critic[6 * t + i][1], ol.agent.twin[t][i])
  _close('log_alpha', ref['agent']['log_alpha'], ol.agent.log_alpha)
  if algorithm == 'DRIL':  # discriminator.pth = the dropout policy's state dict (train.py:238)
    for i, (k, v) in enumerate(ref['discriminator'].items()): _close(f'dril.{k}', v, ol.disc[i])
  if algorithm == 'RED':
    sd = ref['discriminator']
    for i, (k, v) in enumerate((k, v) for k, v in sd.items() if k.startswith('predictor')): _close(f'red.{k}', v, ol.disc.predictor[i])
    for i, (k, v) in enumerate((k, v) for k, v in sd.items() if k.startswith('target')): _close(f'red.{k}', v, ol.disc.target[i])
  if algorithm == 'GAIL':
    sd, sn = ref['discriminator'], ol.disc.g_sn is not None
    for net, params, bufs in (('g', ol.disc.g, ol.disc.g_sn), ('h', ol.disc.h, ol.disc.h_sn)):
      if params is None: continue
      single = net == 'g' and ol.disc.h is not None  # with reward shaping g is one nn.Linear, not a Sequential (models.py:157)
      for l in range(len(params) // 2):
        pre = net if single else f'{net}.{[i for i in range(99) if f"{net}.{i}.bias" in sd][l]}'
        _close(f'{pre}.weight', sd[f'{pre}.parametrizations.weight.original' if sn else f'{pre}.weight'], params[2 * l])
        _close(f'{pre}.bias', sd[f'{pre}.bias'], params[2 * l + 1])
        if sn:
          # singular-vector estimates are ill-conditioned when the two largest singular values are close: 10x looser
          _close(f'{pre}.u', sd[f'{pre}.parametrizations.weight.0._u'], bufs[l][0], atol=10 * ATOL)
          _close(f'{pre}.v', sd[f'{pre}.parametrizations.weight.0._v'], bufs[l][1], atol=10 * ATOL)
    assert sum(k.endswith('bias') for k in sd) == (len(ol.disc.g) + len(ol.disc.h or [])) // 2
  # episode bookkeeping (train.py:161-168) and the logged tensors of the last logging step (train.py:205-210)
  got = [r[0] for r in ref['metrics']['train_returns']]
  assert len(got) == len(ol.episode_returns) and np.allclose(got, ol.episode_returns, rtol=1e-5, atol=1e-6)
  assert ref['metrics']['update_steps'] == [s for s in range(10, STEPS + 1, 10) if s >= START]
  _close('predicted_rewards', ref['metrics']['predicted_rewards'][-1], ol.last['rewards'])
  _close('q_values', ref['metrics']['Q_values'][-1], ol.last['sac']['q_values'])
  _close('entropies', ref['metrics']['entropies'][-1], -ol.last['sac']['log_probs'])


BC_CONFIGS, BC_SEED, BC_ENV = [('BC', 25), ('GAIL', 7)], 5, 'hopper'


def _bc_cfg(algorithm, iterations):
  return _cfg(algorithm, BC_ENV, BC_SEED, [f'bc_pretraining.iterations={iterations}', 'bc_pretraining.learning_rate=0.001', 'bc_pretraining.weight_decay=0.01'])


@pytest.mark.parametrize('algorithm,iterations', BC_CONFIGS)
def test_bc_pretraining_equals_the_reference(algorithm, iterations):
  """train.py:95-115: BC on shuffled expert minibatches (the DataLoader's shuffling stream restated in OracleLoop.bc_pretrain);
  algorithm=BC returns after pretraining + evaluation, any other algorithm continues into the loop with the pretrained actor."""
  from oracle import port
  seed, env = BC_SEED, BC_ENV
  raw = loop.synthesize_raw_dataset(env, True, 5, MAX_EPISODE_STEPS)
  ref = ref_golden.load_train_result(f'bc-{algorithm}-{iterations}')  # the reference's train(_bc_cfg(algorithm, iterations))
  threads = torch.get_num_threads()
  torch.set_num_threads(1)
  try:
    ol = loop.OracleLoop('SAC' if algorithm == 'BC' else algorithm, env, seed=seed, batch_size=B, start=START, memory_size=STEPS, hidden_size=H, trajectories=3,
                         max_episode_steps=MAX_EPISODE_STEPS, expert_raw=raw, build_expert_memory=True)
    ol.bc_pretrain(iterations, 0.001, 0.01)
    if algorithm != 'BC':
      for _ in range(STEPS): ol.run_step()
  finally:
    torch.set_num_threads(threads)
  for i, (k, v) in enumerate(ref['agent']['actor'].items()): _close(f'actor.{k}', v, ol.agent.actor[i])
  if algorithm == 'BC':
    assert set(ref['agent']) == {'actor'}  # train.py:111
    # the evaluation of train.py:104 on the evaluation env's own reset stream (second env made, oracle/ref_train.py)
    g = torch.Generator().manual_seed(seed + 10007)
    eval_env = port.SyntheticEnv(env, True, MAX_EPISODE_STEPS)
    noise = [torch.rand(eval_env.obs, generator=g) for _ in range(2)]
    mine = port.evaluate_agent(ol.agent.actor, eval_env, 2, noise)
    assert np.allclose(ref['metrics']['test_returns'][0], mine, rtol=1e-5, atol=1e-6)
    assert abs(ref['score'] - np.mean(mine) / 1000.0) < 1e-7
  else:
    _close('log_alpha', ref['agent']['log_alpha'], ol.agent.log_alpha)
