"""TEST INFRASTRUCTURE ONLY — seeded parity cases shared by the golden generator and the tests.

`make_inputs(case)` builds every input (weights, batches, injected noise / indices) from
`np.random.RandomState(seed)` (stream stable across numpy versions and machines), so the committed fixtures
in `tests/golden/` only need to store the REFERENCE'S OUTPUTS. `run_reference` drives the unmodified
reference modules (container only); `run_port` drives `oracle/port.py`; the GPU tests drive the CUDA path on
the same inputs (tests/cuda_cases.py).
"""
from __future__ import annotations

import contextlib
import math
from typing import Dict, List

import numpy as np
import torch

from . import port

# name -> config. `full` cases are stored completely; the others as sampled entries + moments.
CASES: Dict[str, dict] = {
  'actor_small': dict(kind='actor', S=12, A=3, H=32, n=16, seed=11),
  'actor_hopper': dict(kind='actor', S=12, A=3, H=256, n=256, seed=12),
  'sac_small': dict(kind='sac', S=12, A=3, H=32, B=16, steps=2, seed=21, discount=0.97, entropy_target=-1.5, polyak=0.99, lr=3e-4, wd=0.0),
  'sac_small_wd': dict(kind='sac', S=18, A=6, H=48, B=24, steps=3, seed=22, discount=0.99, entropy_target=-6.0, polyak=0.995, lr=1e-3, wd=0.01),
  'sac_hopper': dict(kind='sac', S=12, A=3, H=256, B=256, steps=2, seed=23, discount=0.97, entropy_target=-1.5, polyak=0.99, lr=3e-4, wd=0.0),
  'sac_ant_small': dict(kind='sac', S=112, A=8, H=64, B=32, steps=2, seed=24, discount=0.99, entropy_target=-8.0, polyak=0.995, lr=3e-4, wd=0.0),
  'bc_small': dict(kind='bc', S=12, A=3, H=32, B=24, steps=3, seed=25, lr=2.5e-4, wd=0.01),
  'bc_hopper': dict(kind='bc', S=12, A=3, H=256, B=256, steps=2, seed=26, lr=2.5e-4, wd=0.0),
  'gail_default': dict(kind='gail', S=12, A=3, H=64, B=256, steps=2, seed=31, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.0, loss='BCE', lr=3e-5, wd=10.0, reward='AIRL'),
  'gail_entropy_nosn': dict(kind='gail', S=18, A=6, H=32, B=64, steps=2, seed=32, spectral_norm=False, grad_penalty=0.5, entropy_bonus=0.1, loss='BCE', lr=1e-3, wd=0.1, reward='GAIL'),
  'gail_pugail': dict(kind='gail', S=12, A=3, H=64, B=64, steps=2, seed=33, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.0, loss='PUGAIL', lr=1e-3, wd=0.0, reward='FAIRL'),
  'gail_mixup': dict(kind='gail', S=12, A=3, H=64, B=64, steps=2, seed=34, spectral_norm=True, grad_penalty=0.0, entropy_bonus=0.0, loss='Mixup', lr=1e-3, wd=0.0, reward='AIRL'),
  'gail_ant': dict(kind='gail', S=112, A=8, H=64, B=96, steps=2, seed=35, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.05, loss='BCE', lr=3e-5, wd=10.0, reward='AIRL'),
  # the published tuned configurations (conf/optimised_hyperparameters/GAIL_{5,25}_trajectories.yaml): B = 1024 with Mixup + gradient
  # penalty + entropy bonus + spectral norm together; a 128-wide discriminator with the GAIL reward
  'gail_tuned5': dict(kind='gail', S=12, A=3, H=64, B=1024, steps=2, seed=301, spectral_norm=True, grad_penalty=0.2799364347010851, entropy_bonus=0.24145587952807546, loss='Mixup',
                      lr=0.0002778119723405689, wd=8.46588535234332, reward='AIRL'),
  'gail_tuned25': dict(kind='gail', S=12, A=3, H=128, B=256, steps=2, seed=302, spectral_norm=True, grad_penalty=0.3203035416081548, entropy_bonus=0.015492475591599941, loss='BCE',
                       lr=7.299440972507e-05, wd=6.3524082861840725, reward='GAIL'),
  'gmmil_ant': dict(kind='gmmil', S=112, A=8, B=300, seed=43),
  # SURVEY §8f row 3 variants (csrc/gail_general.cu): shaping f = g(s,a) + (1-t)(gamma h(s') - h(s)) with a
  # linear g (models.py:157-160), subtract_log_policy (:175), deeper / tanh / sigmoid / state-only discriminators
  'gailx_shaping': dict(kind='gailx', S=12, A=3, H=32, depth=1, activation='relu', B=48, steps=2, seed=36, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.05, loss='BCE',
                        lr=1e-3, wd=0.1, reward='AIRL', reward_shaping=True, subtract_log_policy=True, state_only=False),
  'gailx_depth2_tanh': dict(kind='gailx', S=12, A=3, H=32, depth=2, activation='tanh', B=48, steps=2, seed=37, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.0, loss='BCE',
                            lr=1e-3, wd=0.1, reward='GAIL', reward_shaping=False, subtract_log_policy=False, state_only=False),
  'gailx_state_only_sigmoid': dict(kind='gailx', S=18, A=6, H=32, depth=2, activation='sigmoid', B=48, steps=2, seed=38, spectral_norm=False, grad_penalty=0.0, entropy_bonus=0.1, loss='Mixup',
                                   lr=1e-3, wd=0.0, reward='FAIRL', reward_shaping=True, subtract_log_policy=False, state_only=True),
  # the rest of the general program's branches: a linear g (depth 0) under the gradient penalty; PUGAIL with a finite margin whose clamp acts;
  # a depth-2 tanh h under Mixup + gradient penalty + log-policy term; a depth-3 sigmoid g (the middle layers of the penalty's double backward)
  'gailx_linear_gp': dict(kind='gailx', S=12, A=3, H=32, depth=0, activation='relu', B=48, steps=2, seed=391, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.0, loss='BCE',
                          lr=1e-3, wd=0.1, reward='AIRL', reward_shaping=False, subtract_log_policy=False, state_only=False),
  'gailx_pugail_margin': dict(kind='gailx', S=12, A=3, H=32, depth=1, activation='tanh', B=48, steps=2, seed=392, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.0,
                              loss='PUGAIL', pos_class_prior=0.7, nonnegative_margin=0.05, lr=1e-3, wd=0.1, reward='GAIL', reward_shaping=False, subtract_log_policy=False,
                              state_only=False),
  'gailx_shaping_deep_mixup': dict(kind='gailx', S=12, A=3, H=32, depth=2, activation='tanh', B=48, steps=2, seed=393, spectral_norm=True, grad_penalty=1.0, entropy_bonus=0.05,
                                   loss='Mixup', lr=1e-3, wd=0.1, reward='AIRL', reward_shaping=True, subtract_log_policy=True, state_only=False),
  'gailx_depth3_sigmoid': dict(kind='gailx', S=18, A=6, H=32, depth=3, activation='sigmoid', B=48, steps=2, seed=394, spectral_norm=False, grad_penalty=0.5, entropy_bonus=0.1,
                               loss='BCE', lr=1e-3, wd=0.0, reward='FAIRL', reward_shaping=False, subtract_log_policy=False, state_only=False),
  # SURVEY §8f row 2: expert-data ingest (environments.py:63-125) on a D4RL-shaped raw buffer — host logic, no CUDA
  'ingest_absorbing_sub4': dict(kind='ingest', cuda=False, obs=11, A=3, N=900, trajectories=4, subsample=4, absorbing=True, seed=71),
  'ingest_plain_all': dict(kind='ingest', cuda=False, obs=17, A=6, N=500, trajectories=0, subsample=1, absorbing=False, seed=72),
  'ingest_absorbing_sub1': dict(kind='ingest', cuda=False, obs=11, A=3, N=700, trajectories=3, subsample=1, absorbing=True, seed=73),
  # a17: evaluation.py:11-35 on the synthetic env twin (greedy policy, sum of rewards per episode)
  'eval_hopper': dict(kind='eval', cuda=False, env='hopper', H=32, episodes=4, max_steps=80, seed=81),
  'eval_halfcheetah': dict(kind='eval', cuda=False, env='halfcheetah', H=32, episodes=3, max_steps=50, seed=82),
  # a7 / a8 / a16 around expert data: ReplayMemory(transitions=...) prefill (memory.py:18-23), transfer_transitions (:46-48), the
  # "never the last row" sampling rule of a pre-filled memory (:22-23, 55) and mix_expert_agent_transitions (models.py:287-290)
  'prefill_mix': dict(kind='mix', S=12, A=3, Ne=40, size=64, extra=9, B=16, seed=91),
  # SURVEY §8f row 4: RED (models.py:252-284, training.py:68-75) and DRIL (models.py:104-120) with every dropout mask injected
  'red_dropout': dict(kind='red', S=12, A=3, H=32, depth=2, activation='relu', input_dropout=0.2, dropout=0.3, B=48, steps=3, seed=101, lr=1e-3, wd=0.1, state_only=False),
  'red_default': dict(kind='red', S=18, A=6, H=32, depth=1, activation='relu', input_dropout=0.0, dropout=0.0, B=64, steps=2, seed=102, lr=3e-5, wd=0.0, state_only=False),
  'dril_small': dict(kind='dril', S=12, A=3, H=32, depth=1, activation='tanh', input_dropout=0.1, dropout=0.1, B=24, N=40, steps=2, seed=103, lr=1e-3, wd=0.0, quantile=0.9),
  'gmmil_hopper': dict(kind='gmmil', S=12, A=3, B=64, seed=41),
  'gmmil_halfcheetah': dict(kind='gmmil', S=18, A=6, B=256, seed=42),
  'pwil_small': dict(kind='pwil', S=12, A=3, N=150, T=40, steps=100, seed=51),
  'replay_ring': dict(kind='replay', S=12, A=3, size=37, appends=90, B=32, seed=61),
}


def _rs(seed): return np.random.RandomState(seed)


def _mlp_weights(rs, sizes, scale=1.0) -> List[np.ndarray]:
  out = []
  for i in range(len(sizes) - 1):
    out.append((rs.standard_normal((sizes[i + 1], sizes[i])) * scale / math.sqrt(sizes[i])).astype(np.float32))
    out.append((rs.standard_normal(sizes[i + 1]) * 0.1).astype(np.float32))
  return out


def _batch(rs, B, S, A, absorbing_frac=0.1) -> Dict[str, np.ndarray]:
  f = lambda *s: rs.standard_normal(s).astype(np.float32)
  states, next_states = f(B, S), f(B, S)
  absb = (rs.uniform(size=B) < absorbing_frac).astype(np.float32)
  states[:, -1] = absb
  states[absb == 1, :-1] = 0
  next_states[:, -1] = (rs.uniform(size=B) < absorbing_frac).astype(np.float32)
  actions = np.tanh(f(B, A))
  actions[absb == 1] = 0
  return dict(step=np.arange(1, B + 1, dtype=np.float32), states=states, actions=actions.astype(np.float32), rewards=f(B), next_states=next_states,
              terminals=(rs.uniform(size=B) < 0.1).astype(np.float32), timeouts=np.zeros(B, np.float32),
              weights=np.where(rs.uniform(size=B) < 0.2, 0.5, 1.0).astype(np.float32), absorbing=absb)


def make_inputs(name: str, seed_offset: int = 0) -> Dict[str, np.ndarray]:
  """seed_offset != 0 gives an independent input set of the same shapes (used to fill the replica axis)."""
  c = CASES[name]
  rs = _rs(c['seed'] + 1000 * seed_offset)
  inp: Dict[str, np.ndarray] = {}
  k = c['kind']
  if k == 'actor':
    for i, w in enumerate(_mlp_weights(rs, [c['S'], c['H'], c['H'], 2 * c['A']])): inp[f'actor_{i}'] = w
    inp['states'] = rs.standard_normal((c['n'], c['S'])).astype(np.float32)
    inp['eps'] = rs.standard_normal((c['n'], c['A'])).astype(np.float32)
    inp['actions'] = np.clip(np.tanh(rs.standard_normal((c['n'], c['A'])) * 2), -1, 1).astype(np.float32)
    inp['actions'][0, 0] = 1.0  # exercises the clamp at models.py:98
  elif k == 'sac':
    S, A, H = c['S'], c['A'], c['H']
    for i, w in enumerate(_mlp_weights(rs, [S, H, H, 2 * A])): inp[f'actor_{i}'] = w
    for t in (1, 2):
      for i, w in enumerate(_mlp_weights(rs, [S + A, H, H, 1])): inp[f'critic{t}_{i}'] = w
      for i, w in enumerate(_mlp_weights(rs, [S + A, H, H, 1])): inp[f'target{t}_{i}'] = w
    inp['log_alpha'] = np.float32([-0.3])
    for s in range(c['steps']):
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'b{s}_{key}'] = v
      inp[f'b{s}_eps_next'] = rs.standard_normal((c['B'], A)).astype(np.float32)
      inp[f'b{s}_eps_new'] = rs.standard_normal((c['B'], A)).astype(np.float32)
  elif k == 'bc':
    for i, w in enumerate(_mlp_weights(rs, [c['S'], c['H'], c['H'], 2 * c['A']])): inp[f'actor_{i}'] = w
    for s in range(c['steps']):
      for key, v in _batch(rs, c['B'], c['S'], c['A']).items(): inp[f'b{s}_{key}'] = v
      inp[f'b{s}_actions'][0, 0] = 1.0  # exercises the clamp at training.py:59
  elif k == 'gail':
    S, A, H = c['S'], c['A'], c['H']
    for i, w in enumerate(_mlp_weights(rs, [S + A, H, 1], scale=1.5)): inp[f'g_{i}'] = w
    for s in range(c['steps']):
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'p{s}_{key}'] = v
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'e{s}_{key}'] = v
      inp[f's{s}_eps_gp'] = rs.uniform(size=c['B']).astype(np.float32)
      inp[f's{s}_eps_mix'] = rs.beta(1.0, 1.0, size=c['B']).astype(np.float32)
    if c['spectral_norm']:
      for l, (h, w) in enumerate(((H, S + A), (1, H))):
        inp[f'u_{l}'] = rs.standard_normal(h).astype(np.float32)
        inp[f'v_{l}'] = rs.standard_normal(w).astype(np.float32)
  elif k == 'gailx':
    S, A, H = c['S'], c['A'], c['H']
    din = S if c['state_only'] else S + A
    g_sizes, h_sizes = ([din, 1], [S] + [H] * c['depth'] + [1]) if c['reward_shaping'] else ([din] + [H] * c['depth'] + [1], None)
    for i, w in enumerate(_mlp_weights(rs, g_sizes, scale=1.5)): inp[f'g_{i}'] = w
    if h_sizes is not None:
      for i, w in enumerate(_mlp_weights(rs, h_sizes, scale=1.5)): inp[f'h_{i}'] = w
    if c['subtract_log_policy']:
      for i, w in enumerate(_mlp_weights(rs, [S, 32, 32, 2 * A])): inp[f'actor_{i}'] = w
    for s in range(c['steps']):
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'p{s}_{key}'] = v
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'e{s}_{key}'] = v
      inp[f's{s}_eps_gp'] = rs.uniform(size=c['B']).astype(np.float32)
      inp[f's{s}_eps_mix'] = rs.beta(1.0, 1.0, size=c['B']).astype(np.float32)
    if c['spectral_norm']:
      for net, sizes in (('g', g_sizes), ('h', h_sizes)):
        if sizes is None: continue
        for l in range(len(sizes) - 1):
          inp[f'{net}u_{l}'] = rs.standard_normal(sizes[l + 1]).astype(np.float32)
          inp[f'{net}v_{l}'] = rs.standard_normal(sizes[l]).astype(np.float32)
  elif k in ('red', 'dril'):
    S, A, H = c['S'], c['A'], c['H']
    def mask(shape, p): return ((rs.uniform(size=shape) >= p) / (1.0 - p)).astype(np.float32) if p > 0 else None
    def masks(prefix, n, din):
      m = mask((n, din), c['input_dropout'])
      if m is not None: inp[f'{prefix}_in'] = m
      for l in range(c['depth']):
        m = mask((n, H), c['dropout'])
        if m is not None: inp[f'{prefix}_h{l}'] = m
    if k == 'red':
      din = S if c['state_only'] else S + A
      sizes = [din] + [H] * c['depth'] + [din]
      for i, w in enumerate(_mlp_weights(rs, sizes)): inp[f'predictor_{i}'] = w
      for i, w in enumerate(_mlp_weights(rs, sizes)): inp[f'target_{i}'] = w
      for s_ in range(c['steps']):
        for key, v in _batch(rs, c['B'], S, A).items(): inp[f'b{s_}_{key}'] = v
        masks(f'm{s_}', c['B'], din)
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'sig_{key}'] = v
      masks('msig', c['B'], din)
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'p_{key}'] = v
    else:
      for i, w in enumerate(_mlp_weights(rs, [S] + [H] * c['depth'] + [2 * A])): inp[f'actor_{i}'] = w
      for s_ in range(c['steps']):
        for key, v in _batch(rs, c['B'], S, A).items(): inp[f'b{s_}_{key}'] = v
        masks(f'm{s_}', c['B'], S)
      inp['expert_states'] = rs.standard_normal((c['N'], S)).astype(np.float32)
      inp['expert_actions'] = np.tanh(rs.standard_normal((c['N'], A))).astype(np.float32)
      masks('mthr', c['N'] * 5, S)
      for key, v in _batch(rs, c['B'], S, A).items(): inp[f'p_{key}'] = v
      masks('mrew', c['B'] * 5, S)
  elif k == 'ingest':
    N = c['N']
    inp['observations'] = rs.standard_normal((N, c['obs'])).astype(np.float32)
    inp['next_observations'] = rs.standard_normal((N, c['obs'])).astype(np.float32)
    inp['actions'] = np.tanh(rs.standard_normal((N, c['A']))).astype(np.float32)
    inp['rewards'] = rs.standard_normal(N).astype(np.float32)
    ends = np.sort(rs.choice(np.arange(20, N - 1), size=6, replace=False))  # 7 episodes of ragged length; the last one ends at N - 1
    terminals, timeouts = np.zeros(N, np.float32), np.zeros(N, np.float32)
    for j, e in enumerate(list(ends) + [N - 1]): (timeouts if j % 3 == 1 else terminals)[e] = 1  # episodes 1, 4 end by time limit
    inp['terminals'], inp['timeouts'] = terminals, timeouts
    inp['np_seed'] = np.int64([c['seed'] + 7])
  elif k == 'eval':
    env = port.SyntheticEnv(c['env'], True, c['max_steps'])
    for i, w in enumerate(_mlp_weights(rs, [env.state_size, c['H'], c['H'], 2 * env.act], scale=2.0)): inp[f'actor_{i}'] = w
    inp['reset_u'] = rs.uniform(size=(c['episodes'], env.obs)).astype(np.float32)
  elif k == 'mix':
    Ne, S, A = c['Ne'], c['S'], c['A']
    for key, v in _batch(rs, Ne, S, A).items(): inp[f'e_{key}'] = v
    inp['e_timeouts'] = (rs.uniform(size=Ne) < 0.05).astype(np.float32)
    for key, v in _batch(rs, c['extra'], S, A).items(): inp[f'x_{key}'] = v
    inp['np_seed'] = np.int64([c['seed'] + 3])
  elif k == 'gmmil':
    for pre in ('p', 'e'):
      for key, v in _batch(rs, c['B'], c['S'], c['A']).items(): inp[f'{pre}_{key}'] = v
    for key, v in _batch(rs, c['B'], c['S'], c['A']).items(): inp[f'p2_{key}'] = v  # second call (frozen bandwidths)
  elif k == 'pwil':
    inp['expert_states'] = rs.standard_normal((c['N'], c['S'])).astype(np.float32)
    inp['expert_states'][:, -1] = 0  # constant feature -> scale 1 (models.py:207)
    inp['expert_actions'] = np.tanh(rs.standard_normal((c['N'], c['A']))).astype(np.float32)
    inp['states'] = rs.standard_normal((c['steps'], c['S'])).astype(np.float32)
    inp['states'][:, -1] = 0
    inp['actions'] = np.tanh(rs.standard_normal((c['steps'], c['A']))).astype(np.float32)
  elif k == 'replay':
    n = c['appends']
    inp['states'] = rs.standard_normal((n, c['S'])).astype(np.float32)
    inp['states'][:, -1] = 0
    inp['next_states'] = rs.standard_normal((n, c['S'])).astype(np.float32)
    inp['next_states'][:, -1] = 0
    inp['actions'] = rs.standard_normal((n, c['A'])).astype(np.float32)
    inp['rewards'] = rs.standard_normal(n).astype(np.float32)
    inp['event'] = rs.choice(3, size=n, p=[0.85, 0.1, 0.05]).astype(np.int64)  # 0 none, 1 early terminal (+wrap), 2 timeout
  return inp


def _t(x): return torch.from_numpy(np.ascontiguousarray(x))


def _np(x): return x.detach().cpu().numpy().copy() if isinstance(x, torch.Tensor) else np.asarray(x)


# ----------------------------------------------------------------------------------------------------------
# Running the oracle PORT
# ----------------------------------------------------------------------------------------------------------
def _batch_from(inp, prefix) -> Dict[str, torch.Tensor]:
  return {key[len(prefix):]: _t(v) for key, v in inp.items() if key.startswith(prefix) and not key[len(prefix):].startswith('eps')}


def _mask_list(inp, prefix, c):
  """Injected dropout masks of one forward pass in consumption order: input mask (if input_dropout > 0), then one per hidden layer (if dropout > 0)."""
  out = []
  if c['input_dropout'] > 0: out.append(_t(inp[f'{prefix}_in']))
  if c['dropout'] > 0: out += [_t(inp[f'{prefix}_h{l}']) for l in range(c['depth'])]
  return out


@contextlib.contextmanager
def injected_dropout(masks: List[torch.Tensor]):
  """nn.Dropout -> F.dropout consumes the case's pre-scaled masks (in call order) instead of torch's RNG; the reference source is untouched."""
  import torch.nn.functional as Fn
  saved = Fn.dropout
  Fn.dropout = lambda x, p=0.5, training=True, inplace=False: (x * masks.pop(0)) if (training and p > 0) else x
  try:
    yield
  finally:
    Fn.dropout = saved


def run_port(name: str, inp: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
  c = CASES[name]
  k = c['kind']
  out: Dict[str, np.ndarray] = {}
  if k == 'actor':
    actor = [_t(inp[f'actor_{i}']) for i in range(6)]
    s = _t(inp['states'])
    mean, log_std = port.actor_mean_logstd(actor, s)
    a, lp = port.actor_sample(actor, s, _t(inp['eps']))
    out.update(mean=_np(mean), log_std=_np(log_std), action=_np(a), log_prob_sample=_np(lp), greedy=_np(port.actor_greedy_action(actor, s)),
               log_prob_action=_np(port.actor_log_prob(actor, s, _t(inp['actions']))))
  elif k == 'sac':
    agent = port.SacAgent([_t(inp[f'actor_{i}']) for i in range(6)], [[_t(inp[f'critic{t}_{i}']) for i in range(6)] for t in (1, 2)], lr=c['lr'], weight_decay=c['wd'],
                          log_alpha=float(inp['log_alpha'][0]), target=[[_t(inp[f'target{t}_{i}']) for i in range(6)] for t in (1, 2)])
    for s in range(c['steps']):
      r = port.sac_update(agent, _batch_from(inp, f'b{s}_'), _t(inp[f'b{s}_eps_next']), _t(inp[f'b{s}_eps_new']), c['discount'], c['entropy_target'], c['polyak'])
      for key in ('log_probs', 'q_values', 'value_loss', 'policy_loss', 'temperature_loss', 'target_values'): out[f's{s}_{key}'] = _np(r[key])
    for i, p in enumerate(agent.actor): out[f'actor_{i}'] = _np(p)
    for t in (0, 1):
      for i, p in enumerate(agent.twin[t]): out[f'critic{t + 1}_{i}'] = _np(p)
      for i, p in enumerate(agent.target[t]): out[f'target{t + 1}_{i}'] = _np(p)
    out['log_alpha'] = _np(agent.log_alpha)
    for which in ('actor', 'critic', 'alpha'):
      m, v = agent.adam_state(which)
      for i, (mi, vi) in enumerate(zip(m, v)): out[f'adam_{which}_m_{i}'], out[f'adam_{which}_v_{i}'] = _np(mi), _np(vi)
  elif k == 'bc':
    actor = [torch.nn.Parameter(_t(inp[f'actor_{i}']).clone()) for i in range(6)]
    opt = torch.optim.AdamW(actor, lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']): out[f's{s}_loss'] = _np(port.behavioural_cloning_update(actor, opt, _batch_from(inp, f'b{s}_')))
    for i, p in enumerate(actor):
      out[f'actor_{i}'] = _np(p)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p]['exp_avg']), _np(opt.state[p]['exp_avg_sq'])
  elif k == 'gail':
    g = [_t(inp[f'g_{i}']) for i in range(4)]
    sn = [(port._l2_normalise(_t(inp[f'u_{l}'])), port._l2_normalise(_t(inp[f'v_{l}']))) for l in range(2)] if c['spectral_norm'] else None
    disc = port.GailDiscriminator(g, sn, discount=0.97, reward_function=c['reward'])
    opt = torch.optim.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']):
      pol, exp = _batch_from(inp, f'p{s}_'), _batch_from(inp, f'e{s}_')
      r = port.gail_update(disc, opt, pol, exp, _t(inp[f's{s}_eps_gp']), loss_function=c['loss'], grad_penalty=c['grad_penalty'], entropy_bonus=c['entropy_bonus'],
                           eps_mixup=_t(inp[f's{s}_eps_mix']))
      with torch.no_grad():
        out[f's{s}_reward'] = _np(disc.predict_reward(pol['states'], pol['actions']))
        out[f's{s}_logits'] = _np(disc.forward(pol['states'], pol['actions']))
    for i, p in enumerate(disc.g):
      out[f'g_{i}'] = _np(p)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p]['exp_avg']), _np(opt.state[p]['exp_avg_sq'])
    if sn is not None:
      for l, (u, v) in enumerate(disc.g_sn): out[f'u_{l}'], out[f'v_{l}'] = _np(u), _np(v)
  elif k == 'gailx':
    ng, nh = sum(key.startswith('g_') for key in inp), sum(key.startswith('h_') for key in inp)
    g, h = [_t(inp[f'g_{i}']) for i in range(ng)], ([_t(inp[f'h_{i}']) for i in range(nh)] if nh else None)
    sn = lambda net, n: [(port._l2_normalise(_t(inp[f'{net}u_{l}'])), port._l2_normalise(_t(inp[f'{net}v_{l}']))) for l in range(n // 2)] if c['spectral_norm'] else None
    actor = [_t(inp[f'actor_{i}']) for i in range(6)] if c['subtract_log_policy'] else None
    disc = port.GailDiscriminator(g, sn('g', ng), discount=0.97, activation=c['activation'], reward_function=c['reward'], state_only=c['state_only'],
                                  subtract_log_policy=c['subtract_log_policy'], h=h, h_sn=sn('h', nh) if nh else None)
    opt = torch.optim.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']):
      pol, exp = _batch_from(inp, f'p{s}_'), _batch_from(inp, f'e{s}_')
      port.gail_update(disc, opt, pol, exp, _t(inp[f's{s}_eps_gp']), loss_function=c['loss'], grad_penalty=c['grad_penalty'], entropy_bonus=c['entropy_bonus'],
                       pos_class_prior=c.get('pos_class_prior', 0.7), nonnegative_margin=c.get('nonnegative_margin', float('inf')), eps_mixup=_t(inp[f's{s}_eps_mix']), actor=actor)
      with torch.no_grad():
        lp = port.actor_log_prob(actor, pol['states'], pol['actions']) if actor is not None else None
        out[f's{s}_reward'] = _np(disc.predict_reward(pol['states'], pol['actions'], pol['next_states'], pol['terminals'], lp))
        out[f's{s}_logits'] = _np(disc.forward(pol['states'], pol['actions'], pol['next_states'], pol['terminals'], lp))
    for net, params, bufs in (('g', disc.g, disc.g_sn), ('h', disc.h, disc.h_sn)):
      if params is None: continue
      for i, p in enumerate(params):
        out[f'{net}_{i}'] = _np(p)
        out[f'adam_{net}_m_{i}'], out[f'adam_{net}_v_{i}'] = _np(opt.state[p]['exp_avg']), _np(opt.state[p]['exp_avg_sq'])
      if bufs is not None:
        for l, (u, v) in enumerate(bufs): out[f'{net}u_{l}'], out[f'{net}v_{l}'] = _np(u), _np(v)
  elif k == 'red':
    n = 2 * (c['depth'] + 1)
    disc = port.RedDiscriminator([_t(inp[f'predictor_{i}']) for i in range(n)], [_t(inp[f'target_{i}']) for i in range(n)], c['state_only'], c['activation'], c['input_dropout'], c['dropout'])
    opt = torch.optim.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']): out[f's{s}_loss'] = _np(port.target_estimation_update(disc, opt, _batch_from(inp, f'b{s}_'), _mask_list(inp, f'm{s}', c)))
    sb = _batch_from(inp, 'sig_')
    with torch.no_grad():
      disc.set_sigma(sb['states'], sb['actions'], _mask_list(inp, 'msig', c))
      disc.training = False
      pb = _batch_from(inp, 'p_')
      out['reward'] = _np(disc.predict_reward(pb['states'], pb['actions']))
    out['sigma'] = np.float32([disc.sigma_1])
    for i, p_ in enumerate(disc.predictor):
      out[f'predictor_{i}'] = _np(p_)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p_]['exp_avg']), _np(opt.state[p_]['exp_avg_sq'])
  elif k == 'dril':
    n = 2 * (c['depth'] + 1)
    actor = [torch.nn.Parameter(_t(inp[f'actor_{i}']).clone()) for i in range(n)]
    opt = torch.optim.AdamW(actor, lr=c['lr'], weight_decay=c['wd'])
    dk = dict(input_dropout=c['input_dropout'], dropout=c['dropout'])
    for s in range(c['steps']): out[f's{s}_loss'] = _np(port.behavioural_cloning_update(actor, opt, _batch_from(inp, f'b{s}_'), c['activation'], masks=_mask_list(inp, f'm{s}', c), **dk))
    with torch.no_grad():
      es, ea, pb = _t(inp['expert_states']), _t(inp['expert_actions']), _batch_from(inp, 'p_')
      out['expert_variance'] = _np(port.dril_action_uncertainty(actor, es, ea, c['activation'], c['input_dropout'], c['dropout'], _mask_list(inp, 'mthr', c)))
      q = port.dril_uncertainty_threshold(actor, es, ea, c['quantile'], c['activation'], c['input_dropout'], c['dropout'], _mask_list(inp, 'mthr', c))
      out['q'] = np.float32([q])
      out['variance'] = _np(port.dril_action_uncertainty(actor, pb['states'], pb['actions'], c['activation'], c['input_dropout'], c['dropout'], _mask_list(inp, 'mrew', c)))
      out['reward'] = _np(port.dril_predict_reward(actor, q, pb['states'], pb['actions'], c['activation'], c['input_dropout'], c['dropout'], _mask_list(inp, 'mrew', c)))
    for i, p_ in enumerate(actor):
      out[f'actor_{i}'] = _np(p_)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p_]['exp_avg']), _np(opt.state[p_]['exp_avg_sq'])
  elif k == 'ingest':
    raw = {key: _t(inp[key]) for key in ('observations', 'next_observations', 'actions', 'terminals', 'timeouts')}
    tr = port.build_expert_transitions(raw, c['trajectories'], c['subsample'], c['absorbing'], rng=np.random.RandomState(int(inp['np_seed'][0])))
    for key in ('states', 'actions', 'next_states', 'terminals', 'timeouts', 'weights', 'rewards'): out[key] = _np(tr[key])
    out['meta'] = np.int64([tr['num_trajectories'], tr['states'].shape[0]])
  elif k == 'eval':
    env = port.SyntheticEnv(c['env'], True, c['max_steps'])
    rets = port.evaluate_agent([_t(inp[f'actor_{i}']) for i in range(6)], env, c['episodes'], [_t(u) for u in inp['reset_u']])
    out['returns'] = np.float32(rets)
  elif k == 'mix':
    S, A = c['S'], c['A']
    tr = {key: _t(inp[f'e_{key}']) for key in ('states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights')}
    tr['num_trajectories'] = 3
    em = port.Replay(c['Ne'], S, A, True, transitions=tr)
    am = port.Replay(c['size'], S, A, True)
    am.transfer_transitions(em)
    for i in range(c['extra']):
      am.append(100 + i, _t(inp['x_states'][i]), _t(inp['x_actions'][i]), float(inp['x_rewards'][i]), _t(inp['x_next_states'][i]), bool(inp['x_terminals'][i]), False)
    rng = np.random.RandomState(int(inp['np_seed'][0]))
    ia, ie = am.draw_indices(c['B'], rng), em.draw_indices(c['B'], rng)
    ta, te = am.gather(ia), em.gather(ie)
    port.mix_expert_agent_transitions(ta, te)
    out['idx_agent'], out['idx_expert'] = ia, ie
    for key, v in ta.items(): out[f'mixed_{key}'] = _np(v)
    out['meta'] = np.int64([am.idx, int(am.full), am.num_trajectories, em.idx, int(em.full), em.num_trajectories])
  elif k == 'gmmil':
    d = port.GmmilDiscriminator()
    p, e, p2 = _batch_from(inp, 'p_'), _batch_from(inp, 'e_'), _batch_from(inp, 'p2_')
    out['reward_1'] = _np(d.predict_reward(p['states'], p['actions'], e['states'], e['actions'], p['weights'], e['weights']))
    out['gammas'] = np.float32([d.gamma_1, d.gamma_2])
    out['reward_2'] = _np(d.predict_reward(p2['states'], p2['actions'], e['states'], e['actions'], p2['weights'], e['weights']))
  elif k == 'pwil':
    d = port.PwilDiscriminator(_t(inp['expert_states']), _t(inp['expert_actions']), c['T'])
    rewards = []
    for i in range(c['steps']):
      rewards.append(d.compute_reward(_t(inp['states'][i:i + 1]), _t(inp['actions'][i:i + 1])))
      if (i + 1) % c['T'] == 0: d.reset()
    out['rewards'] = np.float32(rewards)
  elif k == 'replay':
    mem = port.Replay(c['size'], c['S'], c['A'], absorbing=True)
    _drive_replay(mem, inp, c)
    np.random.seed(c['seed'])
    t = mem.sample(c['B'])
    for key, v in t.items(): out[f'sample_{key}'] = _np(v)
    for key in port.FIELDS: out[f'mem_{key}'] = _np(mem.data[key])
    out['meta'] = np.int64([mem.idx, int(mem.full), mem.num_trajectories])
  return out


def _drive_replay(mem, inp, c):
  """train.py:157-163 append / wrap schedule driven by the seeded `event` stream."""
  for i in range(c['appends']):
    ev = int(inp['event'][i])
    mem.append(i + 1, _t(inp['states'][i]), _t(inp['actions'][i]), float(inp['rewards'][i]), _t(inp['next_states'][i]), ev == 1, ev == 2)
    if ev == 1: mem.wrap_for_absorbing_states()


# ----------------------------------------------------------------------------------------------------------
# Running the unmodified REFERENCE (container only)
# ----------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def injected_noise(normal_eps: List[torch.Tensor], uniform_eps: List[torch.Tensor], beta_eps: List[torch.Tensor]):
  """Patches torch's samplers so the reference consumes the case's injected draws instead of its RNG:
  Normal.sample/rsample -> loc + scale * eps (models.py:93 users), torch.rand_like (training.py:118),
  Beta.sample (training.py:106). The reference source is untouched."""
  from torch.distributions import Normal, Beta
  saved = (Normal.sample, Normal.rsample, torch.rand_like, Beta.sample)
  def _sample(self, sample_shape=torch.Size()):
    with torch.no_grad(): return self.loc + self.scale * normal_eps.pop(0)
  def _rsample(self, sample_shape=torch.Size()): return self.loc + normal_eps.pop(0) * self.scale
  Normal.sample, Normal.rsample = _sample, _rsample
  torch.rand_like = lambda x, **kw: uniform_eps.pop(0)
  Beta.sample = lambda self, sample_shape=torch.Size(): beta_eps.pop(0)
  try:
    yield
  finally:
    Normal.sample, Normal.rsample, torch.rand_like, Beta.sample = saved


def _load_mlp(seq, weights):
  linears = [m for m in seq if isinstance(m, torch.nn.Linear)]
  with torch.no_grad():
    for l, lin in enumerate(linears):
      lin.weight.copy_(_t(weights[2 * l]))
      lin.bias.copy_(_t(weights[2 * l + 1]))


def run_reference(name: str, inp: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
  from . import refstub
  ref = refstub.load()
  DC = ref.DictConfig
  c = CASES[name]
  k = c['kind']
  out: Dict[str, np.ndarray] = {}
  model_cfg = lambda H: DC(hidden_size=H, depth=2, activation='relu')
  if k == 'actor':
    actor = ref.models.SoftActor(c['S'], c['A'], model_cfg(c['H']))
    _load_mlp(actor.actor, [inp[f'actor_{i}'] for i in range(6)])
    s = _t(inp['states'])
    with torch.no_grad(), injected_noise([_t(inp['eps'])], [], []):
      pol = actor(s)
      a = pol.sample()
      out.update(mean=_np(pol.base_dist.mean), log_std=_np(pol.base_dist.stddev.log()), action=_np(a), log_prob_sample=_np(pol.log_prob(a)),
                 greedy=_np(actor.get_greedy_action(s)), log_prob_action=_np(actor.log_prob(s, _t(inp['actions']))))
  elif k == 'sac':
    S, A, H = c['S'], c['A'], c['H']
    actor, critic = ref.models.SoftActor(S, A, model_cfg(H)), ref.models.TwinCritic(S, A, model_cfg(H))
    _load_mlp(actor.actor, [inp[f'actor_{i}'] for i in range(6)])
    _load_mlp(critic.critic_1.critic, [inp[f'critic1_{i}'] for i in range(6)])
    _load_mlp(critic.critic_2.critic, [inp[f'critic2_{i}'] for i in range(6)])
    target = ref.models.create_target_network(critic)
    _load_mlp(target.critic_1.critic, [inp[f'target1_{i}'] for i in range(6)])
    _load_mlp(target.critic_2.critic, [inp[f'target2_{i}'] for i in range(6)])
    log_alpha = torch.tensor(inp['log_alpha'].copy(), requires_grad=True)
    oa = torch.optim.AdamW(actor.parameters(), lr=c['lr'], weight_decay=c['wd'])
    oc = torch.optim.AdamW(critic.parameters(), lr=c['lr'], weight_decay=c['wd'])
    ot = torch.optim.Adam([log_alpha], lr=c['lr'])
    for s in range(c['steps']):
      batch = _batch_from(inp, f'b{s}_')
      with injected_noise([_t(inp[f'b{s}_eps_next']), _t(inp[f'b{s}_eps_new'])], [], []):
        lp, q = ref.training.sac_update(actor, critic, log_alpha, target, batch, oa, oc, ot, c['discount'], c['entropy_target'], c['polyak'])
      out[f's{s}_log_probs'], out[f's{s}_q_values'] = _np(lp), _np(q)
    for i, p in enumerate(actor.parameters()): out[f'actor_{i}'] = _np(p)
    for t, net in ((1, critic.critic_1), (2, critic.critic_2)):
      for i, p in enumerate(net.parameters()): out[f'critic{t}_{i}'] = _np(p)
    for t, net in ((1, target.critic_1), (2, target.critic_2)):
      for i, p in enumerate(net.parameters()): out[f'target{t}_{i}'] = _np(p)
    out['log_alpha'] = _np(log_alpha)
    for which, opt, params in (('actor', oa, list(actor.parameters())), ('critic', oc, list(critic.parameters())), ('alpha', ot, [log_alpha])):
      for i, p in enumerate(params): out[f'adam_{which}_m_{i}'], out[f'adam_{which}_v_{i}'] = _np(opt.state[p]['exp_avg']), _np(opt.state[p]['exp_avg_sq'])
  elif k == 'bc':
    actor = ref.models.SoftActor(c['S'], c['A'], model_cfg(c['H']))
    _load_mlp(actor.actor, [inp[f'actor_{i}'] for i in range(6)])
    opt = torch.optim.AdamW(actor.parameters(), lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']): ref.training.behavioural_cloning_update(actor, _batch_from(inp, f'b{s}_'), opt)
    for i, p in enumerate(actor.parameters()):
      out[f'actor_{i}'] = _np(p)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p]['exp_avg']), _np(opt.state[p]['exp_avg_sq'])
  elif k == 'gail':
    S, A, H = c['S'], c['A'], c['H']
    icfg = DC(state_only=False, spectral_norm=c['spectral_norm'], loss_function=c['loss'], grad_penalty=c['grad_penalty'], mixup_alpha=1, entropy_bonus=c['entropy_bonus'],
              pos_class_prior=0.7, nonnegative_margin=float('inf'),
              discriminator=DC(hidden_size=H, depth=1, activation='relu', input_dropout=0.5, dropout=0.75, reward_shaping=False, subtract_log_policy=False, reward_function=c['reward']))
    disc = ref.models.GAILDiscriminator(S, A, icfg, 0.97)
    lins = [m for m in disc.g if isinstance(m, torch.nn.Linear)]
    with torch.no_grad():
      for l, lin in enumerate(lins):
        if c['spectral_norm']:
          lin.parametrizations.weight.original.copy_(_t(inp[f'g_{2 * l}']))
          lin.parametrizations.weight[0]._u.copy_(port._l2_normalise(_t(inp[f'u_{l}'])))
          lin.parametrizations.weight[0]._v.copy_(port._l2_normalise(_t(inp[f'v_{l}'])))
        else:
          lin.weight.copy_(_t(inp[f'g_{2 * l}']))
        lin.bias.copy_(_t(inp[f'g_{2 * l + 1}']))
    # parameters() order for parametrized Linear is (bias, original); collect as (weight, bias) per layer
    plist = []
    for lin in lins: plist += [lin.parametrizations.weight.original if c['spectral_norm'] else lin.weight, lin.bias]
    opt = torch.optim.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    disc.eval()
    for s in range(c['steps']):
      pol, exp = _batch_from(inp, f'p{s}_'), _batch_from(inp, f'e{s}_')
      disc.train()
      with injected_noise([], [_t(inp[f's{s}_eps_gp'])], [_t(inp[f's{s}_eps_mix'])]):
        ref.training.adversarial_imitation_update(None, disc, pol, exp, opt, icfg)
      disc.eval()
      with torch.inference_mode():
        out[f's{s}_reward'] = _np(disc.predict_reward(**ref.models.make_gail_input(pol['states'], pol['actions'], pol['next_states'], pol['terminals'], None, False, False)))
        out[f's{s}_logits'] = _np(disc(pol['states'], pol['actions']))
    for i, p in enumerate(plist):
      out[f'g_{i}'] = _np(p)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p]['exp_avg']), _np(opt.state[p]['exp_avg_sq'])
    if c['spectral_norm']:
      for l, lin in enumerate(lins): out[f'u_{l}'], out[f'v_{l}'] = _np(lin.parametrizations.weight[0]._u), _np(lin.parametrizations.weight[0]._v)
  elif k == 'gailx':
    S, A, H = c['S'], c['A'], c['H']
    icfg = DC(state_only=c['state_only'], spectral_norm=c['spectral_norm'], loss_function=c['loss'], grad_penalty=c['grad_penalty'], mixup_alpha=1, entropy_bonus=c['entropy_bonus'],
              pos_class_prior=c.get('pos_class_prior', 0.7), nonnegative_margin=c.get('nonnegative_margin', float('inf')),
              discriminator=DC(hidden_size=H, depth=c['depth'], activation=c['activation'], input_dropout=0.5, dropout=0.75, reward_shaping=c['reward_shaping'],
                               subtract_log_policy=c['subtract_log_policy'], reward_function=c['reward']))
    disc = ref.models.GAILDiscriminator(S, A, icfg, 0.97)
    actor = None
    if c['subtract_log_policy']:
      actor = ref.models.SoftActor(S, A, DC(hidden_size=32, depth=2, activation='relu'))
      _load_mlp(actor.actor, [inp[f'actor_{i}'] for i in range(6)])
    nets, plists = {}, {}
    for net in ('g', 'h'):
      mod = getattr(disc, net, None)
      if mod is None: continue
      lins = [mod] if isinstance(mod, torch.nn.Linear) else [m for m in mod if isinstance(m, torch.nn.Linear)]
      nets[net], plists[net] = lins, []
      with torch.no_grad():
        for l, lin in enumerate(lins):
          if c['spectral_norm']:
            lin.parametrizations.weight.original.copy_(_t(inp[f'{net}_{2 * l}']))
            lin.parametrizations.weight[0]._u.copy_(port._l2_normalise(_t(inp[f'{net}u_{l}'])))
            lin.parametrizations.weight[0]._v.copy_(port._l2_normalise(_t(inp[f'{net}v_{l}'])))
          else:
            lin.weight.copy_(_t(inp[f'{net}_{2 * l}']))
          lin.bias.copy_(_t(inp[f'{net}_{2 * l + 1}']))
          plists[net] += [lin.parametrizations.weight.original if c['spectral_norm'] else lin.weight, lin.bias]
    opt = torch.optim.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    disc.eval()
    for s in range(c['steps']):
      pol, exp = _batch_from(inp, f'p{s}_'), _batch_from(inp, f'e{s}_')
      disc.train()
      with injected_noise([], [_t(inp[f's{s}_eps_gp'])], [_t(inp[f's{s}_eps_mix'])]):
        ref.training.adversarial_imitation_update(actor, disc, pol, exp, opt, icfg)
      disc.eval()
      with torch.inference_mode():
        gi = ref.models.make_gail_input(pol['states'], pol['actions'], pol['next_states'], pol['terminals'], actor, c['reward_shaping'], c['subtract_log_policy'])
        out[f's{s}_reward'] = _np(disc.predict_reward(**gi))
        out[f's{s}_logits'] = _np(disc(**gi))
    for net, plist in plists.items():
      for i, p in enumerate(plist):
        out[f'{net}_{i}'] = _np(p)
        out[f'adam_{net}_m_{i}'], out[f'adam_{net}_v_{i}'] = _np(opt.state[p]['exp_avg']), _np(opt.state[p]['exp_avg_sq'])
      if c['spectral_norm']:
        for l, lin in enumerate(nets[net]): out[f'{net}u_{l}'], out[f'{net}v_{l}'] = _np(lin.parametrizations.weight[0]._u), _np(lin.parametrizations.weight[0]._v)
  elif k == 'red':
    S, A = c['S'], c['A']
    icfg = DC(state_only=c['state_only'], reward_bandwidth_scale=None,
              discriminator=DC(hidden_size=c['H'], depth=c['depth'], activation=c['activation'], input_dropout=c['input_dropout'], dropout=c['dropout']))
    disc = ref.models.REDDiscriminator(S, A, icfg)
    n = 2 * (c['depth'] + 1)
    _load_mlp(disc.predictor.embedding, [inp[f'predictor_{i}'] for i in range(n)])
    _load_mlp(disc.target.embedding, [inp[f'target_{i}'] for i in range(n)])
    opt = torch.optim.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']):
      with injected_dropout(_mask_list(inp, f'm{s}', c)):
        ref.training.target_estimation_update(disc, _batch_from(inp, f'b{s}_'), opt)
    sb, pb = _batch_from(inp, 'sig_'), _batch_from(inp, 'p_')
    with torch.inference_mode(), injected_dropout(_mask_list(inp, 'msig', c)):
      disc.set_sigma(sb['states'], sb['actions'])  # train mode here (train.py:129 runs before :147)
    disc.eval()
    with torch.inference_mode(): out['reward'] = _np(disc.predict_reward(pb['states'], pb['actions']))
    out['sigma'] = np.float32([disc.sigma_1])
    plist = [p_ for m in disc.predictor.embedding if isinstance(m, torch.nn.Linear) for p_ in (m.weight, m.bias)]
    for i, p_ in enumerate(plist):
      out[f'predictor_{i}'] = _np(p_)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p_]['exp_avg']), _np(opt.state[p_]['exp_avg_sq'])
  elif k == 'dril':
    S, A = c['S'], c['A']
    actor = ref.models.SoftActor(S, A, DC(hidden_size=c['H'], depth=c['depth'], activation=c['activation'], input_dropout=c['input_dropout'], dropout=c['dropout']))
    n = 2 * (c['depth'] + 1)
    _load_mlp(actor.actor, [inp[f'actor_{i}'] for i in range(n)])
    opt = torch.optim.AdamW(actor.parameters(), lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']):
      with injected_dropout(_mask_list(inp, f'm{s}', c)):
        ref.training.behavioural_cloning_update(actor, _batch_from(inp, f'b{s}_'), opt)
    es, ea, pb = _t(inp['expert_states']), _t(inp['expert_actions']), _batch_from(inp, 'p_')
    with torch.inference_mode():
      with injected_dropout(_mask_list(inp, 'mthr', c)): out['expert_variance'] = _np(actor._get_action_uncertainty(es, ea))
      with injected_dropout(_mask_list(inp, 'mthr', c)): actor.set_uncertainty_threshold(es, ea, c['quantile'])
      out['q'] = np.float32([actor.q])
      with injected_dropout(_mask_list(inp, 'mrew', c)): out['variance'] = _np(actor._get_action_uncertainty(pb['states'], pb['actions']))
      with injected_dropout(_mask_list(inp, 'mrew', c)): out['reward'] = _np(actor.predict_reward(pb['states'], pb['actions']))
    plist = [p_ for m in actor.actor if isinstance(m, torch.nn.Linear) for p_ in (m.weight, m.bias)]
    for i, p_ in enumerate(plist):
      out[f'actor_{i}'] = _np(p_)
      out[f'adam_m_{i}'], out[f'adam_v_{i}'] = _np(opt.state[p_]['exp_avg']), _np(opt.state[p_]['exp_avg_sq'])
  elif k == 'ingest':
    import types
    D4RLEnv = ref.evaluation.D4RLEnv  # evaluation.py:6 imports it from environments.py (gym / d4rl stubbed)
    # copies: get_dataset rewrites terminal flags through views of the dataset arrays (environments.py:100)
    fake = types.SimpleNamespace(dataset={key: inp[key].copy() for key in ('observations', 'next_observations', 'actions', 'rewards', 'terminals', 'timeouts')}, absorbing=c['absorbing'])
    state = np.random.get_state()
    np.random.seed(int(inp['np_seed'][0]))  # environments.py:113 draws the subsampling offsets from the global numpy stream
    try:
      mem = D4RLEnv.get_dataset(fake, trajectories=c['trajectories'], subsample=c['subsample'])
    finally:
      np.random.set_state(state)
    for key in ('states', 'actions', 'next_states', 'terminals', 'timeouts', 'weights', 'rewards'): out[key] = _np(getattr(mem, key))
    out['meta'] = np.int64([mem.num_trajectories, mem.states.shape[0]])
  elif k == 'eval':
    env = port.SyntheticEnv(c['env'], True, c['max_steps'])
    actor = ref.models.SoftActor(env.state_size, env.act, model_cfg(c['H']))
    _load_mlp(actor.actor, [inp[f'actor_{i}'] for i in range(6)])
    noise = [_t(u) for u in inp['reset_u']]

    class Adapter:  # the D4RLEnv surface evaluate_agent touches (environments.py:29-40): reset() / step(action)
      def reset(self): return env.reset(noise.pop(0))
      def step(self, action): return env.step(action)
    out['returns'] = np.float32(ref.evaluation.evaluate_agent(actor, Adapter(), c['episodes']))
  elif k == 'mix':
    S, A = c['S'], c['A']
    tr = {key: _t(inp[f'e_{key}']) for key in ('states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights')}
    tr['num_trajectories'] = 3
    em = ref.memory.ReplayMemory(c['Ne'], S, A, True, transitions=tr)
    am = ref.memory.ReplayMemory(c['size'], S, A, True)
    am.transfer_transitions(em)
    for i in range(c['extra']):
      am.append(100 + i, _t(inp['x_states'][i]), _t(inp['x_actions'][i]), float(inp['x_rewards'][i]), _t(inp['x_next_states'][i]), bool(inp['x_terminals'][i]), False)
    # record the index stream of memory.py:51-56 while sampling with the global numpy RNG
    drawn = []
    orig = ref.memory.ReplayMemory._sample_idx
    def spy(self):
      i = orig(self)
      drawn.append(i)
      return i
    state = np.random.get_state()
    np.random.seed(int(inp['np_seed'][0]))
    ref.memory.ReplayMemory._sample_idx = spy
    try:
      ta = am.sample(c['B'])
      te = em.sample(c['B'])
    finally:
      ref.memory.ReplayMemory._sample_idx = orig
      np.random.set_state(state)
    ref.models.mix_expert_agent_transitions(ta, te)
    out['idx_agent'], out['idx_expert'] = np.int64(drawn[:c['B']]), np.int64(drawn[c['B']:])
    for key, v in ta.items(): out[f'mixed_{key}'] = _np(v)
    out['meta'] = np.int64([am.idx, int(am.full), am.num_trajectories, em.idx, int(em.full), em.num_trajectories])
  elif k == 'gmmil':
    d = ref.models.GMMILDiscriminator(c['S'], c['A'], DC(state_only=False))
    p, e, p2 = _batch_from(inp, 'p_'), _batch_from(inp, 'e_'), _batch_from(inp, 'p2_')
    out['reward_1'] = _np(d.predict_reward(p['states'], p['actions'], e['states'], e['actions'], p['weights'], e['weights']))
    out['gammas'] = np.float32([d.gamma_1, d.gamma_2])
    out['reward_2'] = _np(d.predict_reward(p2['states'], p2['actions'], e['states'], e['actions'], p2['weights'], e['weights']))
  elif k == 'pwil':
    n = c['N']
    z = torch.zeros
    mem = ref.memory.ReplayMemory(n, c['S'], c['A'], True, transitions=dict(states=_t(inp['expert_states']), actions=_t(inp['expert_actions']), rewards=z(n), next_states=z(n, c['S']),
                                                                            terminals=z(n), timeouts=z(n), weights=torch.ones(n), num_trajectories=1))
    d = ref.models.PWILDiscriminator(c['S'], c['A'], DC(state_only=False, reward_scale=5, reward_bandwidth_scale=5), mem, c['T'])
    rewards = []
    for i in range(c['steps']):
      rewards.append(d.compute_reward(_t(inp['states'][i:i + 1]), _t(inp['actions'][i:i + 1])))
      if (i + 1) % c['T'] == 0: d.reset()
    out['rewards'] = np.float32(rewards)
  elif k == 'replay':
    mem = ref.memory.ReplayMemory(c['size'], c['S'], c['A'], True)
    for key in ('step', 'states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights'): getattr(mem, key).zero_()  # torch.empty -> defined
    _drive_replay(mem, inp, c)
    np.random.seed(c['seed'])
    t = mem.sample(c['B'])
    for key, v in t.items(): out[f'sample_{key}'] = _np(v)
    for key in port.FIELDS: out[f'mem_{key}'] = _np(getattr(mem, key))
    out['meta'] = np.int64([mem.idx, int(mem.full), mem.num_trajectories])
  return out


# ----------------------------------------------------------------------------------------------------------
# Compact storage: full arrays for small outputs, sampled entries + moments for large ones
# ----------------------------------------------------------------------------------------------------------
SAMPLE_THRESHOLD, SAMPLES = 4096, 192


def compress(outputs: Dict[str, np.ndarray]) -> Dict[str, np.ndarray]:
  z = {}
  for key, v in outputs.items():
    v = np.asarray(v)
    if v.size <= SAMPLE_THRESHOLD:
      z[key] = v
    else:
      idx = _rs(v.size).choice(v.size, SAMPLES, replace=False)
      z[key + '@idx'], z[key + '@val'] = idx.astype(np.int64), v.reshape(-1)[idx]
      z[key + '@mom'] = np.float64([v.astype(np.float64).sum(), (v.astype(np.float64) ** 2).sum()])
  return z


def compare(golden: Dict[str, np.ndarray], outputs: Dict[str, np.ndarray], rtol: float, atol: float, keys=None) -> List[str]:
  """Returns a list of mismatch descriptions (empty = parity) of `outputs` against a compressed golden."""
  bad = []
  names = sorted({k.split('@')[0] for k in golden.keys()})
  for key in names:
    if keys is not None and key not in keys: continue
    if key not in outputs:
      bad.append(f'{key}: missing')
      continue
    v = np.asarray(outputs[key])
    if key in golden:
      ref, got = golden[key], v
    else:
      ref, got = golden[key + '@val'], v.reshape(-1)[golden[key + '@idx']]
      mom = np.float64([v.astype(np.float64).sum(), (v.astype(np.float64) ** 2).sum()])
      if not np.allclose(mom, golden[key + '@mom'], rtol=max(rtol, 1e-4) * 10, atol=atol * v.size): bad.append(f'{key}: moments {mom} vs {golden[key + "@mom"]}')
    if ref.shape != got.shape:
      bad.append(f'{key}: shape {got.shape} vs {ref.shape}')
    elif not np.allclose(got, ref, rtol=rtol, atol=atol):
      err = np.abs(got.astype(np.float64) - ref.astype(np.float64))
      bad.append(f'{key}: max abs err {err.max():.3e} (ref scale {np.abs(ref).max():.3e})')
  return bad
