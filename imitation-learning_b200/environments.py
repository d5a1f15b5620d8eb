"""Batched environment adapter with the reference's `D4RLEnv` surface (environments.py:20-125).

gym / d4rl / MuJoCo are not available offline (SURVEY.md §8c), so the physics behind `reset` / `step` is the
deterministic synthetic locomotion-shaped system of SURVEY §8d with the real D4RL shapes, stepped on the device
for all replicas at once (csrc/env.cu). The D4RL-shaped expert dataset is produced by rolling a fixed random
tanh-MLP "expert" in that env; `get_dataset` then applies the reference's trajectory split / absorbing wrap /
subsampling logic (environments.py:63-125) and returns a ReplayMemory shared by all replicas.
"""
from __future__ import annotations

import ctypes as C
import math
from types import SimpleNamespace
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib
from .memory import ReplayMemory

ENVS = ['ant', 'halfcheetah', 'hopper', 'walker2d']  # environments.py:17
ENV_DIMS = {'ant': (111, 8), 'halfcheetah': (17, 6), 'hopper': (11, 3), 'walker2d': (17, 6)}  # D4RL *-expert-v2 observation / action sizes
EARLY_TERMINATION = {'ant': True, 'halfcheetah': False, 'hopper': True, 'walker2d': True}
TERM_THRESHOLD = {'ant': 0.85, 'halfcheetah': 2.0, 'hopper': 0.72, 'walker2d': 0.85}  # |x'_0| above this ends the episode early


def synthetic_env_params(env_name: str) -> Dict[str, Tensor]:
  """Fixed per-environment dynamics / reward parameters (host-side setup, deterministic per env name)."""
  obs, act = ENV_DIMS[env_name]
  g = torch.Generator().manual_seed(1234 + ENVS.index(env_name))
  M = torch.randn(obs, obs, generator=g) * (0.3 / math.sqrt(obs)) + torch.eye(obs) * 0.9
  N = torch.randn(act, obs, generator=g) * (0.3 / math.sqrt(act))
  c = torch.randn(obs, generator=g) * 0.05
  w_r = torch.randn(obs, generator=g) / math.sqrt(obs)
  return dict(M=M, N=N, c=c, w_r=w_r)


def expert_policy_params(env_name: str, absorbing: bool, hidden: int = 64) -> List[Tensor]:
  """Weights of the fixed tanh-MLP expert that synthesises the D4RL-shaped buffer."""
  obs, act = ENV_DIMS[env_name]
  S = obs + (1 if absorbing else 0)
  g = torch.Generator().manual_seed(4321 + ENVS.index(env_name))
  W0 = torch.randn(hidden, S, generator=g) / math.sqrt(S)
  W1 = torch.randn(2 * act, hidden, generator=g) / math.sqrt(hidden)
  return [W0, torch.zeros(hidden), W1, torch.zeros(2 * act)]


class _Box:
  def __init__(self, low: np.ndarray, high: np.ndarray):
    self.low, self.high, self.shape = low, high, low.shape


class EnvBatch:
  """n independent environment instances on the device (physical state x [n, obs], step counters t [n])."""

  def __init__(self, params: Dict[str, Tensor], obs: int, act: int, absorbing: bool, n_envs: int, max_episode_steps: int, early_termination: bool, term_threshold: float,
               device):
    self.p, self.obs, self.act, self.absorbing, self.n = params, obs, act, absorbing, n_envs
    self.S = obs + (1 if absorbing else 0)
    self.max_episode_steps, self.early, self.thr, self.device = max_episode_steps, early_termination, term_threshold, device
    self.x = torch.zeros(n_envs, obs, device=device)
    self.t = torch.zeros(n_envs, dtype=torch.int32, device=device)

  def c_struct(self) -> _lib.Env:
    e = _lib.Env()
    e.M, e.N, e.c, e.w_r = self.p['M'].data_ptr(), self.p['N'].data_ptr(), self.p['c'].data_ptr(), self.p['w_r'].data_ptr()
    e.x, e.t = self.x.data_ptr(), self.t.data_ptr()
    e.obs, e.act, e.absorbing, e.max_episode_steps, e.early_termination, e.term_threshold = self.obs, self.act, int(self.absorbing), self.max_episode_steps, int(self.early), self.thr
    return e

  def reset(self, u: Tensor, state: Tensor, mask: Optional[Tensor] = None, else_state: Optional[Tensor] = None):
    e = self.c_struct()
    _lib.check(_lib.lib().il_env_reset(_lib.handle(), C.byref(e), self.n, u.data_ptr(), _lib.ptr(mask), state.data_ptr(), _lib.ptr(else_state), _lib.stream()))

  def step(self, action: Tensor, next_state: Tensor, reward: Tensor, done: Tensor, timeout: Optional[Tensor] = None, terminal_f: Optional[Tensor] = None,
           timeout_f: Optional[Tensor] = None, frozen: Optional[Tensor] = None):
    e = self.c_struct()
    _lib.check(_lib.lib().il_env_step(_lib.handle(), C.byref(e), self.n, action.data_ptr(), next_state.data_ptr(), reward.data_ptr(), _lib.ptr(done), _lib.ptr(timeout),
                                      _lib.ptr(terminal_f), _lib.ptr(timeout_f), _lib.ptr(frozen), _lib.stream()))


class D4RLEnv:
  """environments.py:20-61 surface. `replicas` environments are stepped together; with replicas == 1 `reset` /
  `step` return the reference's types ([1, S] tensor, float reward, bool terminal)."""

  def __init__(self, env_name: str, absorbing: bool, load_data: bool = False, replicas: int = 1, device=None, max_episode_steps: int = 1000, term_threshold: Optional[float] = None):
    assert env_name in ENVS
    self.env_name, self.absorbing, self.replicas = env_name, absorbing, replicas
    self.device = torch.device('cuda') if device is None else torch.device(device)
    self.obs, self.act = ENV_DIMS[env_name]
    self.params = {k: v.to(self.device).contiguous() for k, v in synthetic_env_params(env_name).items()}
    self._max_episode_steps, self.term_threshold = max_episode_steps, (TERM_THRESHOLD[env_name] if term_threshold is None else term_threshold)
    self.batch = EnvBatch(self.params, self.obs, self.act, absorbing, replicas, max_episode_steps, EARLY_TERMINATION[env_name], self.term_threshold, self.device)
    S = self.obs + (1 if absorbing else 0)
    self._obs_space = _Box(np.concatenate([-np.ones(self.obs), np.zeros(1)]) if absorbing else -np.ones(self.obs), np.ones(S))  # environments.py:27
    self._act_space = _Box(-np.ones(self.act, dtype=np.float32), np.ones(self.act, dtype=np.float32))
    self.env = SimpleNamespace(ref_min_score=0.0, ref_max_score=1000.0, _max_episode_steps=max_episode_steps)  # train.py:58 placeholders (no D4RL reference scores offline)
    self._seed = 0
    self._gen = torch.Generator().manual_seed(0)
    self.load_data = load_data
    # persistent device buffers for the reference-style single-call API
    self._state = torch.zeros(replicas, S, device=self.device)
    self._reward = torch.zeros(replicas, device=self.device)
    self._done = torch.zeros(replicas, dtype=torch.int32, device=self.device)
    self._eval_batches: Dict[int, EnvBatch] = {}

  # ---- reference surface ----
  def seed(self, seed: Union[int, Sequence[int]]) -> List[int]:  # environments.py:42-43
    """One seed, or one per replica (seed sweeps): replica r then draws its reset noise from its own generator, as a single-replica env
    seeded seed[r] does."""
    if isinstance(seed, int):
      self._seed, self._gen = seed, torch.Generator().manual_seed(seed)
      return [seed]
    assert len(seed) == self.replicas, f'{len(seed)} seeds for {self.replicas} replicas'
    self._seed, self._gen = list(seed), [torch.Generator().manual_seed(s) for s in seed]
    return list(seed)

  def reset_noise(self, n: int) -> Tensor:
    """U[0,1) initial-state draws [n, obs] from the env's seeded host generator (the analogue of gym's seeded reset). With per-replica seeds,
    n is replica-major and replica r's n / R rows come from its own generator."""
    if isinstance(self._gen, torch.Generator): return torch.rand(n, self.obs, generator=self._gen).to(self.device)
    assert n % self.replicas == 0
    return torch.cat([torch.rand(n // self.replicas, self.obs, generator=g) for g in self._gen]).to(self.device)

  def reset(self, u: Optional[Tensor] = None) -> Tensor:  # environments.py:29-33
    u = self.reset_noise(self.replicas) if u is None else torch.as_tensor(u, dtype=torch.float32).to(self.device).reshape(self.replicas, self.obs).contiguous()
    self.batch.reset(u, self._state)
    return self._state.clone()

  def step(self, action: Tensor):  # environments.py:35-40
    a = torch.as_tensor(action, dtype=torch.float32).to(self.device).reshape(self.replicas, self.act).contiguous()
    self.batch.step(a, self._state, self._reward, self._done)
    if self.replicas == 1: return self._state.clone(), float(self._reward[0]), bool(self._done[0])
    return self._state.clone(), self._reward.clone(), self._done.clone()

  def render(self): return None

  def close(self): pass

  @property
  def observation_space(self): return self._obs_space

  @property
  def action_space(self): return self._act_space

  @property
  def max_episode_steps(self) -> int: return self._max_episode_steps

  def eval_batch(self, episodes: int) -> EnvBatch:
    """Separate env instances for replicas x episodes parallel evaluation rollouts (train.py:55: eval_env)."""
    if episodes not in self._eval_batches:
      self._eval_batches[episodes] = EnvBatch(self.params, self.obs, self.act, self.absorbing, self.replicas * episodes, self._max_episode_steps, EARLY_TERMINATION[self.env_name],
                                              self.term_threshold, self.device)
    return self._eval_batches[episodes]

  # ---- expert data ----
  def synthesize_raw_dataset(self, episodes: int) -> Dict[str, Tensor]:
    """D4RL-shaped raw arrays (observations / actions / next_observations / rewards / terminals / timeouts) from
    `episodes` rollouts of the fixed expert in this env, generated on the device by the product kernels."""
    from .models import SoftActor
    S = self.obs + (1 if self.absorbing else 0)
    with torch.random.fork_rng():  # keep the global RNG stream untouched (the reference constructs nothing here)
      expert = SoftActor(S, self.act, SimpleNamespace(hidden_size=64, depth=1, activation='tanh', get=lambda k, d=None: d), replicas=1, device=self.device)
    expert.mlp.load_params(0, 0, expert_policy_params(self.env_name, self.absorbing))
    eb = EnvBatch(self.params, self.obs, self.act, self.absorbing, episodes, self._max_episode_steps, EARLY_TERMINATION[self.env_name], self.term_threshold, self.device)
    g = torch.Generator().manual_seed(977 + ENVS.index(self.env_name))
    state = torch.zeros(episodes, S, device=self.device)
    eb.reset(torch.rand(episodes, self.obs, generator=g).to(self.device), state)
    nxt, rew = torch.zeros_like(state), torch.zeros(episodes, device=self.device)
    done, tout = torch.zeros(episodes, dtype=torch.int32, device=self.device), torch.zeros(episodes, dtype=torch.int32, device=self.device)
    frozen = torch.zeros(episodes, dtype=torch.int32, device=self.device)
    rec = []
    for _ in range(self._max_episode_steps):
      action = expert.get_greedy_action(state.unsqueeze(0)).reshape(episodes, self.act).contiguous()
      eb.step(action, nxt, rew, done, timeout=tout, frozen=frozen)
      rec.append((state[:, :self.obs].clone(), action.clone(), nxt[:, :self.obs].clone(), rew.clone(), done.clone(), tout.clone(), frozen.clone()))
      frozen |= done
      state.copy_(nxt)
      if bool(frozen.all()): break
    obs_l, act_l, nobs_l, rew_l, term_l, tout_l = [], [], [], [], [], []
    for e in range(episodes):  # concatenate episode by episode like a D4RL file
      for (s, a, ns, r, d, to, fr) in rec:
        if fr[e]: break
        obs_l.append(s[e]); act_l.append(a[e]); nobs_l.append(ns[e]); rew_l.append(r[e])
        term_l.append(float(bool(d[e]) and not bool(to[e]))); tout_l.append(float(bool(to[e])))
    st = lambda l: torch.stack(l).cpu()
    return dict(observations=st(obs_l), actions=st(act_l), next_observations=st(nobs_l), rewards=st(rew_l), terminals=torch.tensor(term_l), timeouts=torch.tensor(tout_l))

  def get_dataset(self, trajectories: int = 0, subsample: int = 1, raw: Optional[Dict[str, Tensor]] = None, replicas: Optional[int] = None) -> ReplayMemory:
    """environments.py:63-125 on the (synthetic) raw dataset; the result is one read-only memory shared by all replicas."""
    raw = self.synthesize_raw_dataset(max(trajectories, 5)) if raw is None else raw
    tr = build_expert_transitions(raw, trajectories, subsample, self.absorbing)
    S = self.obs + (1 if self.absorbing else 0)
    return ReplayMemory(tr['states'].size(0), S, self.act, self.absorbing, transitions=tr, replicas=self.replicas if replicas is None else replicas, shared=True, device=self.device)


def build_expert_transitions(raw: Dict[str, Tensor], trajectories: int, subsample: int, absorbing: bool) -> Dict[str, Tensor]:
  """The preprocessing of environments.py:63-125: split into trajectories at terminals / timeouts, keep the first
  `trajectories`, append the absorbing bit and (for early terminations) the absorbing-state transition with
  importance weight 1/subsample, then subsample every `subsample`-th step from a random offset (np.random.choice)."""
  f32 = lambda k: torch.as_tensor(raw[k], dtype=torch.float32)
  states, actions, next_states, terminals, timeouts = f32('observations'), f32('actions'), f32('next_observations'), f32('terminals'), f32('timeouts')
  obs_size, action_size = states.size(1), actions.size(1)
  ends = torch.sort(torch.cat([torch.tensor([-1]), terminals.nonzero().flatten(), timeouts.nonzero().flatten()]))[0].tolist()
  episodes = []
  for lo, hi in zip(ends[:-1], ends[1:]):
    sl = slice(lo + 1, hi + 1)
    episodes.append(dict(states=states[sl], actions=actions[sl], next_states=next_states[sl], terminals=terminals[sl].clone(), timeouts=timeouts[sl].clone(),
                         weights=torch.ones(hi - lo)))
  if trajectories > 0: episodes = episodes[:trajectories]
  if absorbing:
    absorbing_state = torch.cat([torch.zeros(1, obs_size), torch.ones(1, 1)], dim=1)
    for ep in episodes:
      n = ep['states'].size(0)
      ep['states'] = torch.cat([ep['states'], torch.zeros(n, 1)], dim=1)
      ep['next_states'] = torch.cat([ep['next_states'], torch.zeros(n, 1)], dim=1)
      if not ep['timeouts'][-1]:  # early termination: rewrite the last transition, add absorbing -> absorbing
        ep['next_states'][-1], ep['terminals'][-1], ep['weights'][-1] = absorbing_state[0], 0, 1 / subsample
        ep['states'] = torch.cat([ep['states'], absorbing_state])
        ep['actions'] = torch.cat([ep['actions'], torch.zeros(1, action_size)])
        ep['next_states'] = torch.cat([ep['next_states'], absorbing_state])
        for k, v in (('terminals', 0.0), ('timeouts', 0.0), ('weights', 1 / subsample)): ep[k] = torch.cat([ep[k], torch.tensor([v])])
  if subsample > 1:
    for ep in episodes:
      start, T = np.random.choice(subsample), ep['states'].size(0)
      keep = set(range(start, T, subsample))
      if absorbing: keep |= {T - 2, T - 1}
      keep = sorted(keep)
      for k in ep: ep[k] = ep[k][keep]
  out = {k: torch.cat([ep[k] for ep in episodes]) for k in ('states', 'actions', 'next_states', 'terminals', 'timeouts', 'weights')}
  out['num_trajectories'] = len(episodes)
  out['rewards'] = torch.zeros_like(out['terminals'])  # environments.py:124: rewards are not leaked to the IL algorithm
  return out
