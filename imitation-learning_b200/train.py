"""The training orchestrator (reference train.py:26-243) for R seed-sharded replicas on one GPU.

`Trainer.rollout()` is train.py:150-168 and `Trainer.update()` is train.py:171-203, each a fixed sequence of C-ABI
calls on one CUDA stream with every piece of per-step state (env state, replay ring indices, optimiser step
counts, RNG counters, the `step` counter) resident on the device — so both sequences are captured once as CUDA
graphs and replayed without host involvement. Replica r is a reference-equivalent run with seed `cfg.seed + r`; with per-replica seeds
(`per_replica={'seed': [...]}`, a seed sweep) replica r draws every random number as the single run with seed[r] does, so it is that run.

`Trainer(per_replica={key: R values})` gives the replicas their own values of the shape-preserving hyper-parameters
(config.PER_REPLICA_KEYS gives each key, the configurations in which it is per replica and the values it accepts); `main` runs a multirun sweep
(`-m key=a,b,...`) as groups of such Trainers, one replica block per job.
"""
from __future__ import annotations

import copy
import ctypes as C
import os
import sys
import time
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch
from torch import Tensor

from . import _lib, checkpoint, distributed
from .config import PER_REPLICA_DROPOUT, Config, SweepError, SweepJob, expand_sweep, get_key, load_config, needs_expert_memory, replica_values, split_per_replica, sweep_groups
from .environments import D4RLEnv, ENVS
from .evaluation import evaluate_agent
from .memory import ReplayMemory, TransitionBatch
from .models import GAILDiscriminator, GMMILDiscriminator, PWILDiscriminator, REDDiscriminator, RewardRelabeller, SoftActor, TwinCritic, _RNG, create_target_network
from .net import ReplicaRNG
from .optim import Adam, AdamW

ACCELERATED = ['AdRIL', 'BC', 'DRIL', 'SAC', 'GAIL', 'GMMIL', 'PWIL', 'RED']


def check_config(cfg: Config):
  """train.py:28-48 (config.split_per_replica checks the per-replica values)."""
  assert cfg.algorithm in ['AdRIL', 'BC', 'DRIL', 'GAIL', 'GMMIL', 'PWIL', 'RED', 'SAC']
  assert cfg.env in ENVS
  cfg.memory.size = min(cfg.steps, cfg.memory.size)
  assert cfg.bc_pretraining.iterations >= 0
  assert cfg.imitation.trajectories >= 0
  assert cfg.imitation.subsample >= 1
  assert cfg.imitation.mix_expert_data in ['none', 'mixed_batch', 'prefill_memory']
  if cfg.algorithm == 'AdRIL':  # train.py:35-37
    assert cfg.imitation.mix_expert_data == 'mixed_batch'
    assert cfg.imitation.update_freq >= 0
  if cfg.algorithm == 'DRIL': assert 0 <= cfg.imitation.quantile_cutoff <= 1  # train.py:38-39
  if cfg.algorithm == 'GAIL':
    assert cfg.imitation.mix_expert_data != 'prefill_memory'
    assert cfg.imitation.discriminator.reward_function in ['AIRL', 'FAIRL', 'GAIL']
    assert cfg.imitation.grad_penalty >= 0
    assert cfg.imitation.entropy_bonus >= 0
    assert cfg.imitation.loss_function in ['BCE', 'Mixup', 'PUGAIL']
    if cfg.imitation.loss_function == 'Mixup': assert cfg.imitation.mixup_alpha > 0
    if cfg.imitation.loss_function == 'PUGAIL': assert 0 <= cfg.imitation.pos_class_prior <= 1 and cfg.imitation.nonnegative_margin >= 0
  assert cfg.logging.interval >= 0
  if cfg.algorithm not in ACCELERATED:
    raise NotImplementedError(f'algorithm={cfg.algorithm} is outside the accelerated hot path (BASELINE.json north_star; SURVEY §8f); supported: {ACCELERATED}')


class Trainer:
  def __init__(self, cfg: Config, replicas: Optional[int] = None, seed_offset: int = 0, fast_init: bool = False, device=None,
               per_replica: Optional[Dict[str, Sequence[float]]] = None):
    """per_replica: dotted config key (config.per_replica_keys) -> R values, replica r training with value r; a key whose values are all equal
    runs as that scalar. None: every replica uses the config's values. Per-replica seeds key every random stream of replica r by seed[r]
    (device Philox draws at replica-local indices, host reset noise, initial weights and pre-training permutations)."""
    R = int(cfg.get('replicas', 1) if replicas is None else replicas)
    self.per_replica: Dict[str, List[float]] = {}
    if per_replica: cfg, self.per_replica = split_per_replica(cfg, per_replica, R)
    seeds = self.seeds = self.per_replica.get('seed')  # None: uniform mode (one program seed, replica r initialised from seed + r)
    if seeds is not None and fast_init: raise SweepError('per-replica seeds need each replica\'s own initial weights; fast_init replicates replica 0\'s')
    check_config(cfg)
    self.cfg = cfg
    self.R = R
    self.device = dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    self.lib, self.h = _lib.lib(), _lib.handle(dev.index)
    _lib.check(self.lib.il_set_gemm_mode(self.h, _lib.GEMM_MODE[cfg.get('gemm_mode', 'fp32')]))
    self.seed = seed = cfg.seed + seed_offset if seeds is None else seeds[0]
    np.random.seed(seed)
    torch.manual_seed(seed)  # train.py:51-52
    self.algorithm = cfg.algorithm
    absorbing = bool(cfg.imitation.absorbing)
    # train.py:55-61
    self.env, self.eval_env = D4RLEnv(cfg.env, absorbing, load_data=True, replicas=R, device=dev), D4RLEnv(cfg.env, absorbing, replicas=R, device=dev)
    self.env.seed(seed if seeds is None else seeds)
    self.eval_env.seed(seed if seeds is None else seeds)
    self.normalization_max, self.normalization_min = self.env.env.ref_max_score, self.env.env.ref_min_score
    self.expert_memory = self.env.get_dataset(trajectories=cfg.imitation.trajectories, subsample=cfg.imitation.subsample) if needs_expert_memory(cfg) else None
    self.S, self.A = S, A = self.env.observation_space.shape[0], self.env.action_space.shape[0]
    # train.py:64-67 — replica r draws its initial weights from the stream of seed + r, or of seeds[r] (fast_init: one stream, replicated).
    # With per-replica seeds the streams go on to draw the pre-training permutations, as the single run's global stream does.
    if seeds is not None: rng = ReplicaRNG(seeds)
    else: rng = None if (R == 1 or fast_init) else ReplicaRNG(seed, R)
    self._init_rng = rng
    nrep = 1 if fast_init else R
    self.actor, self.critic = SoftActor(S, A, cfg.reinforcement.actor, replicas=nrep, rng=rng, device=dev), TwinCritic(S, A, cfg.reinforcement.critic, replicas=nrep, rng=rng, device=dev)
    self.discriminator = None
    pr = self.per_replica
    # per-replica discriminator choices (GAIL sweeps): replica r is initialised with its own spectral-norm flag and width (fast_init: replica 0's
    # draws with spectral norm on when any replica uses it, the flags set after replication; with per-replica widths, each replica draws from
    # replica 0's stream at its own width, so a width class starts where a fast_init run of that width starts)
    rf, sn, hw = pr.get('imitation.discriminator.reward_function'), pr.get('imitation.spectral_norm'), pr.get('imitation.discriminator.hidden_size')
    if self.algorithm == 'GAIL':
      d_rng, d_rep = rng, nrep
      if fast_init and hw is not None: d_rng, d_rep = ReplicaRNG.repeated(torch.get_rng_state(), R), R
      self.discriminator = GAILDiscriminator(S, A, cfg.imitation, cfg.reinforcement.discount, replicas=d_rep, rng=d_rng, device=dev, reward_function=None if fast_init else rf,
                                             spectral_norm=(any(sn) if fast_init else sn) if sn is not None else None, hidden_size=hw)
      if d_rng is not rng: torch.set_rng_state(d_rng.states[0])  # the global stream goes on as after a fast_init run of replica 0's width
    elif self.algorithm in ('DRIL', 'RED'):
      # per-replica activation / dropout rates (RED / DRIL sweeps): replica r is initialised with its own activation's gain (fast_init: every replica
      # redraws from replica 0's stream with its own activation, as for GAIL widths; the rates change no draw)
      drop = {k.rsplit('.', 1)[1]: pr[k] for k in PER_REPLICA_DROPOUT if k in pr}
      d_rng, d_rep = rng, nrep
      if fast_init and drop: d_rng, d_rep = ReplicaRNG.repeated(torch.get_rng_state(), R), R
      if self.algorithm == 'DRIL': self.discriminator = SoftActor(S, A, cfg.imitation.discriminator, replicas=d_rep, rng=d_rng, device=dev, **drop)  # train.py:74
      else: self.discriminator = REDDiscriminator(S, A, cfg.imitation, replicas=d_rep, rng=d_rng, device=dev, **drop)  # train.py:82
      if d_rng is not rng: torch.set_rng_state(d_rng.states[0])
    # the dropout masks are keyed on models.default_rng.seed, which no run sets: single runs of any seed draw the same mask stream, and so do
    # the replicas of a seed sweep, each at its own local indices
    if self.algorithm in ('DRIL', 'RED'): self.discriminator.per_replica_masks = seeds is not None
    if fast_init and R > 1:
      self._replicate()
      if self.algorithm == 'GAIL' and (rf is not None or sn is not None):
        self.discriminator.set_choices(cfg.imitation.discriminator.reward_function if rf is None else rf, cfg.imitation.spectral_norm if sn is None else sn)
    self.log_alpha = torch.zeros(R, device=dev)
    self.target_critic, self.entropy_target = create_target_network(self.critic), cfg.reinforcement.target_temperature * A
    # per-replica values: float64 lists for the optimisers (Python floats in the reference), float32 device tensors for the kernels, each
    # rounded once from the double the scalar path computes
    f32 = lambda vals: torch.tensor(vals, dtype=torch.float32, device=dev)
    if 'reinforcement.target_temperature' in pr: self.entropy_target = f32([float(t) * A for t in pr['reinforcement.target_temperature']])
    self.discount = f32(pr['reinforcement.discount']) if 'reinforcement.discount' in pr else cfg.reinforcement.discount
    self.polyak_factor = f32(pr['reinforcement.polyak_factor']) if 'reinforcement.polyak_factor' in pr else cfg.reinforcement.polyak_factor
    self.imitation_cfg = Config(dict(cfg.imitation, **{k.split('.')[1]: f32(pr[k]) for k in ('imitation.grad_penalty', 'imitation.entropy_bonus', 'imitation.mixup_alpha',
                                                                                             'imitation.pos_class_prior', 'imitation.nonnegative_margin') if k in pr}))
    if 'imitation.loss_function' in pr: self.imitation_cfg.loss_function = list(pr['imitation.loss_function'])  # one name per replica
    self._grad_penalty_on = max(pr.get('imitation.grad_penalty', [cfg.imitation.get('grad_penalty', 0)])) > 0  # GAIL only (GAIL.yaml)
    # the general discriminator's per-replica arrays (il_gailx_update_args), made once before any graph capture: the loss-function codes and the
    # replicas that take the gradient-penalty pass (grad_penalty > 0; the others run as a single run without a penalty)
    self.gail_penalty_pass = None
    if self.algorithm == 'GAIL' and self.discriminator.general:
      from .training import _choice_codes
      if 'imitation.loss_function' in pr: _choice_codes(self.discriminator, 'loss_function', pr['imitation.loss_function'], _lib.LOSS)
      if 'imitation.grad_penalty' in pr: self.gail_penalty_pass = torch.tensor([int(x > 0) for x in pr['imitation.grad_penalty']], dtype=torch.int32, device=dev)
    # the Mixup noise (training.py:106) is drawn for every replica when any replica uses Mixup: U(0, 1) when every alpha is 1, Beta(alpha_r, alpha_r)
    # otherwise (equal to the uniform draw where alpha_r is 1)
    self._mixup_on = self.algorithm == 'GAIL' and 'Mixup' in pr.get('imitation.loss_function', [cfg.imitation.get('loss_function')])
    alphas = pr.get('imitation.mixup_alpha', [float(cfg.imitation.get('mixup_alpha', 1))] * R)
    self.mixup_alpha = None if all(a == 1.0 for a in alphas) else f32(alphas)
    if self.algorithm == 'GAIL' and isinstance(self.discount, Tensor): self.discriminator.discount = self.discount  # reward shaping (models.py:174)
    hp = lambda k: pr.get(k, get_key(cfg, k))
    lr, wd = hp('training.learning_rate'), hp('training.weight_decay')
    self.actor_optimiser, self.critic_optimiser = AdamW(self.actor.parameters(), lr=lr, weight_decay=wd), AdamW(self.critic.parameters(), lr=lr, weight_decay=wd)
    self.temperature_optimiser = Adam([self.log_alpha], lr=lr)
    need = R * int(cfg.memory.size) * _lib.py_row_layout(S, A)[1] * 4
    free = torch.cuda.mem_get_info(dev)[0]
    if need > 0.9 * free:
      raise MemoryError(f'replay rings need {need / 2**30:.1f} GiB ({R} replicas x memory.size {cfg.memory.size} rows x {_lib.py_row_layout(S, A)[1] * 4} B) but only {free / 2**30:.1f} GiB '
                        f'are free on {dev}; lower memory.size (train.py:30 caps it at `steps`) or `replicas`')
    self.memory = ReplayMemory(cfg.memory.size, S, A, absorbing, replicas=R, device=dev)
    self.memory.seed = seed if seeds is None else seeds
    # train.py:70-84
    if self.algorithm in ('DRIL', 'GAIL', 'RED'):
      self.discriminator_optimiser = AdamW(self.discriminator.parameters(), lr=hp('imitation.learning_rate'), weight_decay=hp('imitation.weight_decay'))  # train.py:83-84
    if self.algorithm == 'GAIL':
      self.discriminator.eval()  # train.py:147
    elif self.algorithm == 'AdRIL':
      self.discriminator = RewardRelabeller(hp('imitation.update_freq'), hp('imitation.balanced'), device=dev)  # train.py:72
      self._expert_trajectories = int(self.expert_memory.num_trajectories)  # constant: read once, outside any graph capture
    elif self.algorithm == 'GMMIL':
      self.discriminator = GMMILDiscriminator(S, A, cfg.imitation, replicas=R, device=dev)
    elif self.algorithm == 'PWIL':
      self.discriminator = PWILDiscriminator(S, A, cfg.imitation, self.expert_memory, self.env.max_episode_steps, replicas=R, device=dev,
                                             reward_scale=hp('imitation.reward_scale'), reward_bandwidth_scale=hp('imitation.reward_bandwidth_scale'))
    if self.expert_memory is not None: self.expert_memory.seed = seed + 7919 if seeds is None else [s + 7919 for s in seeds]
    if self.algorithm == 'PWIL' and cfg.imitation.mix_expert_data != 'none': self._pwil_relabel_expert()  # train.py:136-140
    if self.algorithm in ('GMMIL', 'PWIL') and cfg.imitation.mix_expert_data == 'prefill_memory': self.memory.transfer_transitions(self.expert_memory)  # train.py:141,143
    # ---- per-step device state -------------------------------------------------------------------------------
    B = self.B = cfg.training.batch_size
    f = lambda *shape: torch.zeros(*shape, device=dev)
    i32 = lambda *shape: torch.zeros(*shape, dtype=torch.int32, device=dev)
    self.state, self.next_state, self.action = f(R, S), f(R, S), f(R, A)
    self.env_reward, self.store_reward = f(R), f(R)
    self.done, self.timeout, self.terminal_f, self.timeout_f = i32(R), i32(R), f(R), f(R)
    self.step_f = torch.ones(R, device=dev)  # train.py:149: steps count from 1
    self.running_return, self.last_return, self.return_sum, self.episodes = f(R), f(R), f(R), i32(R)
    self.eps_act, self.u_reset = f(R, A), f(R, self.env.obs)
    self.idx_pol, self.idx_exp = i32(R, B), i32(R, B)
    self.u_pol, self.u_exp = f(R, B), f(R, B)  # host-drawn uniforms (device_rng: false)
    row = self.memory.row
    self.batch = TransitionBatch(f(R, B, row), S, A, absorbing)
    self.expert_batch = TransitionBatch(f(R, B, row), S, A, absorbing)
    self.eps_gp, self.eps_mix, self.eps_next, self.eps_new = f(R, B), f(R, B), f(R, B, A), f(R, B, A)
    self.sac_out = dict(log_probs=f(R, B), q_values=f(R, B), losses=f(R, 3))
    self.gail_losses = f(R, 2)
    self.rng = _RNG(seed if seeds is None else seeds, dev)
    self.inject = False  # tests: True = all noise / index buffers are filled by the caller before each step
    self.dril_masks = None  # tests (inject): the dropout masks of this step's DRIL ensemble pass
    self.device_rng = bool(cfg.get('device_rng', True))
    self.actor_ws = torch.empty(self.lib.il_actor_workspace_bytes(C.byref(self.actor.mlp.c_struct()), R, 1), dtype=torch.uint8, device=dev)
    self._sac_args = None
    self.step = 0
    self.updates = 0
    self.graphs: Dict[str, torch.cuda.CUDAGraph] = {}
    self.graph_launches: Dict[str, int] = {}
    self.use_graphs = bool(cfg.get('cuda_graphs', True))
    self.metrics = dict(train_steps=[], train_returns=[], test_steps=[], test_returns=[], test_returns_normalized=[], update_steps=[], predicted_rewards=[], alphas=[],
                        entropies=[], Q_values=[])  # train.py:87
    self.score: List[float] = []
    self.block_scores: List[List[float]] = []  # per output block (_train): the normalised evaluation means so far
    self.active_time = 0.0  # seconds of training before this process resumed the run (check_time_usage)
    self.env.batch.reset(self.env.reset_noise(R), self.state)  # train.py:146

  def _pwil_relabel_expert(self):
    """train.py:136-140: the expert's own transitions get their greedy PWIL reward, walking the expert memory in order and
    restoring the atoms at every episode end. The expert memory is shared by all replicas and every replica would compute the
    same numbers, so one single-replica coupling state does the walk (one-off setup: one small launch per expert transition)."""
    em, d = self.expert_memory, self.discriminator
    one = PWILDiscriminator(self.S, self.A, self.cfg.imitation, em, self.env.max_episode_steps, replicas=1, device=self.device)
    ends = ((em.rows[0, :, em.off['terminals']] != 0) | (em.rows[0, :, em.off['timeouts']] != 0)).cpu().numpy()  # setup-time read of the episode boundaries
    states, actions, rewards = em.rows[0, :, em.off['states']:em.off['states'] + self.S], em.rows[0, :, em.off['actions']:em.off['actions'] + self.A], em.rows[0, :, em.off['rewards']]
    out = torch.empty(1, device=self.device)
    for i in range(em.size):
      one.compute_reward_batch(states[i:i + 1], actions[i:i + 1], out=out)
      rewards[i:i + 1].copy_(out)  # expert_memory.rewards[i] = ...
      if ends[i]: one.reset()
    # the reference walks the expert data with THE discriminator, so whatever atoms the last (unfinished) expert episode consumed
    # stay consumed when training starts: every replica inherits the walk's remaining-weight vector
    d.expert_weights.copy_(one.expert_weights.expand_as(d.expert_weights))

  def _replicate(self):
    """fast_init: every replica starts from replica 0's initial weights (throughput runs; replicas still diverge
    through their own env / noise streams)."""
    for mod in (self.actor, self.critic, self.discriminator):
      if mod is None: continue
      if getattr(mod, 'general', False):  # general GAIL discriminator: one flat [R, g | h] buffer with two net views
        g_total = mod.h_mlp.flat.storage_offset() - mod.flat.storage_offset() if mod.h_mlp is not None else 0
        mod.flat = mod.flat.expand(self.R, -1).contiguous()
        mod.g_mlp.flat, mod.g_mlp.replicas = mod.flat, self.R
        if mod.h_mlp is not None: mod.h_mlp.flat, mod.h_mlp.replicas = mod.flat[:, g_total:], self.R
        mod.replicas = self.R
        for n in ('g_u', 'g_v', 'h_u', 'h_v'):
          if getattr(mod, n, None) is not None: setattr(mod, n, getattr(mod, n).expand(self.R, -1).contiguous())
        continue
      mod.mlp.flat = mod.mlp.flat.expand(self.R, -1).contiguous()
      mod.mlp.replicas = self.R
      mod.replicas = self.R
      if isinstance(mod, REDDiscriminator):  # the frozen target network and the bandwidths as well
        mod.target.flat, mod.target.replicas = mod.target.flat.expand(self.R, -1).contiguous(), self.R
        mod.sigma = mod.sigma.expand(self.R).contiguous()
      if getattr(mod, 'u', None) is not None: mod.u, mod.v = mod.u.expand(self.R, -1).contiguous(), mod.v.expand(self.R, -1).contiguous()

  # ---- train.py:150-168 -------------------------------------------------------------------------------------------
  def rollout(self):
    lib, h, st, R = self.lib, self.h, _lib.stream(), self.R
    if not self.inject: self.rng.normal(None, self.device, stream_id=1, out=self.eps_act)
    m = self.actor.mlp.c_struct()
    _lib.check(lib.il_actor_forward(h, C.byref(m), R, 1, self.state.data_ptr(), self.S, self.S, self.eps_act.data_ptr(), None, self.action.data_ptr(), None, None, None,
                                    self.actor_ws.data_ptr(), self.actor_ws.numel(), st))  # train.py:152
    self.env.batch.step(self.action, self.next_state, self.env_reward, self.done, timeout=self.timeout, terminal_f=self.terminal_f, timeout_f=self.timeout_f)  # train.py:153
    reward = self.env_reward
    if self.algorithm == 'PWIL': reward = self.discriminator.compute_reward_batch(self.state, self.action, out=self.store_reward)  # train.py:156
    mem = self.memory.c_struct()
    _lib.check(lib.il_replay_append(h, C.byref(mem), R, self.step_f.data_ptr(), self.state.data_ptr(), self.action.data_ptr(), reward.data_ptr(), self.next_state.data_ptr(),
                                    self.terminal_f.data_ptr(), self.timeout_f.data_ptr(), None, int(self.memory.absorbing), st))  # train.py:157,162
    _lib.check(lib.il_rollout_bookkeep(h, R, self.env_reward.data_ptr(), self.done.data_ptr(), self.running_return.data_ptr(), self.last_return.data_ptr(),
                                       self.return_sum.data_ptr(), self.episodes.data_ptr(), self.step_f.data_ptr(), st))  # train.py:155,165-166
    if self.algorithm == 'PWIL': self.discriminator.reset(mask=self.done)  # train.py:163
    if not self.inject: self.rng.uniform(None, self.device, stream_id=2, out=self.u_reset)
    self.env.batch.reset(self.u_reset, self.state, mask=self.done, else_state=self.next_state)  # train.py:158,168

  # ---- train.py:171-203 -------------------------------------------------------------------------------------------
  def update(self):
    cfg, B = self.cfg, self.B
    uni = None if self.device_rng else (self.u_pol, self.u_exp)
    if not self.inject: self.memory.sample_indices_device(B, out=self.idx_pol, stream_id=3, uniform=None if uni is None else uni[0])
    self.memory.gather(self.idx_pol, out=self.batch)  # train.py:173
    if self.expert_memory is not None:
      if not self.inject: self.expert_memory.sample_indices_device(B, out=self.idx_exp, stream_id=4, uniform=None if uni is None else uni[1])
      self.expert_memory.gather(self.idx_exp, out=self.expert_batch)
    if self.algorithm == 'GAIL':
      from .training import adversarial_imitation_update
      if self._grad_penalty_on and not self.inject: self.rng.uniform(None, self.device, stream_id=5, out=self.eps_gp)
      eps_mix = None
      if self._mixup_on:  # training.py:106: Beta(a, a) draws; a == 1 (all published configs) is U(0, 1)
        if not self.inject:
          if self.mixup_alpha is None: self.rng.uniform(None, self.device, stream_id=8, out=self.eps_mix)
          else: self.rng.beta(None, self.mixup_alpha, self.device, stream_id=8, out=self.eps_mix)
        eps_mix = self.eps_mix
      self.discriminator.train()  # train.py:178-180
      adversarial_imitation_update(self.actor, self.discriminator, self.batch, self.expert_batch, self.discriminator_optimiser, self.imitation_cfg, eps_gp=self.eps_gp,
                                   eps_mix=eps_mix, out_losses=self.gail_losses, penalty_pass=self.gail_penalty_pass)
      self.discriminator.eval()
    if self.algorithm in ('GAIL', 'GMMIL'):
      if cfg.imitation.mix_expert_data == 'mixed_batch':
        from .models import mix_expert_agent_transitions
        mix_expert_agent_transitions(self.batch, self.expert_batch)  # train.py:183
      if self.algorithm == 'GAIL': self.discriminator.predict_reward_batch(self.batch, write_rewards=True, actor=self.actor)  # train.py:194
      else: self.discriminator.predict_reward_batch(self.batch, self.expert_batch, reward_out=self.batch.rows[..., self.batch.off['rewards']])  # train.py:196
    if self.algorithm in ('DRIL', 'RED'):  # train.py:183,190-191,196-197
      if cfg.imitation.mix_expert_data == 'mixed_batch':
        from .models import mix_expert_agent_transitions
        mix_expert_agent_transitions(self.batch, self.expert_batch)
      view = self.batch.rows[..., self.batch.off['rewards']]
      if self.algorithm == 'DRIL':
        masks = self.dril_masks if self.inject else None
        self.discriminator.predict_reward(self.batch.rows[..., :self.S], self.batch.rows[..., self.S:self.S + self.A], masks=masks, out=view)
      else: self.discriminator.predict_reward_batch(self.batch, reward_out=view)
    if self.algorithm == 'AdRIL':  # train.py:188-189; `step` of the reference = step_f - 1 here (the rollout has already advanced the counter)
      self.discriminator.resample_and_relabel(self.batch, self.expert_batch, self.step_f, self.memory._num_trajectories, self._expert_trajectories, step_offset=-1.0)
    from .training import sac_update
    if cfg.imitation.bc_aux_loss:  # train.py:201
      from .training import behavioural_cloning_update
      behavioural_cloning_update(self.actor, self.expert_batch, self.actor_optimiser)
    if not self.inject:
      self.rng.normal(None, self.device, stream_id=6, out=self.eps_next)
      self.rng.normal(None, self.device, stream_id=7, out=self.eps_new)
    sac_update(self.actor, self.critic, self.log_alpha, self.target_critic, self.batch, self.actor_optimiser, self.critic_optimiser, self.temperature_optimiser,
               self.discount, self.entropy_target, self.polyak_factor, eps_next=self.eps_next, eps_new=self.eps_new, out=self.sac_out)  # train.py:203

  def bc_pretrain(self, iterations: Optional[int] = None) -> Tensor:
    """train.py:93-99: `iterations` behavioural-cloning steps on epoch-wise shuffled expert minibatches (drop_last), with a
    separate AdamW (bc_pretraining.learning_rate / weight_decay). Every replica draws its own permutations (host RNG, like
    the reference's DataLoader; the exact DataLoader stream is not reproduced). Returns the last per-replica loss."""
    from .training import behavioural_cloning_update
    cfg, B, n = self.cfg, self.B, self.expert_memory.size
    iterations = cfg.bc_pretraining.iterations if iterations is None else iterations
    pr = self.per_replica
    opt = AdamW(self.actor.parameters(), lr=pr.get('bc_pretraining.learning_rate', cfg.bc_pretraining.learning_rate),
                weight_decay=pr.get('bc_pretraining.weight_decay', cfg.bc_pretraining.weight_decay))
    loss = torch.zeros(self.R, device=self.device)
    per_epoch = max(n // B, 1)
    perm = None
    for it in range(iterations):
      if it % per_epoch == 0: perm = self._permutations(n)
      j = it % per_epoch
      idx = perm[:, j * B:(j + 1) * B] if n >= B else perm[:, torch.arange(B) % n]
      self.expert_memory.gather(idx.contiguous(), out=self.expert_batch)
      behavioural_cloning_update(self.actor, self.expert_batch, opt, out_loss=loss)
    return loss

  def pretrain_discriminator(self, iterations: Optional[int] = None, batches=None, masks=None, threshold_masks=None):
    """train.py:117-133 for DRIL / RED: `iterations` updates of the dropout policy ensemble (behavioural cloning) / the RED predictor (regression onto its random
    target) on epoch-wise shuffled expert minibatches (every replica draws its own permutations; `batches` injects the index rows instead), then the uncertainty
    threshold (all expert transitions) / the kernel bandwidth (first minibatch) is fixed, and the expert data optionally pre-fills the replay memory."""
    from .training import behavioural_cloning_update, target_estimation_update
    cfg, B, n, d = self.cfg, self.B, self.expert_memory.size, self.discriminator
    iterations = cfg.imitation.pretraining.iterations if iterations is None else iterations
    per_epoch, perm = max(n // B, 1), None
    for it in range(iterations):
      if batches is not None: idx = torch.as_tensor(batches[it], dtype=torch.int32).to(self.device).reshape(-1, B)
      else:
        if it % per_epoch == 0: perm = self._permutations(n)
        j = it % per_epoch
        idx = perm[:, j * B:(j + 1) * B] if n >= B else perm[:, torch.arange(B) % n]
      self.expert_memory.gather(idx.contiguous(), out=self.expert_batch)
      m = None if masks is None else masks[it]
      if self.algorithm == 'DRIL': behavioural_cloning_update(d, self.expert_batch, self.discriminator_optimiser, masks=m)
      else: target_estimation_update(d, self.expert_batch, self.discriminator_optimiser, masks=m)
    em = self.expert_memory
    if self.algorithm == 'DRIL':
      cutoff = self.per_replica.get('imitation.quantile_cutoff', cfg.imitation.quantile_cutoff)
      d.set_uncertainty_threshold(em.rows[0, :, :self.S], em.rows[0, :, self.S:self.S + self.A], cutoff, masks=threshold_masks)  # train.py:127
    else:
      first = torch.arange(B, dtype=torch.int32, device=self.device).unsqueeze(0).expand(self.R, -1).contiguous() % n
      self.expert_memory.gather(first, out=self.expert_batch)
      d.set_sigma_batch(self.expert_batch, masks=threshold_masks)  # train.py:129: estimated on one minibatch
      d.eval()  # train.py:147
    if cfg.imitation.mix_expert_data == 'prefill_memory': self.memory.transfer_transitions(self.expert_memory)  # train.py:133
    self._pretrained = True

  def _permutations(self, n: int) -> Tensor:
    """[R, n] epoch permutations of the expert rows: from the global torch stream in replica order, or with per-replica seeds from each
    replica's own stream (the draws its single run makes)."""
    if self.seeds is None: perms = [torch.randperm(n) for _ in range(self.R)]
    else:
      perms = []
      for r in range(self.R):
        with self._init_rng.replica(r): perms.append(torch.randperm(n))
    return torch.stack(perms).to(self.device, torch.int32)

  def _will_update(self, step: int) -> bool:
    return step >= self.cfg.training.start and step % self.cfg.training.interval == 0  # train.py:171

  def _run(self, name: str, fn):
    """Eager for the first calls (lazy allocations, GMMIL bandwidths), then captured as a CUDA graph and replayed."""
    if not self.use_graphs:
      fn()
      return
    g = self.graphs.get(name)
    if g is None:
      n = self.graph_launches.get(name + '#eager', 0)
      if n < 2:
        fn()
        self.graph_launches[name + '#eager'] = n + 1
        return
      torch.cuda.synchronize()
      before = _lib.launch_count()
      g = torch.cuda.CUDAGraph()
      with torch.cuda.graph(g):
        fn()
      self.graph_launches[name] = _lib.launch_count() - before  # kernels recorded into the graph (capture does not execute)
      self.graphs[name] = g
    g.replay()
    self.replayed_launches = getattr(self, 'replayed_launches', 0) + self.graph_launches[name]

  def train_step(self, host_uniform: bool = False):
    """One iteration of the loop at train.py:149: rollout, then (after `training.start`) one update."""
    self.step += 1
    if self._will_update(self.step):
      if not self.device_rng:  # host-drawn index uniforms (the reference draws its indices on the host: memory.py:54)
        self._host_stream()
        slot = self.step & 1
        if self._pin_ev[slot] is not None: self._pin_ev[slot].synchronize()  # the H2D copy that last used this buffer is done
        self._host_rng.random(out=self._pin[slot].numpy(), dtype=np.float32)
        self.u_pol.copy_(self._pin[slot][0], non_blocking=True)
        self.u_exp.copy_(self._pin[slot][1], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._pin_ev[slot] = ev
      self._run('step+update', lambda: (self.rollout(), self.update()))
      self.updates += 1
    else:
      self._run('step', self.rollout)

  def _host_stream(self):
    """device_rng=false: the host stream of the index uniforms and its double-buffered pinned staging, made at the first update."""
    if getattr(self, '_pin', None) is None:
      self._pin = [torch.empty(2, self.R, self.B, pin_memory=True) for _ in range(2)]  # double-buffered pinned staging
      self._pin_ev = [None, None]
      self._host_rng = np.random.default_rng(self.seed)  # per-rank stream: seed + first replica of this shard

  def total_launches(self) -> int:
    """Kernels launched by this library for this process (eager launches + kernels replayed through CUDA graphs)."""
    captured = sum(v for k, v in self.graph_launches.items() if not k.endswith('#eager'))
    return _lib.launch_count() - captured + getattr(self, 'replayed_launches', 0)

  def evaluate(self) -> Tensor:
    """train.py:213-219 for all replicas; returns [R, episodes]."""
    r = evaluate_agent(self.actor, self.eval_env, self.cfg.evaluation.episodes)
    return torch.as_tensor(r, device=self.device).reshape(self.R, -1) if self.R == 1 else r

  def log_aux(self):
    """train.py:205-210."""
    m = self.metrics
    m['update_steps'].append(self.step)
    m['predicted_rewards'].append(self.batch['rewards'].cpu().numpy())
    m['alphas'].append(self.log_alpha.exp().cpu().numpy())
    m['entropies'].append((-self.sac_out['log_probs']).cpu().numpy())
    m['Q_values'].append(self.sac_out['q_values'].cpu().numpy())

  def state_dicts(self) -> Dict[str, Dict[str, Tensor]]:
    """train.py:237: agent.pth contents."""
    return dict(actor=self.actor.state_dict(), critic=self.critic.state_dict(), log_alpha=self.log_alpha.detach().clone().cpu())

  # ---- checkpoints (checkpoint.py) --------------------------------------------------------------------------------------------
  # The discriminator's state per algorithm (dotted attribute paths; an attribute that is None or not yet made is left out)
  _DISCRIMINATOR_STATE = {'GMMIL': ('gamma', ), 'PWIL': ('expert_weights', ), 'RED': ('predictor.flat', 'target.flat', 'sigma', '_rng.counter'),
                          'DRIL': ('mlp.flat', '_q', '_drop_rng.counter'), 'AdRIL': ('_flag', ), 'SAC': (), 'BC': ()}

  def _discriminator_state(self) -> Sequence[str]:
    if self.algorithm != 'GAIL': return self._DISCRIMINATOR_STATE[self.algorithm]
    return ('flat', 'g_u', 'g_v', 'h_u', 'h_v') if self.discriminator.general else ('mlp.flat', 'u', 'v')

  def _state_tensors(self) -> Dict[str, Tensor]:
    """Every device tensor a later loop iteration reads, by name: the live tensors that checkpoint_state copies and load_checkpoint_state
    overwrites in place. Everything else on the device is set up by the constructor or rewritten before it is read (tests/test_gpu_resume.py
    walks the Trainer to keep it so)."""
    t = dict(actor=self.actor.mlp.flat, critic=self.critic.mlp.flat, target_critic=self.target_critic.mlp.flat, log_alpha=self.log_alpha)
    for name in ('actor_optimiser', 'critic_optimiser', 'temperature_optimiser', 'discriminator_optimiser'):
      o = getattr(self, name, None)
      if o is not None: t.update({f'{name}.exp_avg': o.exp_avg, f'{name}.exp_avg_sq': o.exp_avg_sq, f'{name}.step_count': o.step_count})
    for n in ('rows', '_idx', '_full', '_num_trajectories', '_rng_counter'): t[f'memory.{n}'] = getattr(self.memory, n)
    if self.expert_memory is not None: t['expert_memory._rng_counter'] = self.expert_memory._rng_counter
    for n in ('state', 'next_state', 'step_f', 'running_return', 'last_return', 'return_sum', 'episodes'): t[n] = getattr(self, n)
    t['env.x'], t['env.t'] = self.env.batch.x, self.env.batch.t  # the training envs' physical state and step counters
    if self.rng.counter is not None: t['rng.counter'] = self.rng.counter
    for n in self._discriminator_state():
      v = _attr(self.discriminator, n)
      if v is not None: t[f'discriminator.{n}'] = v
    return t

  def _expert_digest(self) -> Optional[str]:
    if self.expert_memory is None: return None
    if getattr(self, '_expert_sha', None) is None:
      from .checkpoint import expert_digest
      self._expert_sha = expert_digest(self.expert_memory.rows)
    return self._expert_sha

  def checkpoint_state(self) -> Dict[str, object]:
    """Host copies of all state a later loop iteration reads (the filled rows of each replay ring only), the host random streams and the
    loop bookkeeping. load_checkpoint_state(checkpoint_state()) on a freshly constructed Trainer of the same configuration continues the run
    bit for bit."""
    m = self.memory
    filled = m.size if bool(m._full.any()) else int(m._idx.max())
    tensors = {k: (v[:, :filled] if k == 'memory.rows' else v).detach().to('cpu', copy=True).contiguous() for k, v in self._state_tensors().items()}
    d = self.discriminator
    host = dict(step=self.step, updates=self.updates, metrics=copy.deepcopy(self.metrics), scores=copy.deepcopy(self.block_scores), active_time=float(self.active_time),
                env_gen=_gen_state(self.env._gen), eval_env_gen=_gen_state(self.eval_env._gen),
                host_rng=None if getattr(self, '_host_rng', None) is None else self._host_rng.bit_generator.state,
                torch_rng=torch.get_rng_state(), numpy_rng=np.random.get_state(), discriminator_training=getattr(d, 'training', None), sigma_set=getattr(d, '_sigma_set', None))
    return dict(replicas=self.R, algorithm=self.algorithm, expert_digest=self._expert_digest(), tensors=tensors, host=host)

  def load_checkpoint_state(self, state: Dict[str, object]):
    """Restores checkpoint_state() into this freshly constructed Trainer, in place (copy_ into the existing tensors, whose pointers the C
    structs, the evaluation cache and captured graphs hold), before its first step. A checkpoint of another algorithm, replica count or
    expert memory is refused."""
    from .checkpoint import CheckpointError
    if self.step != 0 or self.graphs: raise CheckpointError('load a checkpoint into a fresh Trainer, before its first step')
    if state['algorithm'] != self.algorithm or state['replicas'] != self.R:
      raise CheckpointError(f'checkpoint of {state["algorithm"]} x {state["replicas"]} replica(s); this run is {self.algorithm} x {self.R}')
    if state['expert_digest'] != self._expert_digest(): raise CheckpointError('the expert memory differs from the one the checkpoint was trained on')
    saved, d, dev = state['tensors'], self.discriminator, self.device
    # state made lazily by the first draws / updates of a run: made here, before any graph capture
    if 'rng.counter' in saved: self.rng._ctr(dev)
    if 'discriminator._rng.counter' in saved or 'discriminator._drop_rng.counter' in saved: d.mask_source()._ctr(dev)
    if 'discriminator.gamma' in saved and d.gamma is None: d.gamma = torch.empty(saved['discriminator.gamma'].shape, device=dev)
    if 'discriminator._q' in saved and getattr(d, '_q', None) is None: d._q = torch.empty(saved['discriminator._q'].shape, device=dev)
    live = self._state_tensors()
    if set(live) != set(saved): raise CheckpointError(f'checkpoint state {sorted(set(saved) ^ set(live))} does not match this run\'s')
    for k, v in live.items():
      src = saved[k]
      if k == 'memory.rows':  # the filled part of each ring; the rest is as a fresh ring
        if src.shape[0] != v.shape[0] or src.shape[1] > v.shape[1] or src.shape[2] != v.shape[2]: raise CheckpointError(f'{k}: {tuple(src.shape)} does not fit {tuple(v.shape)}')
        v[:, :src.shape[1]].copy_(src)
        v[:, src.shape[1]:].zero_()
        continue
      if src.shape != v.shape or src.dtype != v.dtype: raise CheckpointError(f'{k}: {src.dtype} {tuple(src.shape)} does not match {v.dtype} {tuple(v.shape)}')
      v.copy_(src)
    h = state['host']
    if self.algorithm == 'DRIL': d.q = float(d._q[0]) if self.R == 1 else d._q
    if h['discriminator_training'] is not None: d.training = h['discriminator_training']
    if h['sigma_set'] is not None: d._sigma_set = h['sigma_set']
    self.step, self.updates, self.metrics, self.block_scores, self.active_time = h['step'], h['updates'], h['metrics'], h['scores'], h['active_time']
    _set_gen_state(self.env._gen, h['env_gen'])
    _set_gen_state(self.eval_env._gen, h['eval_env_gen'])
    if h['host_rng'] is not None:
      self._host_stream()
      self._host_rng.bit_generator.state = h['host_rng']
    torch.set_rng_state(h['torch_rng'])
    np.random.set_state(h['numpy_rng'])


def _attr(obj, dotted: str):
  for p in dotted.split('.'):
    obj = getattr(obj, p, None)
    if obj is None: return None
  return obj


def _gen_state(gen):
  return gen.get_state() if isinstance(gen, torch.Generator) else [g.get_state() for g in gen]


def _set_gen_state(gen, state):
  if isinstance(gen, torch.Generator): gen.set_state(state)
  else:
    for g, s in zip(gen, state): g.set_state(s)


def _block(x, lo: int, hi: int, total: int):
  """Replicas [lo, hi) of an output that a single-replica run writes without its replica axis (the reference's shapes)."""
  if total == 1 or lo is None: return x
  if isinstance(x, dict): return {k: _block(v, lo, hi, total) for k, v in x.items()}
  return x[lo] if hi - lo == 1 else x[lo:hi]


def train(cfg: Config, file_prefix: str = '', overrides: Sequence[str] = ()) -> float:
  """train.py:26-243 (accelerated algorithms). Multi-GPU: launched one process per GPU (torch.distributed.run); the
  replica axis is split across ranks and evaluation returns are reduced over NCCL (distributed.py). With checkpoint.interval, the run
  checkpoints into <file_prefix's directory>/checkpoint (`overrides`, the command line, is recorded there)."""
  ckpt_dir = os.path.join(os.path.dirname(file_prefix) or '.', 'checkpoint') if checkpoint.interval_of(cfg) else None
  return _train(cfg, [(file_prefix, '', None, None)], checkpoint_dir=ckpt_dir, overrides=overrides)[0]


def _train(cfg: Config, blocks, per_replica: Optional[Dict[str, Sequence[float]]] = None, checkpoint_dir: Optional[str] = None, overrides: Sequence[str] = (),
           resume: bool = False, stop_at: Optional[int] = None) -> Optional[List[float]]:
  """The loop of train(). `blocks`: (file prefix, console label, lo, hi) per output set; lo = None is the whole run (and its shards
  across ranks), otherwise replicas [lo, hi) of a single-rank run — one job of a sweep, written and scored as its own run.

  checkpoint_dir: where the checkpoints of checkpoint.interval go (checkpoint.py), each taken after its step's logging and evaluation;
  resume: continue from the latest of them, skipping the pre-training phases its state already holds. stop_at (tests): return None right
  after the checkpoint of that step, writing no output."""
  interval = checkpoint.interval_of(cfg)
  if interval and checkpoint_dir is None: raise checkpoint.CheckpointError('checkpoint.interval needs a checkpoint directory')
  rank, world = distributed.init('nccl')
  total = int(cfg.get('replicas', 1))
  lo, hi = distributed.shard(total, rank, world)
  trainer = Trainer(cfg, replicas=hi - lo, seed_offset=lo, per_replica=per_replica)
  trainer.block_scores = [[] for _ in blocks]
  first = 1
  if resume:
    _, state = checkpoint.load(checkpoint_dir, rank, world)
    trainer.load_checkpoint_state(state)
    first = trainer.step + 1
    if rank == 0: print(f'resuming at step {first} from {checkpoint.latest(checkpoint_dir)}', flush=True)
  metrics, scores = trainer.metrics, trainer.block_scores
  cut = lambda x, b: _block(x, b[2], b[3], total)
  part = lambda x, b: x if b[2] is None else x[b[2]:b[3]]  # outputs that keep the replica axis at one replica
  flat_of = lambda b: (total if b[2] is None else b[3] - b[2]) == 1  # the reference's schema for a single replica (train.py:214-219)
  stats_of = lambda returns, b: distributed.return_statistics(returns if b[2] is None else returns[b[2]:b[3]])
  start_time = time.time() - trainer.active_time
  if cfg.algorithm == 'BC' and interval and rank == 0: print('checkpoint.interval: algorithm=BC trains before the loop, which takes checkpoints; none is written', flush=True)
  if not resume and cfg.bc_pretraining.iterations > 0:  # train.py:93-112
    trainer.bc_pretrain()
    if cfg.algorithm == 'BC':
      returns = trainer.evaluate()
      normalized = (returns.cpu().numpy() - trainer.normalization_min) / (trainer.normalization_max - trainer.normalization_min)
      out = []
      for b in blocks:
        mean, std, n = stats_of(returns, b)
        r_b, n_b, flat = cut(returns.cpu().numpy(), b), cut(normalized, b), flat_of(b)
        m = dict(metrics, test_steps=[0], test_returns=[r_b.reshape(-1).tolist() if flat else r_b.tolist()], test_returns_normalized=[n_b.reshape(-1).tolist() if flat else n_b.tolist()])
        if rank == 0:
          print(f'{b[1]}BC: test return {mean:.3f} +- {std:.3f} over {n} episodes', flush=True)
          torch.save(dict(actor=cut(trainer.actor.state_dict(), b)), f'{b[0]}agent.pth')  # train.py:108
          torch.save(m, f'{b[0]}metrics.pth')
        out.append(float(np.mean(n_b)))
      return out
  if not resume and cfg.algorithm in ('DRIL', 'RED'): trainer.pretrain_discriminator()  # train.py:117-133
  meta = dict(config=cfg, overrides=list(overrides), replicas=total, per_replica=per_replica or {})
  for step in range(first, cfg.steps + 1):
    trainer.train_step()
    if cfg.logging.interval > 0 and step % cfg.logging.interval == 0 and trainer._will_update(step): trainer.log_aux()  # train.py:205: only inside the update branch
    if step % cfg.evaluation.interval == 0 and not cfg.check_time_usage:  # train.py:213
      returns = trainer.evaluate()
      normalized = (returns.cpu().numpy() - trainer.normalization_min) / (trainer.normalization_max - trainer.normalization_min)
      metrics['test_steps'].append(step)
      for i, b in enumerate(blocks):
        mean, std, n = stats_of(returns, b)
        scores[i].append(float((mean - trainer.normalization_min) / (trainer.normalization_max - trainer.normalization_min)))
        r_b, n_b, flat = cut(returns.cpu().numpy(), b), cut(normalized, b), flat_of(b)
        metrics.setdefault('_blocks', [dict(test_returns=[], test_returns_normalized=[]) for _ in blocks])
        metrics['_blocks'][i]['test_returns'].append(r_b.reshape(-1).tolist() if flat else r_b.tolist())
        metrics['_blocks'][i]['test_returns_normalized'].append(n_b.reshape(-1).tolist() if flat else n_b.tolist())
        if rank == 0: print(f'{b[1]}step {step}: test return {mean:.3f} +- {std:.3f} over {n} episodes ({world} rank(s))', flush=True)
    if interval and step % interval == 0:
      trainer.active_time = time.time() - start_time
      checkpoint.save(checkpoint_dir, step, trainer.checkpoint_state(), meta, rank, world, barrier=distributed.barrier)
    if stop_at == step: return None
  trainer.score = scores[0]
  if cfg.check_time_usage: metrics['training_time'] = time.time() - start_time  # train.py:229-230
  eps = trainer.episodes.cpu().numpy()
  metrics['train_returns'] = trainer.return_sum.cpu().numpy() / np.maximum(eps, 1)
  trajectories = None
  if cfg.save_trajectories:  # train.py:232-235: trajectories of the trained agent (every rank writes its own shard of the replica axis; rank 0 keeps the reference's file name)
    if cfg.render: raise NotImplementedError('render=true needs a PyBullet window (environments.py:52-53); the synthetic device env has none')
    _, trajectories = evaluate_agent(trainer.actor, trainer.eval_env, cfg.evaluation.episodes, return_trajectories=True)
  per_block = metrics.pop('_blocks', [dict(test_returns=[], test_returns_normalized=[]) for _ in blocks])
  for i, b in enumerate(blocks):
    m = {k: ([cut(x, b) for x in v] if k == 'predicted_rewards' else [part(x, b) for x in v] if k in ('alphas', 'entropies', 'Q_values') else v) for k, v in metrics.items()}
    m.update(per_block[i], train_returns=part(metrics['train_returns'], b).tolist())
    if trajectories is not None: torch.save(cut(trajectories, b), f'{b[0]}trajectories.pth' if rank == 0 else f'{b[0]}trajectories.rank{rank}.pth')
    if rank == 0:  # train.py:237-239
      sd = trainer.state_dicts()
      torch.save(dict(actor=cut(sd['actor'], b), critic=cut(sd['critic'], b), log_alpha=part(sd['log_alpha'], b)), f'{b[0]}agent.pth')
      if cfg.algorithm in ('DRIL', 'GAIL', 'RED'):  # train.py:238; a job of a spectral-norm / width sweep writes the layout of its own flag and width
        d, kw = trainer.discriminator, {}
        if b[2] is not None and getattr(d, 'spectral_norm_r', None) is not None: kw['spectral_norm'] = d.spectral_norm_r[b[2]]
        if b[2] is not None and getattr(d, 'hidden_size_r', None) is not None: kw['hidden_size'] = d.hidden_size_r[b[2]]
        sd = d.state_dict(**kw)
        torch.save(cut(sd, b), f'{b[0]}discriminator.pth')
      torch.save(m, f'{b[0]}metrics.pth')
  return [float(np.mean(sc)) if sc else float('nan') for sc in scores]


def run_sweep(jobs: List[SweepJob], argv: Optional[Sequence[str]] = None, resume_dir: Optional[str] = None) -> List[float]:
  """A multirun on one GPU: the jobs are partitioned into groups (config.sweep_groups); a group of J jobs is exactly the run
  `train.py <group overrides> replicas=J*R` with job j's vectorised values given to replica block [jR, (j+1)R) — so replica jR+k starts
  like a run with seed `seed + jR + k`. A swept seed s_j is per replica instead: replica jR+k is the single run with seed s_j + k, so with
  replicas=1 job j is `train.py <its overrides>` bit for bit. Groups run one after another. Job j writes the single-run files of its replicas, plus
  overrides.yaml, to <output_dir>/<ALG>_<ENV>_sweeper/<timestamp>/<j>/ (hydra.sweep.dir). Returns the per-job scores.

  With checkpoint.interval the sweep directory also holds multirun.yaml (`argv`), checkpoint/group<k>/ (the running group's checkpoint)
  and checkpoint/scores.json (the scores of the finished groups). resume_dir: continue that sweep (checkpoint.sweep_plan): finished groups
  are skipped, the interrupted one continues from its checkpoint, the rest run."""
  import yaml
  if int(os.environ.get('WORLD_SIZE', '1')) > 1: raise NotImplementedError('a multirun sweep runs on one GPU; sweeps across ranks are not supported')
  groups = sweep_groups(jobs)
  cfgs = [load_config(g.overrides) for g in groups]
  ckpt_on = any(checkpoint.interval_of(c) for c in cfgs)
  cfg0 = load_config(jobs[0].overrides)
  base = resume_dir or os.path.join(cfg0.get('output_dir', './outputs'), f'{cfg0.algorithm}_{cfg0.env}_sweeper', time.strftime('%m-%d_%H-%M-%S'))
  root = os.path.join(base, 'checkpoint')
  plan = checkpoint.sweep_plan(base, [[j.num for j in g.jobs] for g in groups]) if resume_dir else ['run'] * len(groups)
  if ckpt_on and not resume_dir:
    os.makedirs(base, exist_ok=True)
    with open(os.path.join(base, 'multirun.yaml'), 'w') as f: yaml.safe_dump(list(argv or []), f)
  print(f'sweep: {len(jobs)} job(s) in {len(groups)} group(s)', flush=True)
  done = {int(k): v for k, v in checkpoint.read_scores(root).items()} if resume_dir else {}
  scores: Dict[int, float] = {}
  try:
    for k, (g, cfg) in enumerate(zip(groups, cfgs)):
      if plan[k] == 'skip':
        for j in g.jobs: scores[j.num] = done[j.num]
        print(f'group of jobs {[j.num for j in g.jobs]}: finished before the resume', flush=True)
        continue
      R, J = int(cfg.get('replicas', 1)), len(g.jobs)
      cfg.replicas = J * R
      per_replica = {k: replica_values(k, vals, R) for k, vals in g.per_job.items()}
      blocks = []
      for i, j in enumerate(g.jobs):
        d = os.path.join(base, str(j.num))
        os.makedirs(d, exist_ok=True)
        with open(os.path.join(d, 'overrides.yaml'), 'w') as f: yaml.safe_dump(j.overrides, f)
        blocks.append((d + os.sep, f'job {j.num}: ', i * R, (i + 1) * R))
      print(f'group of jobs {[j.num for j in g.jobs]}: {J} x {R} replica(s), per-replica {sorted(per_replica) or "none"}', flush=True)
      gdir = os.path.join(root, f'group{k}') if checkpoint.interval_of(cfg) else None
      for j, s in zip(g.jobs, _train(cfg, blocks, per_replica, checkpoint_dir=gdir, overrides=g.overrides, resume=plan[k] == 'continue')): scores[j.num] = s
      if ckpt_on:
        checkpoint.write_scores(root, {str(n): s for n, s in scores.items()})
        checkpoint.remove(gdir)
  finally:
    distributed.shutdown()
  for j in jobs: print(f'job {j.num}: {" ".join(j.overrides)}: score {scores[j.num]:.4f}', flush=True)
  return [scores[j.num] for j in jobs]


def resume(target: str, others: Sequence[str] = ()):
  """`train.py resume=<dir>`: continues the run or multirun in <dir> from its checkpoint, writing into the same directory. The configuration
  comes from the checkpoint (a run's meta.json, a multirun's multirun.yaml); any other override, a missing checkpoint, another world size or
  library version, or a file whose checksum does not match is refused."""
  import yaml
  if others: raise checkpoint.CheckpointError(f'resume= takes no other override (the configuration comes from the checkpoint); got {" ".join(others)}')
  if os.path.isfile(os.path.join(target, 'multirun.yaml')):
    with open(os.path.join(target, 'multirun.yaml')) as f: argv = yaml.safe_load(f)
    _, jobs = expand_sweep(argv)
    return run_sweep(jobs, argv, resume_dir=target)
  meta = checkpoint.resume_run_meta(target, others, int(os.environ.get('WORLD_SIZE', '1')))
  try:
    return _train(Config(meta['config']), [(target.rstrip(os.sep) + os.sep, '', None, None)], checkpoint_dir=os.path.join(target, 'checkpoint'), overrides=meta['overrides'],
                  resume=True)[0]
  finally:
    distributed.shutdown()


def main(argv: Optional[List[str]] = None):
  """`python train.py algorithm=<ALG> env=<ENV> [key=value ...]` (train.py:21-23, 246): returns the score. With `-m` / `--multirun` and
  comma-separated values (`reinforcement.discount=0.97,0.98,0.99`): Hydra's basic sweep, run by run_sweep; returns the per-job scores.
  `python train.py resume=<dir>`: continues a checkpointed run or multirun (resume)."""
  argv = list(sys.argv[1:] if argv is None else argv)
  target = [a for a in argv if a.startswith('resume=')]
  if target:
    try:
      return resume(target[0].partition('=')[2], [a for a in argv if a != target[0]])
    except checkpoint.CheckpointError as e:
      raise SystemExit(f'resume refused: {e}')
  multirun, jobs = expand_sweep(argv)
  if multirun: return run_sweep(jobs, argv)
  cfg = load_config(jobs[0].overrides)
  checkpoint.interval_of(cfg)
  out_dir = os.path.join(cfg.get('output_dir', './outputs'), f'{cfg.algorithm}_{cfg.env}', time.strftime('%m-%d_%H-%M-%S'))  # conf/train_config.yaml:54-60
  os.makedirs(out_dir, exist_ok=True)
  try:
    return train(cfg, file_prefix=out_dir + os.sep, overrides=jobs[0].overrides)
  finally:
    distributed.shutdown()
