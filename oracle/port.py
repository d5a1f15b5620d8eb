"""TEST INFRASTRUCTURE ONLY — CPU restatement (torch CPU, fp32) of the reference hot path.

This file is the *oracle port*: a from-scratch restatement of the algorithms on the path named by
BASELINE.json `north_star` (SURVEY.md §8a), written functionally over explicit weight tensors with all
randomness *injected* (noise, indices) so the CUDA path can be compared on identical inputs. It is pinned
against the unmodified reference (imported from /root/reference by `oracle/refstub.py`) by
`tests/test_oracle_vs_reference.py` and against the committed fixtures in `tests/golden/` (generated from the
reference by `oracle/make_golden.py`). PARITY IS PINNED (not "unpinned"): see DESIGN.md §Oracle.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference` leg may import it.
The product package (`imitation-learning_b200/`) never imports anything from `oracle/`.

torch autograd / torch.optim / numpy are third-party runtime shared with the reference (SURVEY.md §8c (i)).
Every function cites the reference file:line it follows (paths relative to /root/reference).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch
from torch import Tensor
from torch.nn import functional as F

LOG_STD_MIN, LOG_STD_MAX = -20.0, 2.0  # models.py:87


# ----------------------------------------------------------------------------------------------------------
# MLPs (models.py:48-69): Linear -> act -> ... -> Linear ; parameters kept as [W0, b0, W1, b1, ...]
# ----------------------------------------------------------------------------------------------------------
def _act(x: Tensor, activation: str) -> Tensor:
  if activation == 'relu': return torch.relu(x)
  if activation == 'tanh': return torch.tanh(x)
  if activation == 'sigmoid': return torch.sigmoid(x)
  raise ValueError(activation)


def mlp_forward(params: Sequence[Tensor], x: Tensor, activation: str = 'relu', input_dropout: float = 0.0, dropout: float = 0.0, training: bool = False,
                masks: Optional[List[Tensor]] = None) -> Tensor:
  """models.py:48-69 (`_create_fcnn` as an nn.Sequential): [Dropout(input_dropout)], then per hidden layer Linear -> [Dropout(dropout)] -> activation,
  then the linear head. Train-mode dropout draws its masks with torch's own F.dropout (the reference's RNG consumption); `masks` (a list consumed
  front to back of pre-scaled {0, 1/(1-p)} tensors) injects them instead — used for the CUDA parity cases."""
  n_layers = len(params) // 2
  active = training or masks is not None
  def drop(t, p):
    if p <= 0 or not active: return t
    return t * masks.pop(0) if masks is not None else F.dropout(t, p, True)
  x = drop(x, input_dropout)
  for l in range(n_layers):
    x = F.linear(x, params[2 * l], params[2 * l + 1])
    if l < n_layers - 1: x = _act(drop(x, dropout), activation)
  return x


def init_mlp(sizes: Sequence[int], activation: str = 'relu', final_gain: float = 1.0) -> List[Tensor]:
  """models.py:52-66 initialisation: nn.Linear construction (consumes RNG) then orthogonal_/zero bias."""
  params = []
  for l in range(len(sizes) - 1):
    layer = torch.nn.Linear(sizes[l], sizes[l + 1])
    gain = torch.nn.init.calculate_gain(activation) if l < len(sizes) - 2 else final_gain
    torch.nn.init.orthogonal_(layer.weight, gain=gain)
    torch.nn.init.constant_(layer.bias, 0)
    params += [layer.weight.detach().clone(), layer.bias.detach().clone()]
  return params


# ----------------------------------------------------------------------------------------------------------
# Soft actor (models.py:84-102) and the tanh-Gaussian policy (torch TransformedDistribution semantics)
# ----------------------------------------------------------------------------------------------------------
def actor_mean_logstd(actor: Sequence[Tensor], state: Tensor, activation: str = 'relu', **drop) -> Tuple[Tensor, Tensor]:
  """models.py:90-92: chunk the head into mean / log-std, clamp log-std to [-20, 2]. `drop`: the dropout arguments of mlp_forward (DRIL, models.py:88)."""
  mean, log_std = mlp_forward(actor, state, activation, **drop).chunk(2, dim=1)
  return mean, torch.clamp(log_std, min=LOG_STD_MIN, max=LOG_STD_MAX)


def gaussian_pre_tanh(mean: Tensor, log_std: Tensor, eps: Tensor) -> Tensor:
  """Normal.sample / .rsample with injected standard-normal `eps`: x = mean + std * eps (models.py:93)."""
  return mean + log_std.exp() * eps


def tanh_gaussian_logprob_from_pre_tanh(mean: Tensor, log_std: Tensor, x: Tensor) -> Tensor:
  """log pi(tanh(x)) as torch computes it for TransformedDistribution(Independent(Normal), TanhTransform)
  when the inverse is served from the transform cache (training.py:22,36; SURVEY §2.1 K2)."""
  std = log_std.exp()
  var = std ** 2
  normal_lp = -((x - mean) ** 2) / (2 * var) - std.log() - math.log(math.sqrt(2 * math.pi))
  ladj = 2.0 * (math.log(2.0) - x - F.softplus(-2.0 * x))
  return (0.0 - ladj.sum(dim=-1)) + normal_lp.sum(dim=-1)


def actor_log_prob(actor: Sequence[Tensor], state: Tensor, action: Tensor, activation: str = 'relu', **drop) -> Tensor:
  """models.py:97-99: clamp the action into (-1, 1), invert tanh (atanh), evaluate the density."""
  action = action.clamp(-1 + 1e-6, 1 - 1e-6)
  mean, log_std = actor_mean_logstd(actor, state, activation, **drop)
  return tanh_gaussian_logprob_from_pre_tanh(mean, log_std, torch.atanh(action))


def actor_greedy_action(actor: Sequence[Tensor], state: Tensor, activation: str = 'relu') -> Tensor:
  """models.py:101-102."""
  return torch.tanh(actor_mean_logstd(actor, state, activation)[0])


def actor_sample(actor: Sequence[Tensor], state: Tensor, eps: Tensor, activation: str = 'relu') -> Tuple[Tensor, Tensor]:
  """train.py:152 / training.py:20-22: sample an action (and its log-prob via the cached pre-tanh value)."""
  mean, log_std = actor_mean_logstd(actor, state, activation)
  x = gaussian_pre_tanh(mean, log_std, eps)
  return torch.tanh(x), tanh_gaussian_logprob_from_pre_tanh(mean, log_std, x)


# ----------------------------------------------------------------------------------------------------------
# Twin critic (models.py:123-141)
# ----------------------------------------------------------------------------------------------------------
def critic_forward(critic: Sequence[Tensor], state: Tensor, action: Tensor, activation: str = 'relu') -> Tensor:
  """models.py:128-130 with `_join_state_action` (models.py:20-21)."""
  return mlp_forward(critic, torch.cat([state, action], dim=1), activation).squeeze(dim=1)


def twin_critic_forward(twin: Sequence[Sequence[Tensor]], state: Tensor, action: Tensor, activation: str = 'relu') -> Tuple[Tensor, Tensor]:
  """models.py:139-141."""
  return critic_forward(twin[0], state, action, activation), critic_forward(twin[1], state, action, activation)


# ----------------------------------------------------------------------------------------------------------
# SAC agent state + update (training.py:14-54, train.py:64-66)
# ----------------------------------------------------------------------------------------------------------
class SacAgent:
  """One reference-equivalent agent: actor, twin critic, target critic, log_alpha and the three optimisers
  (train.py:64-66: AdamW(actor), AdamW(critic), Adam([log_alpha]))."""

  def __init__(self, actor: Sequence[Tensor], twin: Sequence[Sequence[Tensor]], lr: float = 3e-4, weight_decay: float = 0.0,
               log_alpha: float = 0.0, activation: str = 'relu', target: Optional[Sequence[Sequence[Tensor]]] = None):
    self.activation = activation
    self.actor = [torch.nn.Parameter(p.detach().clone().float()) for p in actor]
    self.twin = [[torch.nn.Parameter(p.detach().clone().float()) for p in c] for c in twin]
    src = twin if target is None else target
    self.target = [[p.detach().clone().float() for p in c] for c in src]  # models.py:72-76
    self.log_alpha = torch.nn.Parameter(torch.full((1, ), float(log_alpha)))
    self.opt_actor = torch.optim.AdamW(self.actor, lr=lr, weight_decay=weight_decay)
    self.opt_critic = torch.optim.AdamW([p for c in self.twin for p in c], lr=lr, weight_decay=weight_decay)
    self.opt_alpha = torch.optim.Adam([self.log_alpha], lr=lr)

  def adam_state(self, which: str) -> Tuple[List[Tensor], List[Tensor]]:
    opt, params = {'actor': (self.opt_actor, self.actor), 'critic': (self.opt_critic, [p for c in self.twin for p in c]), 'alpha': (self.opt_alpha, [self.log_alpha])}[which]
    return [opt.state[p]['exp_avg'] for p in params], [opt.state[p]['exp_avg_sq'] for p in params]


def sac_update(agent: SacAgent, batch: Dict[str, Tensor], eps_next: Tensor, eps_new: Tensor, discount: float, entropy_target: float,
               polyak_factor: float) -> Dict[str, Tensor]:
  """training.py:14-54 with the two policy noise draws injected (`eps_next` for :21, `eps_new` for :35)."""
  states, actions, rewards, next_states = batch['states'], batch['actions'], batch['rewards'], batch['next_states']
  terminals, weights, absorbing = batch['terminals'], batch['weights'], batch['absorbing']
  act = agent.activation
  alpha = agent.log_alpha.exp()  # :16
  with torch.no_grad():  # :19-25
    next_actions, next_log_probs = actor_sample(agent.actor, next_states, eps_next, act)
    next_actions = (1 - absorbing.unsqueeze(dim=1)) * next_actions
    target_values = torch.min(*twin_critic_forward(agent.target, next_states, next_actions, act)) - (1 - absorbing) * alpha * next_log_probs
    target_values = rewards + (1 - terminals) * discount * target_values
  values_1, values_2 = twin_critic_forward(agent.twin, states, actions, act)  # :26
  value_loss = (weights * (values_1 - target_values).pow(2)).mean() + (weights * (values_2 - target_values).pow(2)).mean()  # :27
  agent.opt_critic.zero_grad(set_to_none=True)
  value_loss.backward()
  agent.opt_critic.step()  # :29-31

  mean, log_std = actor_mean_logstd(agent.actor, states, act)  # :34
  x = gaussian_pre_tanh(mean, log_std, eps_new)  # :35
  new_actions = torch.tanh(x)
  new_log_probs = tanh_gaussian_logprob_from_pre_tanh(mean, log_std, x)  # :36
  new_values = torch.min(*twin_critic_forward(agent.twin, states, new_actions, act))  # :37 (updated critic)
  policy_loss = (weights * (1 - absorbing) * alpha.detach() * new_log_probs - new_values).mean()  # :38
  agent.opt_actor.zero_grad(set_to_none=True)
  policy_loss.backward()
  agent.opt_actor.step()  # :40-42

  temperature_loss = -(weights * (1 - absorbing) * alpha * (new_log_probs.detach() + entropy_target)).mean()  # :45
  agent.opt_alpha.zero_grad(set_to_none=True)
  temperature_loss.backward()
  agent.opt_alpha.step()  # :47-49

  with torch.no_grad():  # :52, models.py:79-81
    for c, t in zip(agent.twin, agent.target):
      for p, tp in zip(c, t):
        tp.mul_(polyak_factor).add_((1 - polyak_factor) * p.data)
  return dict(log_probs=new_log_probs.detach(), q_values=torch.min(values_1, values_2).detach(), value_loss=value_loss.detach(),
              policy_loss=policy_loss.detach(), temperature_loss=temperature_loss.detach(), target_values=target_values)


def behavioural_cloning_update(actor_params: Sequence[torch.nn.Parameter], optimiser, expert: Dict[str, Tensor], activation: str = 'relu', **drop) -> Tensor:
  """training.py:57-64 (`drop`: dropout arguments when the "actor" is DRIL's dropout policy ensemble, train.py:120)."""
  expert_action = expert['actions'].clamp(min=-1 + 1e-6, max=1 - 1e-6)
  optimiser.zero_grad(set_to_none=True)
  loss = (expert['weights'] * -actor_log_prob(actor_params, expert['states'], expert_action, activation, **drop)).mean()
  loss.backward()
  optimiser.step()
  return loss.detach()


# ----------------------------------------------------------------------------------------------------------
# Spectral norm (torch parametrizations.spectral_norm; sites models.py:58,66,159) — SURVEY §8a a12
# ----------------------------------------------------------------------------------------------------------
def _l2_normalise(x: Tensor, eps: float = 1e-12) -> Tensor:
  return x / x.norm().clamp_min(eps)


def spectral_norm_init(weight: Tensor) -> Tuple[Tensor, Tensor]:
  """_SpectralNorm.__init__: draw u, v ~ N(0,1) (global RNG), normalise, run 15 power iterations."""
  h, w = weight.shape
  u = _l2_normalise(torch.empty(h).normal_(0, 1))
  v = _l2_normalise(torch.empty(w).normal_(0, 1))
  for _ in range(15):
    u = _l2_normalise(torch.mv(weight, v))
    v = _l2_normalise(torch.mv(weight.t(), u))
  return u, v


def spectral_norm_weight(weight: Tensor, u: Tensor, v: Tensor, training: bool) -> Tensor:
  """_SpectralNorm.forward: (train mode) one in-place power iteration, then W / (u^T W v) with u, v constants."""
  if training:
    with torch.no_grad():
      u.copy_(_l2_normalise(torch.mv(weight.detach(), v)))
      v.copy_(_l2_normalise(torch.mv(weight.detach().t(), u)))
  sigma = torch.vdot(u.clone(), torch.mv(weight, v.clone()))
  return weight / sigma


# ----------------------------------------------------------------------------------------------------------
# GAIL discriminator (models.py:152-180) and its update (training.py:85-134)
# ----------------------------------------------------------------------------------------------------------
class GailDiscriminator:
  """`g` network of models.py:162 (no reward shaping: GAIL.yaml:16) or g (linear) + h (MLP) with shaping
  (models.py:157-160). Parameters are the `original` weights; `sn` holds the (u, v) buffers per layer."""

  def __init__(self, g: Sequence[Tensor], g_sn: Optional[Sequence[Tuple[Tensor, Tensor]]], discount: float, activation: str = 'relu',
               reward_function: str = 'AIRL', state_only: bool = False, subtract_log_policy: bool = False,
               h: Optional[Sequence[Tensor]] = None, h_sn: Optional[Sequence[Tuple[Tensor, Tensor]]] = None):
    self.g = [torch.nn.Parameter(p.detach().clone().float()) for p in g]
    self.g_sn = None if g_sn is None else [(u.detach().clone(), v.detach().clone()) for u, v in g_sn]
    self.h = None if h is None else [torch.nn.Parameter(p.detach().clone().float()) for p in h]
    self.h_sn = None if h_sn is None else [(u.detach().clone(), v.detach().clone()) for u, v in h_sn]
    self.discount, self.activation, self.reward_function = discount, activation, reward_function
    self.state_only, self.subtract_log_policy = state_only, subtract_log_policy
    self.training = False  # train.py:147 puts the discriminator in eval mode outside the update

  @property
  def reward_shaping(self) -> bool:
    return self.h is not None

  def parameters(self) -> List[torch.nn.Parameter]:
    return list(self.g) + (list(self.h) if self.h is not None else [])

  def _net(self, params, sn, x: Tensor) -> Tensor:
    eff = []
    for l in range(len(params) // 2):
      W = params[2 * l] if sn is None else spectral_norm_weight(params[2 * l], sn[l][0], sn[l][1], self.training)
      eff += [W, params[2 * l + 1]]
    return mlp_forward(eff, x, self.activation).squeeze(dim=1)

  def forward(self, state: Tensor, action: Tensor, next_state: Optional[Tensor] = None, terminal: Optional[Tensor] = None, log_policy: Optional[Tensor] = None) -> Tensor:
    """models.py:164-175."""
    x = state if self.state_only else torch.cat([state, action], dim=1)
    f = self._net(self.g, self.g_sn, x)
    if self.reward_shaping:  # models.py:174; evaluation order: g(s,a), h(s'), h(s)
      f = f + (1 - terminal) * (self.discount * self._net(self.h, self.h_sn, next_state) - self._net(self.h, self.h_sn, state))
    return f - log_policy if self.subtract_log_policy else f

  def predict_reward(self, state: Tensor, action: Tensor, next_state=None, terminal=None, log_policy=None) -> Tensor:
    """models.py:177-180."""
    D = torch.sigmoid(self.forward(state, action, next_state, terminal, log_policy))
    h = -torch.log1p(-D + 1e-6) if self.reward_function == 'GAIL' else torch.log(D + 1e-6) - torch.log1p(-D + 1e-6)
    return torch.exp(h) * -h if self.reward_function == 'FAIRL' else h


def _mix(x_1: Tensor, x_2: Tensor, eps: Tensor) -> Tensor:
  """training.py:79-81."""
  mix = eps.unsqueeze(dim=1) if x_1.ndim == 2 else eps
  return mix * x_1 + (1 - mix) * x_2


def gail_update(disc: GailDiscriminator, optimiser, policy: Dict[str, Tensor], expert: Dict[str, Tensor], eps_gp: Optional[Tensor],
                loss_function: str = 'BCE', grad_penalty: float = 1.0, entropy_bonus: float = 0.0, pos_class_prior: float = 0.7,
                nonnegative_margin: float = float('inf'), eps_mixup: Optional[Tensor] = None, actor=None, actor_activation: str = 'relu') -> Dict[str, Tensor]:
  """training.py:85-134 with the U(0,1) gradient-penalty draw (:118) and the Beta mixup draw (:106) injected."""
  def gail_input(s, a, ns, t):  # models.py:145-149
    inp = dict(state=s, action=a)
    if disc.reward_shaping: inp.update(next_state=ns, terminal=t)
    if disc.subtract_log_policy:
      with torch.no_grad(): inp.update(log_policy=actor_log_prob(actor, s, a, actor_activation))
    return inp

  es, ea, ens, et, ew = expert['states'], expert['actions'], expert['next_states'], expert['terminals'], expert['weights']
  s, a, ns, t, w = policy['states'], policy['actions'], policy['next_states'], policy['terminals'], policy['weights']
  out = {}
  disc.training = True  # train.py:178
  optimiser.zero_grad(set_to_none=True)  # :92
  if loss_function in ('BCE', 'PUGAIL'):
    D_policy, D_expert = disc.forward(**gail_input(s, a, ns, t)), disc.forward(**gail_input(es, ea, ens, et))  # :95
    if loss_function == 'BCE':  # :98-99
      expert_loss = F.binary_cross_entropy_with_logits(D_expert, torch.ones_like(D_expert), weight=ew)
      policy_loss = F.binary_cross_entropy_with_logits(D_policy, torch.zeros_like(D_policy), weight=w)
    else:  # :101-102
      expert_loss = pos_class_prior * F.binary_cross_entropy_with_logits(D_expert, torch.ones_like(D_expert), weight=ew)
      policy_loss = torch.clamp(pos_class_prior * F.binary_cross_entropy_with_logits(D_expert, torch.zeros_like(D_expert), weight=ew)
                                - F.binary_cross_entropy_with_logits(D_policy, torch.zeros_like(D_policy), weight=w), min=-nonnegative_margin)
    (expert_loss + policy_loss).backward(retain_graph=True)  # :103
    out['bce_loss'] = (expert_loss + policy_loss).detach()
    entropy_Ds, entropy_ws = [D_expert, D_policy], [ew, w]
  elif loss_function == 'Mixup':  # :105-114
    eps = eps_mixup
    ms, ma, mns, mt, mw = _mix(es, s, eps), _mix(ea, a, eps), _mix(ens, ns, eps), _mix(et, t, eps), _mix(ew, w, eps)
    D_mix = disc.forward(**gail_input(ms, ma, mns, mt))
    mix_loss = eps * F.binary_cross_entropy_with_logits(D_mix, torch.ones_like(D_mix), weight=mw, reduction='none') \
        + (1 - eps) * F.binary_cross_entropy_with_logits(D_mix, torch.zeros_like(D_mix), weight=mw, reduction='none')
    mix_loss.mean(dim=0).backward(retain_graph=True)
    out['bce_loss'] = mix_loss.mean(dim=0).detach()
    entropy_Ds, entropy_ws = [D_mix], [mw]
  else:
    raise ValueError(loss_function)
  if grad_penalty > 0:  # :117-127
    eps = eps_gp
    ms, ma, mns, mt, mw = _mix(es, s, eps), _mix(ea, a, eps), _mix(ens, ns, eps), _mix(et, t, eps), _mix(ew, w, eps)
    ms.requires_grad_()
    ma.requires_grad_()
    D_mix = disc.forward(**gail_input(ms, ma, mns, mt))
    grads = torch.autograd.grad(D_mix, (ms, ma), torch.ones_like(D_mix), create_graph=True)
    gp_loss = grad_penalty * mw * sum([g.norm(2, dim=1) ** 2 for g in grads])
    gp_loss.mean(dim=0).backward()
    out['gp_loss'] = gp_loss.mean(dim=0).detach()
  if entropy_bonus > 0:  # :130-132 ; H(Bernoulli(logits=l)) = softplus(l) - l * sigmoid(l)
    ent = sum([w_ * torch.distributions.Bernoulli(logits=l).entropy() for l, w_ in zip(entropy_Ds, entropy_ws)])
    (-entropy_bonus * ent.mean()).backward()
  optimiser.step()  # :134
  disc.training = False  # train.py:180
  return out


# ----------------------------------------------------------------------------------------------------------
# DRIL (models.py:104-120): the "discriminator" is a dropout policy trained by behavioural cloning; reward = agreement of a 5-member MC-dropout ensemble
# ----------------------------------------------------------------------------------------------------------
DRIL_ENSEMBLE = 5  # models.py:105


def dril_action_uncertainty(policy: Sequence[Tensor], state: Tensor, action: Tensor, activation: str, input_dropout: float, dropout: float, masks: Optional[List[Tensor]] = None) -> Tensor:
  """models.py:104-107: variance over the ensemble of pi(a|s) under independent dropout masks (always train mode: train.py:147 leaves DRIL's policy in train())."""
  state, action = torch.repeat_interleave(state, DRIL_ENSEMBLE, dim=0), torch.repeat_interleave(action, DRIL_ENSEMBLE, dim=0)
  prob = actor_log_prob(policy, state, action, activation, input_dropout=input_dropout, dropout=dropout, training=True, masks=masks).exp()
  return prob.view(-1, DRIL_ENSEMBLE).var(dim=1)


def dril_uncertainty_threshold(policy, expert_state, expert_action, quantile_cutoff: float, activation: str, input_dropout: float, dropout: float, masks=None) -> float:
  """models.py:110-111."""
  return torch.quantile(dril_action_uncertainty(policy, expert_state, expert_action, activation, input_dropout, dropout, masks), quantile_cutoff).item()


def dril_predict_reward(policy, q: float, state, action, activation: str, input_dropout: float, dropout: float, masks=None) -> Tensor:
  """models.py:113-120: +1 where the ensemble variance is at most the threshold, -1 elsewhere."""
  cost = dril_action_uncertainty(policy, state, action, activation, input_dropout, dropout, masks)
  neg = cost.less_equal(q)
  cost[neg], cost[~neg] = -1, 1
  return -cost


# ----------------------------------------------------------------------------------------------------------
# RED (models.py:252-284, training.py:68-75): random network distillation on the expert data
# ----------------------------------------------------------------------------------------------------------
class RedDiscriminator:
  def __init__(self, predictor: Sequence[Tensor], target: Sequence[Tensor], state_only: bool = False, activation: str = 'relu', input_dropout: float = 0.0, dropout: float = 0.0,
               sigma_1: Optional[float] = None):
    self.predictor = [torch.nn.Parameter(p.detach().clone().float()) for p in predictor]
    self.target = [p.detach().clone().float() for p in target]  # requires_grad = False (models.py:267-268)
    self.state_only, self.activation, self.input_dropout, self.dropout, self.sigma_1 = state_only, activation, input_dropout, dropout, sigma_1
    self.training = True  # nn.Module default; train.py:147 switches RED to eval() before the loop

  def parameters(self): return list(self.predictor)

  def forward(self, state: Tensor, action: Tensor, masks: Optional[List[Tensor]] = None) -> Tuple[Tensor, Tensor]:
    """models.py:271-274 (dropout only in the predictor, models.py:265-266)."""
    x = state if self.state_only else torch.cat([state, action], dim=1)
    prediction = mlp_forward(self.predictor, x, self.activation, self.input_dropout, self.dropout, self.training, masks)
    return prediction, mlp_forward(self.target, x, self.activation)

  def set_sigma(self, expert_state: Tensor, expert_action: Tensor, masks=None):
    """models.py:277-280: kernel median heuristic on one minibatch (the module is still in train mode here: dropout is active)."""
    if not self.sigma_1:
      prediction, target = self.forward(expert_state, expert_action, masks)
      self.sigma_1 = 1 / squared_distance_mean(prediction, target).median().item()

  def predict_reward(self, state: Tensor, action: Tensor) -> Tensor:
    """models.py:282-284."""
    prediction, target = self.forward(state, action)
    return torch.exp(-self.sigma_1 * (prediction - target).pow(2).mean(dim=1))


def target_estimation_update(disc: RedDiscriminator, optimiser, expert: Dict[str, Tensor], masks=None) -> Tensor:
  """training.py:68-75."""
  optimiser.zero_grad(set_to_none=True)
  prediction, target = disc.forward(expert['states'], expert['actions'], masks)
  loss = (expert['weights'] * (prediction - target).pow(2).mean(dim=1)).mean()
  loss.backward()
  optimiser.step()
  return loss.detach()


# ----------------------------------------------------------------------------------------------------------
# AdRIL / SQIL reward relabelling (models.py:293-318)
# ----------------------------------------------------------------------------------------------------------
class RewardRelabeller:
  def __init__(self, update_freq: int, balanced: bool):
    self.update_freq, self.balanced, self.sample_expert = update_freq, balanced, True  # models.py:294-295

  def resample_and_relabel(self, transitions: Dict[str, Tensor], expert_transitions: Dict[str, Tensor], step: int, num_trajectories: int, num_expert_trajectories: int):
    """models.py:297-318; rewrites `transitions` in place."""
    batch_size = transitions['rewards'].size(0)
    if self.balanced:  # :300-308: alternate whole batches of expert / policy data
      if self.sample_expert:
        for key in transitions.keys(): transitions[key] = expert_transitions[key]
        expert_idxs, policy_idxs = range(batch_size), []
      else:
        expert_idxs, policy_idxs = [], range(batch_size)
      self.sample_expert = not self.sample_expert
    else:  # :309-311
      mix_expert_agent_transitions(transitions, expert_transitions)
      expert_idxs, policy_idxs = range(batch_size // 2), range(batch_size // 2, batch_size)
    if self.update_freq > 0:  # AdRIL, :313-316
      transitions['rewards'][expert_idxs] = 1 / num_expert_trajectories
      round_num = math.ceil(step / self.update_freq)
      transitions['rewards'][policy_idxs] = -1 * (round_num > torch.ceil(transitions['step'][policy_idxs] / self.update_freq)).to(dtype=torch.float32) / max(num_trajectories, 1)
    else:  # SQIL, :317-318
      transitions['rewards'][expert_idxs] = 1
      transitions['rewards'][policy_idxs] = 0


# ----------------------------------------------------------------------------------------------------------
# GMMIL reward (models.py:183-201 with helpers :25-44)
# ----------------------------------------------------------------------------------------------------------
def squared_distance_mean(x: Tensor, y: Tensor) -> Tensor:
  """models.py:25-28: pairwise MEAN (over features) squared difference, [n1, n2]. Computed blockwise so the
  [n1, n2, d] tensor of the reference is never held in full; the arithmetic per entry is the same."""
  out = torch.empty(x.size(0), y.size(0), dtype=x.dtype)
  for i in range(0, x.size(0), 64):
    out[i:i + 64] = (x[i:i + 64, None, :] - y[None, :, :]).pow(2).mean(dim=2)
  return out


def weighted_median(x: Tensor, weights: Tensor) -> Tensor:
  """models.py:40-44."""
  x_sorted, indices = torch.sort(x.flatten())
  w_sorted = (weights.flatten() / weights.sum())[indices]
  median_index = torch.min((torch.cumsum(w_sorted, dim=0) >= 0.5).nonzero())
  return x_sorted[median_index]


class GmmilDiscriminator:
  def __init__(self, state_only: bool = False):
    self.state_only, self.gamma_1, self.gamma_2 = state_only, None, None  # models.py:186-187

  def predict_reward(self, state, action, expert_state, expert_action, weight, expert_weight) -> Tensor:
    """models.py:189-201."""
    sa = state if self.state_only else torch.cat([state, action], dim=1)
    esa = expert_state if self.state_only else torch.cat([expert_state, expert_action], dim=1)
    d_pe = squared_distance_mean(sa, esa)
    if self.gamma_1 is None:  # :193-195 (frozen after the first call)
      self.gamma_1 = 1 / (weighted_median(d_pe, torch.outer(weight, expert_weight)).item() + 1e-8)
      self.gamma_2 = 1 / (weighted_median(squared_distance_mean(esa, esa), torch.outer(expert_weight, expert_weight)).item() + 1e-8)
    wn, wen = weight / weight.sum(), expert_weight / expert_weight.sum()
    d_pp = squared_distance_mean(sa, sa)
    sim = lambda D, wx, wy, g: torch.einsum('i,ij,j->i', [wx, torch.exp(-g * D), wy])  # models.py:32-37
    similarity = sim(d_pe, wn, wen, self.gamma_1) + sim(d_pe, wn, wen, self.gamma_2)
    self_similarity = sim(d_pp, wn, wn, self.gamma_1) + sim(d_pp, wn, wn, self.gamma_2)
    return similarity - self_similarity


# ----------------------------------------------------------------------------------------------------------
# PWIL reward (models.py:216-249 with helpers :205-213)
# ----------------------------------------------------------------------------------------------------------
class PwilDiscriminator:
  def __init__(self, expert_states: Tensor, expert_actions: Tensor, time_horizon: int, reward_scale: float = 5.0, reward_bandwidth_scale: float = 5.0, state_only: bool = False):
    self.state_only, self.time_horizon = state_only, time_horizon
    atoms = expert_states if state_only else torch.cat([expert_states, expert_actions], dim=1)
    self._atoms_raw = atoms.clone()
    inv_scale, self.offset = atoms.std(dim=0, keepdim=True), -atoms.mean(dim=0, keepdim=True)  # models.py:205-208
    inv_scale[inv_scale == 0] = 1
    self.scale = 1 / inv_scale
    self.reward_scale = reward_scale
    self.reward_bandwidth = reward_bandwidth_scale * time_horizon / math.sqrt(atoms.size(1))  # models.py:222
    self.reset()

  def reset(self):  # models.py:228-230
    self.atoms = self.scale * (self._atoms_raw + self.offset)
    self.weights = torch.full((self._atoms_raw.size(0), ), 1 / self._atoms_raw.size(0))

  def compute_reward(self, state: Tensor, action: Tensor) -> float:  # models.py:232-249
    atom = state if self.state_only else torch.cat([state, action], dim=1)
    atom = self.scale * (atom + self.offset)
    weight, cost = 1 / self.time_horizon - 1e-6, 0.0
    dists = torch.linalg.norm(self.atoms - atom, dim=1)
    while weight > 0:
      i = dists.argmin().item()
      ew = self.weights[i].item()
      if weight >= ew:
        cost += ew * dists[i].item()
        weight -= ew
        keep = torch.arange(dists.numel()) != i
        self.atoms, self.weights, dists = self.atoms[keep], self.weights[keep], dists[keep]
      else:
        cost += weight * dists[i].item()
        self.weights[i] -= weight
        weight = 0
    return self.reward_scale * math.exp(-self.reward_bandwidth * cost)


# ----------------------------------------------------------------------------------------------------------
# Replay memory (memory.py:12-68)
# ----------------------------------------------------------------------------------------------------------
FIELDS = ('step', 'states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights')


class Replay:
  def __init__(self, size: int, state_size: int, action_size: int, absorbing: bool, transitions: Optional[dict] = None):
    """memory.py:13-23."""
    self.size, self.num_trajectories, self.idx, self.full, self.absorbing = size, 0, 0, False, absorbing
    z = torch.zeros
    self.data = dict(step=z(size), states=z(size, state_size), actions=z(size, action_size), rewards=z(size), next_states=z(size, state_size),
                     terminals=z(size), timeouts=z(size), weights=z(size))
    if transitions is not None:
      n = min(transitions['states'].size(0), size)
      self.data['step'][:n] = torch.arange(1, n + 1, dtype=torch.float32)
      for k in FIELDS[1:]: self.data[k][:n] = transitions[k][:n]
      self.num_trajectories = transitions['num_trajectories']
      self.idx = n % size
      self.full = self.idx == 0 and n > 0

  def __len__(self): return self.size

  def append(self, step, state, action, reward, next_state, terminal, timeout):
    """memory.py:40-44."""
    for k, v in zip(FIELDS, (step, state, action, reward, next_state, terminal, timeout, 1)):
      self.data[k][self.idx] = torch.as_tensor(v, dtype=torch.float32).reshape(self.data[k][self.idx].shape)
    self.idx = (self.idx + 1) % self.size
    self.full = self.full or self.idx == 0
    if terminal or timeout: self.num_trajectories += 1

  def transfer_transitions(self, memory: 'Replay'):
    """memory.py:46-48: every row of `memory` (all `size` of them, in storage order) appended with weight 1."""
    for i in range(memory.size):
      d = memory.data
      self.append(d['step'][i].item(), d['states'][i], d['actions'][i], d['rewards'][i].item(), d['next_states'][i], bool(d['terminals'][i]), bool(d['timeouts'][i]))

  def draw_indices(self, n: int, rng=np.random) -> np.ndarray:
    """memory.py:51-56, n times (memory.py:59): global-RNG randint with rejection of the newest row."""
    out = []
    newest = (self.idx - 1) % self.size
    while len(out) < n:
      i = int(rng.randint(0, self.size if self.full else self.idx - 1))
      if i != newest: out.append(i)
    return np.asarray(out, dtype=np.int64)

  def gather(self, idxs) -> Dict[str, Tensor]:
    """memory.py:60-62 for given indices."""
    idxs = torch.as_tensor(np.asarray(idxs), dtype=torch.long)
    t = {k: self.data[k][idxs].clone() for k in FIELDS}
    t['absorbing'] = t['states'][:, -1] if self.absorbing else torch.zeros_like(t['terminals'])
    return t

  def sample(self, n: int) -> Dict[str, Tensor]:
    return self.gather(self.draw_indices(n))

  def wrap_for_absorbing_states(self):
    """memory.py:65-68."""
    S, A = self.data['states'].size(1), self.data['actions'].size(1)
    absorbing_state = torch.cat([torch.zeros(S - 1), torch.ones(1)])
    last = (self.idx - 1) % self.size
    self.data['next_states'][last], self.data['terminals'][last] = absorbing_state, 0
    self.append(self.data['step'][last].item(), absorbing_state, torch.zeros(A), 0, absorbing_state, False, False)


def mix_expert_agent_transitions(transitions: Dict[str, Tensor], expert: Dict[str, Tensor]):
  """models.py:287-290."""
  half = transitions['rewards'].size(0) // 2
  for k in transitions.keys(): transitions[k][:half] = expert[k][:half]


# ----------------------------------------------------------------------------------------------------------
# Synthetic environment (SURVEY.md §8d) — CPU twin with the D4RLEnv interface (environments.py:20-61)
# ----------------------------------------------------------------------------------------------------------
ENV_DIMS = {'ant': (111, 8), 'halfcheetah': (17, 6), 'hopper': (11, 3), 'walker2d': (17, 6)}  # obs (without absorbing bit), act
ENVS = ['ant', 'halfcheetah', 'hopper', 'walker2d']  # environments.py:17
EARLY_TERMINATION = {'ant': True, 'halfcheetah': False, 'hopper': True, 'walker2d': True}
TERM_THRESHOLD = {'ant': 0.85, 'halfcheetah': 2.0, 'hopper': 0.72, 'walker2d': 0.85}  # |x'_0| above this ends the episode early


def synthetic_env_params(env_name: str) -> Dict[str, Tensor]:
  """x' = tanh(x M + a N + c); reward = x'.w_r - 1e-3 |a|^2 (SURVEY §8d). Deterministic per env name."""
  obs, act = ENV_DIMS[env_name]
  g = torch.Generator().manual_seed(1234 + ENVS.index(env_name))
  M = torch.randn(obs, obs, generator=g) * (0.3 / math.sqrt(obs)) + torch.eye(obs) * 0.9
  N = torch.randn(act, obs, generator=g) * (0.3 / math.sqrt(act))
  c = torch.randn(obs, generator=g) * 0.05
  w_r = torch.randn(obs, generator=g) / math.sqrt(obs)
  return dict(M=M, N=N, c=c, w_r=w_r)


class SyntheticEnv:
  """CPU twin of the device environment; same call surface as D4RLEnv (environments.py:29-61), B = 1."""

  def __init__(self, env_name: str, absorbing: bool, max_episode_steps: int = 1000, term_threshold: Optional[float] = None):
    self.p = synthetic_env_params(env_name)
    self.obs, self.act = ENV_DIMS[env_name]
    self.absorbing, self.max_episode_steps = absorbing, max_episode_steps
    self.early, self.thr = EARLY_TERMINATION[env_name], (TERM_THRESHOLD[env_name] if term_threshold is None else term_threshold)
    self.x, self.t = None, 0
    self.reset_noise = None  # iterator of [obs] U(0,1) draws, injected

  @property
  def state_size(self): return self.obs + (1 if self.absorbing else 0)

  def _wrap(self, x: Tensor) -> Tensor:
    x = x.unsqueeze(0)
    return torch.cat([x, torch.zeros(1, 1)], dim=1) if self.absorbing else x  # environments.py:32,39

  def reset(self, u: Optional[Tensor] = None) -> Tensor:
    u = next(self.reset_noise) if u is None else u
    self.x, self.t = (u * 2 - 1) * 0.1, 0
    return self._wrap(self.x)

  def step(self, action: Tensor) -> Tuple[Tensor, float, bool]:
    a = action.clamp(min=-1, max=1)[0]  # environments.py:36
    pre = torch.mv(self.p['M'].t(), self.x) + torch.mv(self.p['N'].t(), a) + self.p['c']
    self.x = torch.tanh(pre)
    self.t += 1
    reward = (torch.dot(self.x, self.p['w_r']) - 1e-3 * torch.dot(a, a)).item()
    terminal = (self.early and abs(self.x[0].item()) > self.thr) or self.t >= self.max_episode_steps
    return self._wrap(self.x), reward, bool(terminal)


def evaluate_agent(actor: Sequence[Tensor], env: SyntheticEnv, num_episodes: int, reset_noise: Sequence[Tensor], activation: str = 'relu') -> List[float]:
  """evaluation.py:11-35 (returns only)."""
  returns = []
  with torch.inference_mode():
    for e in range(num_episodes):
      state, terminal, total = env.reset(reset_noise[e]), False, []
      while not terminal:
        state, reward, terminal = env.step(actor_greedy_action(actor, state, activation))
        total.append(reward)
      returns.append(sum(total))
  return returns


def expert_policy_params(env_name: str, absorbing: bool, hidden: int = 64) -> List[Tensor]:
  """Fixed random tanh-MLP 'expert' used to synthesise the D4RL-shaped buffer (SURVEY §8d)."""
  obs, act = ENV_DIMS[env_name]
  S = obs + (1 if absorbing else 0)
  g = torch.Generator().manual_seed(4321 + ENVS.index(env_name))
  W0 = torch.randn(hidden, S, generator=g) / math.sqrt(S)
  W1 = torch.randn(2 * act, hidden, generator=g) / math.sqrt(hidden)
  return [W0, torch.zeros(hidden), W1, torch.zeros(2 * act)]


def build_expert_transitions(raw: Dict[str, Tensor], trajectories: int, subsample: int, absorbing: bool, rng=np.random) -> Dict[str, Tensor]:
  """environments.py:63-125 (`get_dataset`) on a D4RL-shaped dict of tensors."""
  states, actions, next_states, terminals, timeouts = raw['observations'], raw['actions'], raw['next_observations'], raw['terminals'], raw['timeouts']
  state_size, action_size = states.size(1), actions.size(1)
  ends = torch.sort(torch.cat([torch.tensor([-1]), terminals.nonzero().flatten(), timeouts.nonzero().flatten()]))[0]
  trajs = []
  for i in range(len(ends) - 1):
    sl = slice(int(ends[i]) + 1, int(ends[i + 1]) + 1)
    trajs.append(dict(states=states[sl], actions=actions[sl], next_states=next_states[sl], terminals=terminals[sl].clone(), timeouts=timeouts[sl].clone(), weights=torch.ones_like(terminals[sl])))
  if trajectories > 0: trajs = trajs[:trajectories]
  if absorbing:
    abs_state, abs_action = torch.cat([torch.zeros(1, state_size), torch.ones(1, 1)], dim=1), torch.zeros(1, action_size)
    for tr in trajs:
      n = tr['states'].size(0)
      tr['states'] = torch.cat([tr['states'], torch.zeros(n, 1)], dim=1)
      tr['next_states'] = torch.cat([tr['next_states'], torch.zeros(n, 1)], dim=1)
      if not tr['timeouts'][-1]:
        tr['next_states'][-1] = abs_state
        tr['terminals'][-1] = 0
        tr['weights'][-1] = 1 / subsample
        tr['states'] = torch.cat([tr['states'], abs_state], dim=0)
        tr['actions'] = torch.cat([tr['actions'], abs_action], dim=0)
        tr['next_states'] = torch.cat([tr['next_states'], abs_state], dim=0)
        tr['terminals'] = torch.cat([tr['terminals'], torch.zeros(1)])
        tr['timeouts'] = torch.cat([tr['timeouts'], torch.zeros(1)])
        tr['weights'] = torch.cat([tr['weights'], torch.full((1, ), 1 / subsample)])
  if subsample > 1:
    for tr in trajs:
      start, T = rng.choice(subsample), tr['states'].size(0)
      idxs = range(start, T, subsample)
      if absorbing: idxs = sorted(list(set(idxs) | set([T - 2, T - 1])))
      idxs = list(idxs)
      for k in list(tr.keys()): tr[k] = tr[k][idxs]
  out = {k: torch.cat([tr[k] for tr in trajs], dim=0) for k in ('states', 'actions', 'next_states', 'terminals', 'timeouts', 'weights')}
  out['num_trajectories'] = len(trajs)
  out['rewards'] = torch.zeros_like(out['terminals'])
  return out
