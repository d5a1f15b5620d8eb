"""Host-side mirror of the reference's training.py (same function names and argument order); each call is one
C-ABI entry point that runs the whole update for all replicas on the current CUDA stream.

The scalar hyper-parameters that leave every shape unchanged (discount, entropy_target, polyak_factor, grad_penalty,
entropy_bonus, mixup_alpha, pos_class_prior, nonnegative_margin) are a float (every replica) or an [R] tensor (one value per replica, for hyper-parameter sweeps). Keep such a
tensor on the device and alive for as long as a CUDA graph that captured the call is replayed."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple, Union

import torch
from torch import Tensor

from . import _lib
from .memory import TransitionBatch
from .models import GAILDiscriminator, SoftActor, TwinCritic, default_rng
from .optim import Adam

def _workspace(owner, key: str, nbytes: int, device) -> Tensor:
  """Scratch for one fused update, owned by the module that is updated (so two trainers never share it and a buffer whose
  address is baked into a captured CUDA graph is never freed behind the graph's back: a larger request allocates a new
  buffer and the old one stays alive in `owner._ws_retired`). Zero-initialised once: the 4 / 32-float alignment pads of
  the flat gradient buffers are never written by the kernels but are streamed by the AdamW pass."""
  cache = owner.__dict__.setdefault('_ws_cache', {})
  ws = cache.get(key)
  if ws is None or ws.numel() < nbytes:
    if ws is not None: owner.__dict__.setdefault('_ws_retired', []).append(ws)
    ws = torch.zeros(max(nbytes, 256), dtype=torch.uint8, device=device)
    cache[key] = ws
  return ws


def _per_replica(x, R: int, device) -> Tuple[float, Optional[Tensor]]:
  """(scalar, None) for a float; (0.0, [R] float32 device tensor) for per-replica values."""
  if isinstance(x, (int, float)): return float(x), None
  t = torch.as_tensor(x, dtype=torch.float32).to(device).reshape(-1).contiguous()
  assert t.numel() == R, f'per-replica hyper-parameter has {t.numel()} values for {R} replicas'
  return 0.0, t


def _choice_codes(owner, key: str, values, table) -> Tensor:
  """[R] int32 device tensor of table[v] for per-replica string choices, made once per distinct list and kept by `owner` (a captured CUDA graph
  keeps reading it)."""
  cache = owner.__dict__.setdefault('_choice_cache', {})
  k = (key, tuple(values))
  if k not in cache: cache[k] = torch.tensor([table[v] for v in values], dtype=torch.int32, device=owner.device)
  return cache[k]


def _as_batch(t: Union[TransitionBatch, Dict[str, Tensor]], device) -> Tuple[TransitionBatch, Optional[Tensor]]:
  if isinstance(t, TransitionBatch): return t, None
  tb = TransitionBatch.from_dict(t, device=device)
  absorbing = None
  if 'absorbing' in t and not tb.absorbing: absorbing = torch.as_tensor(t['absorbing'], dtype=torch.float32).to(device).reshape(tb.R, tb.B).contiguous()
  return tb, absorbing


def sac_update(actor: SoftActor, critic: TwinCritic, log_alpha: Tensor, target_critic: TwinCritic, transitions, actor_optimiser: Adam, critic_optimiser: Adam,
               temperature_optimiser: Adam, discount, entropy_target, polyak_factor, eps_next: Optional[Tensor] = None, eps_new: Optional[Tensor] = None,
               out: Optional[Dict[str, Tensor]] = None) -> Tuple[Tensor, Tensor]:
  """training.py:14-54. `eps_next` / `eps_new` inject the two policy noise draws (:21, :35); when omitted they are
  drawn on the device. Returns (new_log_probs, min(values_1, values_2)) like the reference (:54)."""
  R, device = actor.replicas, actor.device
  batch, absorbing = _as_batch(transitions, device)
  B, A = batch.B, actor.action_size
  assert batch.R == R and log_alpha.is_cuda and log_alpha.numel() == R
  if eps_next is None: eps_next = default_rng.normal((R, B, A), device, stream_id=11)
  if eps_new is None: eps_new = default_rng.normal((R, B, A), device, stream_id=12)
  eps_next = torch.as_tensor(eps_next, dtype=torch.float32).to(device).reshape(R, B, A).contiguous()
  eps_new = torch.as_tensor(eps_new, dtype=torch.float32).to(device).reshape(R, B, A).contiguous()
  out = {} if out is None else out
  for k, shape in (('log_probs', (R, B)), ('q_values', (R, B)), ('losses', (R, 3))):
    if k not in out: out[k] = torch.empty(shape, device=device)
  a = _lib.SacArgs()
  a.actor, a.critic, a.target = actor.mlp.c_struct(), critic.mlp.c_struct(), target_critic.mlp.c_struct()
  a.actor_opt, a.critic_opt, a.alpha_opt = actor_optimiser.c_struct(), critic_optimiser.c_struct(), temperature_optimiser.c_struct()
  a.log_alpha, a.batch = log_alpha.data_ptr(), batch.c_struct()
  a.absorbing, a.absorbing_from_state, a.R = _lib.ptr(absorbing), int(batch.absorbing and absorbing is None), R
  a.eps_next, a.eps_new = eps_next.data_ptr(), eps_new.data_ptr()
  (a.discount, discount_r), (a.entropy_target, entropy_target_r), (a.polyak_factor, polyak_r) = (_per_replica(x, R, device) for x in (discount, entropy_target, polyak_factor))
  a.discount_r, a.entropy_target_r, a.polyak_r = _lib.ptr(discount_r), _lib.ptr(entropy_target_r), _lib.ptr(polyak_r)
  if polyak_r is not None: a.critic_opt.replica_floats = critic.mlp.flat.numel() // R  # the target shares the twin critic's layout
  a.out_log_probs, a.out_q_values, a.out_losses = out['log_probs'].data_ptr(), out['q_values'].data_ptr(), out['losses'].data_ptr()
  need = _lib.lib().il_sac_workspace_bytes(C.byref(a))
  ws = _workspace(actor, 'sac', need, device)
  a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
  _lib.check(_lib.lib().il_sac_update(_lib.handle(), C.byref(a), _lib.stream()))
  sq = (lambda t: t[0]) if R == 1 else (lambda t: t)
  return sq(out['log_probs']), sq(out['q_values'])


def adversarial_imitation_update(actor: SoftActor, discriminator: GAILDiscriminator, transitions, expert_transitions, discriminator_optimiser: Adam, imitation_cfg,
                                 eps_gp: Optional[Tensor] = None, eps_mix: Optional[Tensor] = None, out_losses: Optional[Tensor] = None,
                                 penalty_pass: Optional[Tensor] = None):
  """training.py:85-134. `eps_gp` injects the U(0,1) draw of :118 and `eps_mix` the Beta draw of :106.

  imitation_cfg.loss_function is a name or one name per replica; mixup_alpha, pos_class_prior and nonnegative_margin are floats or [R] values.
  Without `eps_mix`, a scalar mixup_alpha draws as in the reference (U(0, 1) on the device at 1, torch's Beta otherwise) and per-replica values
  draw Beta(alpha_r, alpha_r) on the device.

  penalty_pass ([R] int32 device tensor of 0 / 1, general discriminator only): replica r takes part in the gradient-penalty pass only where it
  is 1, so a replica whose grad_penalty is 0 runs as a call without a penalty (Trainer passes grad_penalty > 0). None: with per-replica
  grad_penalty every replica takes the pass, its spectral-norm power iterations included. The fused discriminator always skips the pass for
  replicas at 0."""
  R, device = discriminator.replicas, discriminator.device
  pol, _ = _as_batch(transitions, device)
  exp, _ = _as_batch(expert_transitions, device)
  B = pol.B
  losses = [imitation_cfg.loss_function] * R if isinstance(imitation_cfg.loss_function, str) else list(imitation_cfg.loss_function)
  assert len(losses) == R and all(x in _lib.LOSS for x in losses), f'loss_function: one of {sorted(_lib.LOSS)} or R = {R} of them'
  loss_function = losses[0] if len(set(losses)) == 1 else None  # None: per replica
  (grad_penalty, grad_penalty_r), (entropy_bonus, entropy_bonus_r) = _per_replica(imitation_cfg.grad_penalty, R, device), _per_replica(imitation_cfg.entropy_bonus, R, device)
  (pos_class_prior, pos_class_prior_r), (nonnegative_margin, nonnegative_margin_r) = (_per_replica(getattr(imitation_cfg, k), R, device) for k in ('pos_class_prior', 'nonnegative_margin'))
  # per-replica grad_penalty: the gradient-penalty pass runs (replicas at 0 skip their contribution inside it)
  if (grad_penalty > 0 or grad_penalty_r is not None) and eps_gp is None: eps_gp = default_rng.uniform((R, B), device, stream_id=21)
  if 'Mixup' in losses and eps_mix is None:
    alpha, alpha_r = _per_replica(imitation_cfg.mixup_alpha, R, device)  # training.py:106
    if alpha_r is not None: eps_mix = default_rng.beta((R, B), alpha_r, device, stream_id=22)
    elif alpha == 1.0: eps_mix = default_rng.uniform((R, B), device, stream_id=22)  # Beta(1, 1) = U(0, 1): every published config uses mixup_alpha 1
    else: eps_mix = torch.distributions.Beta(torch.full((R, B), alpha, device=device), torch.full((R, B), alpha, device=device)).sample()
  as_dev = lambda t: None if t is None else torch.as_tensor(t, dtype=torch.float32).to(device).reshape(R, B).contiguous()
  eps_gp, eps_mix = as_dev(eps_gp), as_dev(eps_mix)
  hyper = (grad_penalty, grad_penalty_r, entropy_bonus, entropy_bonus_r)
  if discriminator.general:
    loss_codes = None if loss_function is not None else _choice_codes(discriminator, 'loss_function', losses, _lib.LOSS)
    pu = (pos_class_prior, pos_class_prior_r, nonnegative_margin, nonnegative_margin_r)
    return _general_adversarial_update(actor, discriminator, pol, exp, discriminator_optimiser, losses, loss_codes, pu, hyper, eps_gp, eps_mix, out_losses, penalty_pass)
  a = _lib.GailUpdateArgs()
  a.disc, a.opt, a.policy, a.expert = discriminator.c_struct(), discriminator_optimiser.c_struct(), pol.c_struct(), exp.c_struct()
  a.eps_gp, a.eps_mix, a.R, a.loss_function, a.training = _lib.ptr(eps_gp), _lib.ptr(eps_mix), R, _lib.LOSS[losses[0]], int(discriminator.training)
  if loss_function is None: a.loss_function_r = _choice_codes(discriminator, 'loss_function', losses, _lib.LOSS).data_ptr()
  a.grad_penalty, a.grad_penalty_r, a.entropy_bonus, a.entropy_bonus_r = grad_penalty, _lib.ptr(grad_penalty_r), entropy_bonus, _lib.ptr(entropy_bonus_r)
  a.pos_class_prior, a.pos_class_prior_r, a.nonnegative_margin, a.nonnegative_margin_r = pos_class_prior, _lib.ptr(pos_class_prior_r), nonnegative_margin, _lib.ptr(nonnegative_margin_r)
  a.out_losses = _lib.ptr(out_losses)
  _lib.check(_lib.lib().il_gail_update(_lib.handle(), C.byref(a), _lib.stream()))


def _general_adversarial_update(actor, disc: GAILDiscriminator, pol: TransitionBatch, exp: TransitionBatch, opt: Adam, losses, loss_codes, pu, hyper, eps_gp, eps_mix,
                                out_losses, penalty_pass):
  """training.py:85-134 for the non-default discriminator configurations (reward shaping, subtract_log_policy, depth > 1, tanh / sigmoid):
  the log-policy inputs of make_gail_input (models.py:148, evaluated under no_grad) of every pass that runs are computed first, then one
  il_gailx_update call. With per-replica loss functions (loss_codes) the policy and expert passes always run and the Mixup pass runs when any
  replica is Mixup."""
  R, B, device, lib = disc.replicas, pol.B, disc.device, _lib.lib()
  mixup = 'Mixup' in losses
  passes = ('policy', 'expert') + (('mix', ) if mixup else ()) if loss_codes is not None else ('mix', ) if mixup else ('policy', 'expert')
  if loss_codes is not None and not mixup: eps_mix = None  # the Mixup pass runs when eps_mix is passed
  logp = {}
  if disc.subtract_log_policy:
    lp = lambda tb: actor._run(tb.rows[..., :tb.S], given=tb.rows[..., tb.S:tb.S + tb.A], want=('log_prob', ))['log_prob']
    if 'policy' in passes: logp['policy'], logp['expert'] = lp(pol), lp(exp)
    if 'mix' in passes:  # make_gail_input on the mixed state / action (training.py:107-108)
      mix = TransitionBatch(torch.empty_like(pol.rows), pol.S, pol.A, pol.absorbing)
      e, p_, m = exp.c_struct(), pol.c_struct(), mix.c_struct()
      _lib.check(lib.il_gail_mix_batch(_lib.handle(), C.byref(e), C.byref(p_), eps_mix.data_ptr(), R, C.byref(m), _lib.stream()))
      logp['mix'] = lp(mix)
  a = _lib.GailxUpdateArgs()
  a.disc, a.opt, a.params_floats, a.policy, a.expert = disc.cx_struct(), opt.c_struct(), disc.flat.numel(), pol.c_struct(), exp.c_struct()
  a.eps_gp, a.eps_mix = _lib.ptr(eps_gp), _lib.ptr(eps_mix)
  a.logp_policy, a.logp_expert, a.logp_mix = _lib.ptr(logp.get('policy')), _lib.ptr(logp.get('expert')), _lib.ptr(logp.get('mix'))
  a.R, a.loss_function, a.training, a.loss_function_r = R, _lib.LOSS[losses[0]], int(disc.training), _lib.ptr(loss_codes)
  grad_penalty, grad_penalty_r, entropy_bonus, entropy_bonus_r = hyper
  a.grad_penalty, a.grad_penalty_r, a.entropy_bonus, a.entropy_bonus_r = grad_penalty, _lib.ptr(grad_penalty_r), entropy_bonus, _lib.ptr(entropy_bonus_r)
  a.pos_class_prior, a.pos_class_prior_r, a.nonnegative_margin, a.nonnegative_margin_r = pu[0], _lib.ptr(pu[1]), pu[2], _lib.ptr(pu[3])
  a.penalty_pass_r = _lib.ptr(penalty_pass)
  a.out_losses = _lib.ptr(out_losses)
  need = lib.il_gailx_workspace_bytes(C.byref(a))
  ws = _workspace(disc, 'gailx', need, device)
  a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
  _lib.check(lib.il_gailx_update(_lib.handle(), C.byref(a), _lib.stream()))


def behavioural_cloning_update(actor: SoftActor, expert_transition, actor_optimiser: Adam, out_loss: Optional[Tensor] = None, masks=None):
  """training.py:57-64: one maximum-likelihood step of the actor on expert (state, action, weight) rows. A policy with dropout in train mode (DRIL's
  ensemble, train.py:120) runs on the dropout program; `masks` injects its dropout draws ([input mask, hidden masks...], pre-scaled)."""
  R, device = actor.replicas, actor.device
  batch, _ = _as_batch(expert_transition, device)
  a = _lib.BcArgs()
  a.actor, a.opt, a.batch, a.R, a.out_loss = actor.mlp.c_struct(), actor_optimiser.c_struct(), batch.c_struct(), R, _lib.ptr(out_loss)
  if getattr(actor, 'has_dropout', False) and (actor.training or masks is not None):
    if masks is None: masks = actor.draw_masks(batch.B)
    masks = [None if m is None else torch.as_tensor(m, dtype=torch.float32).to(device).reshape(R, batch.B, -1).contiguous() for m in masks]
    need = _lib.lib().il_actor_dropout_workspace_bytes(C.byref(a.actor), R, batch.B)
    ws = _workspace(actor, 'bc_dropout', need, device)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    act_r = getattr(getattr(actor, '_choices', None), 'act_r', None)
    _lib.check(_lib.lib().il_bc_update_dropout(_lib.handle(), C.byref(a), _lib.ptr(masks[0]), _lib.mask_array(masks[1:]), _lib.stream(), _lib.ptr(act_r)))
    return
  if getattr(actor, 'activation_r', None) is not None: raise NotImplementedError('per-replica activations run on the dropout program only')
  need = _lib.lib().il_bc_workspace_bytes(C.byref(a))
  ws = _workspace(actor, 'bc', need, device)
  a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
  _lib.check(_lib.lib().il_bc_update(_lib.handle(), C.byref(a), _lib.stream()))


def target_estimation_update(discriminator, expert_transition, discriminator_optimiser: Adam, out_loss: Optional[Tensor] = None, masks=None):
  """training.py:68-75: one regression step of RED's predictor onto its frozen random target on expert rows (dropout masks drawn on the device in train mode,
  or injected through `masks`)."""
  R, device = discriminator.replicas, discriminator.device
  batch, _ = _as_batch(expert_transition, device)
  if masks is None and discriminator.training and (discriminator.input_dropout > 0 or discriminator.dropout > 0): masks = discriminator.draw_masks(batch.B)
  masks = [None if m is None else torch.as_tensor(m, dtype=torch.float32).to(device).reshape(R, batch.B, -1).contiguous() for m in (masks or [None] * discriminator.predictor.n_layers)]
  a = _lib.RedUpdateArgs()
  a.disc, a.opt, a.batch, a.R = discriminator.c_struct(), discriminator_optimiser.c_struct(), batch.c_struct(), R
  a.mask_in = _lib.ptr(masks[0])
  for i, m in enumerate(masks[1:]): a.mask_hid[i] = _lib.ptr(m)
  a.out_loss = _lib.ptr(out_loss)
  ws = discriminator.workspace(batch.B)
  a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
  _lib.check(_lib.lib().il_red_update(_lib.handle(), C.byref(a), _lib.stream()))
