"""Drives the CUDA path (through the Python mirror -> C ABI) on the seeded cases of oracle/cases.py.
`run_cuda(name, [inputs_r for each replica])` runs ALL replicas in one batched call and returns one output dict
per replica, keyed like the oracle's outputs."""
from types import SimpleNamespace

import numpy as np
import torch

import il_b200
from il_b200 import _lib
from oracle.cases import CASES

DEV = 'cuda'


class Cfg(dict):
  def __getattr__(self, k):
    v = self[k]
    return Cfg(v) if isinstance(v, dict) and not isinstance(v, Cfg) else v

  def get(self, k, d=None): return dict.get(self, k, d)


def _t(x): return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _np(x): return x.detach().float().cpu().numpy().copy()


def _stack(inps, key): return _t(np.stack([i[key] for i in inps]))


def _load_mlp(mlp, inps, prefix, net=0, n=6):
  for r, inp in enumerate(inps): mlp.load_params(r, net, [torch.from_numpy(inp[f'{prefix}_{i}']) for i in range(n)])


def _batch(inps, prefix, S, A, absorbing=True):
  keys = ('step', 'states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights')
  return il_b200.TransitionBatch.from_dict({k: _stack(inps, prefix + k) for k in keys}, absorbing=absorbing, device=DEV)


def _export(mlp, r, net, prefix, out, flat=None):
  views = mlp.layer_views(flat)[net]
  for i, v in enumerate(views): out[f'{prefix}_{i}'] = _np(v[r])


def run_cuda(name, inps):
  c, R = CASES[name], len(inps)
  k = c['kind']
  outs = [dict() for _ in range(R)]
  mcfg = Cfg(hidden_size=c.get('H', 0), depth=2, activation='relu')
  if k == 'actor':
    actor = il_b200.SoftActor(c['S'], c['A'], mcfg, replicas=R)
    _load_mlp(actor.mlp, inps, 'actor')
    s = _stack(inps, 'states')
    o = actor._run(s, eps=_stack(inps, 'eps'), want=('action', 'log_prob', 'mean', 'log_std'))
    g = actor._run(s, want=('action', ))['action']
    lp = actor._run(s, given=_stack(inps, 'actions'), want=('log_prob', ))['log_prob']
    for r in range(R):
      outs[r].update(mean=_np(o['mean'][r]), log_std=_np(o['log_std'][r]), action=_np(o['action'][r]), log_prob_sample=_np(o['log_prob'][r]), greedy=_np(g[r]),
                     log_prob_action=_np(lp[r]))
  elif k == 'sac':
    S, A = c['S'], c['A']
    actor, critic = il_b200.SoftActor(S, A, mcfg, replicas=R), il_b200.TwinCritic(S, A, mcfg, replicas=R)
    _load_mlp(actor.mlp, inps, 'actor')
    _load_mlp(critic.mlp, inps, 'critic1', 0)
    _load_mlp(critic.mlp, inps, 'critic2', 1)
    target = il_b200.create_target_network(critic)
    _load_mlp(target.mlp, inps, 'target1', 0)
    _load_mlp(target.mlp, inps, 'target2', 1)
    log_alpha = _stack(inps, 'log_alpha').reshape(R).contiguous()
    oa = il_b200.AdamW(actor.parameters(), lr=c['lr'], weight_decay=c['wd'])
    oc = il_b200.AdamW(critic.parameters(), lr=c['lr'], weight_decay=c['wd'])
    ot = il_b200.Adam([log_alpha], lr=c['lr'])
    for s in range(c['steps']):
      res = {}
      batch = _batch(inps, f'b{s}_', S, A)
      il_b200.sac_update(actor, critic, log_alpha, target, batch, oa, oc, ot, c['discount'], c['entropy_target'], c['polyak'], eps_next=_stack(inps, f'b{s}_eps_next'),
                         eps_new=_stack(inps, f'b{s}_eps_new'), out=res)
      for r in range(R):
        outs[r][f's{s}_log_probs'], outs[r][f's{s}_q_values'] = _np(res['log_probs'][r]), _np(res['q_values'][r])
        outs[r][f's{s}_value_loss'], outs[r][f's{s}_policy_loss'], outs[r][f's{s}_temperature_loss'] = (_np(res['losses'][r, i]) for i in range(3))
    for r in range(R):
      _export(actor.mlp, r, 0, 'actor', outs[r])
      for t in (0, 1):
        _export(critic.mlp, r, t, f'critic{t + 1}', outs[r])
        _export(target.mlp, r, t, f'target{t + 1}', outs[r])
        _export(critic.mlp, r, t, f'adam_critic_m@{t}', outs[r], oc.exp_avg)
        _export(critic.mlp, r, t, f'adam_critic_v@{t}', outs[r], oc.exp_avg_sq)
      for t in (0, 1):  # oracle numbers critic optimiser params 0..11 across both nets
        for i in range(6):
          outs[r][f'adam_critic_m_{6 * t + i}'] = outs[r].pop(f'adam_critic_m@{t}_{i}')
          outs[r][f'adam_critic_v_{6 * t + i}'] = outs[r].pop(f'adam_critic_v@{t}_{i}')
      _export(actor.mlp, r, 0, 'adam_actor_m', outs[r], oa.exp_avg)
      _export(actor.mlp, r, 0, 'adam_actor_v', outs[r], oa.exp_avg_sq)
      outs[r]['log_alpha'] = _np(log_alpha[r:r + 1])
      outs[r]['adam_alpha_m_0'], outs[r]['adam_alpha_v_0'] = _np(ot.exp_avg[r:r + 1]), _np(ot.exp_avg_sq[r:r + 1])
  elif k == 'bc':
    S, A = c['S'], c['A']
    actor = il_b200.SoftActor(S, A, mcfg, replicas=R)
    _load_mlp(actor.mlp, inps, 'actor')
    opt = il_b200.AdamW(actor.parameters(), lr=c['lr'], weight_decay=c['wd'])
    for s in range(c['steps']):
      loss = torch.empty(R, device=DEV)
      il_b200.behavioural_cloning_update(actor, _batch(inps, f'b{s}_', S, A), opt, out_loss=loss)
      for r in range(R): outs[r][f's{s}_loss'] = _np(loss[r])
    for r in range(R):
      _export(actor.mlp, r, 0, 'actor', outs[r])
      _export(actor.mlp, r, 0, 'adam_m', outs[r], opt.exp_avg)
      _export(actor.mlp, r, 0, 'adam_v', outs[r], opt.exp_avg_sq)
  elif k == 'gail':
    S, A, H = c['S'], c['A'], c['H']
    icfg = Cfg(state_only=False, spectral_norm=c['spectral_norm'], loss_function=c['loss'], grad_penalty=c['grad_penalty'], mixup_alpha=1, entropy_bonus=c['entropy_bonus'],
               pos_class_prior=0.7, nonnegative_margin=float('inf'),
               discriminator=Cfg(hidden_size=H, depth=1, activation='relu', input_dropout=0.5, dropout=0.75, reward_shaping=False, subtract_log_policy=False, reward_function=c['reward']))
    disc = il_b200.GAILDiscriminator(S, A, icfg, 0.97, replicas=R)
    _load_mlp(disc.mlp, inps, 'g', 0, 4)
    nz = lambda x: x / np.maximum(np.linalg.norm(x), 1e-12)
    if c['spectral_norm']:
      for r, inp in enumerate(inps):
        disc.u[r].copy_(_t(np.concatenate([nz(inp['u_0']), nz(inp['u_1'])]).astype(np.float32)))
        disc.v[r].copy_(_t(np.concatenate([nz(inp['v_0']), nz(inp['v_1'])]).astype(np.float32)))
    opt = il_b200.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    disc.eval()
    for s in range(c['steps']):
      pol, exp = _batch(inps, f'p{s}_', S, A), _batch(inps, f'e{s}_', S, A)
      disc.train()
      il_b200.adversarial_imitation_update(None, disc, pol, exp, opt, icfg, eps_gp=_stack(inps, f's{s}_eps_gp'), eps_mix=_stack(inps, f's{s}_eps_mix'))
      disc.eval()
      res = disc._run(pol, want_logits=True)
      for r in range(R): outs[r][f's{s}_reward'], outs[r][f's{s}_logits'] = _np(res['reward'][r]), _np(res['logits'][r])
    for r in range(R):
      _export(disc.mlp, r, 0, 'g', outs[r])
      _export(disc.mlp, r, 0, 'adam_m', outs[r], opt.exp_avg)
      _export(disc.mlp, r, 0, 'adam_v', outs[r], opt.exp_avg_sq)
      if c['spectral_norm']:
        d = S + A
        outs[r]['u_0'], outs[r]['u_1'], outs[r]['v_0'], outs[r]['v_1'] = _np(disc.u[r, :H]), _np(disc.u[r, H:H + 1]), _np(disc.v[r, :d]), _np(disc.v[r, d:d + H])
  elif k == 'gailx':  # reward shaping / subtract_log_policy / depth 2 / tanh / sigmoid / state-only (models.py:157-175) on the general CUDA path
    S, A, H = c['S'], c['A'], c['H']
    icfg = Cfg(state_only=c['state_only'], spectral_norm=c['spectral_norm'], loss_function=c['loss'], grad_penalty=c['grad_penalty'], mixup_alpha=1, entropy_bonus=c['entropy_bonus'],
               pos_class_prior=c.get('pos_class_prior', 0.7), nonnegative_margin=c.get('nonnegative_margin', float('inf')),
               discriminator=Cfg(hidden_size=H, depth=c['depth'], activation=c['activation'], input_dropout=0.5, dropout=0.75, reward_shaping=c['reward_shaping'],
                                 subtract_log_policy=c['subtract_log_policy'], reward_function=c['reward']))
    disc = il_b200.GAILDiscriminator(S, A, icfg, 0.97, replicas=R)
    assert disc.general
    nz = lambda x: x / np.maximum(np.linalg.norm(x), 1e-12)
    nets = [('g', disc.g_mlp, 'g_u', 'g_v')] + ([('h', disc.h_mlp, 'h_u', 'h_v')] if disc.h_mlp is not None else [])
    for name, mlp, un, vn in nets:
      _load_mlp(mlp, inps, name, 0, 2 * mlp.n_layers)
      if c['spectral_norm']:
        for r, inp in enumerate(inps):
          getattr(disc, un)[r].copy_(_t(np.concatenate([nz(inp[f'{name}u_{l}']) for l in range(mlp.n_layers)]).astype(np.float32)))
          getattr(disc, vn)[r].copy_(_t(np.concatenate([nz(inp[f'{name}v_{l}']) for l in range(mlp.n_layers)]).astype(np.float32)))
    actor = None
    if c['subtract_log_policy']:
      actor = il_b200.SoftActor(S, A, Cfg(hidden_size=32, depth=2, activation='relu'), replicas=R)
      _load_mlp(actor.mlp, inps, 'actor')
    opt = il_b200.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
    disc.eval()
    for s in range(c['steps']):
      pol, exp = _batch(inps, f'p{s}_', S, A), _batch(inps, f'e{s}_', S, A)
      disc.train()
      il_b200.adversarial_imitation_update(actor, disc, pol, exp, opt, icfg, eps_gp=_stack(inps, f's{s}_eps_gp'), eps_mix=_stack(inps, f's{s}_eps_mix'))
      disc.eval()
      lp = actor._run(pol.rows[..., :S], given=pol.rows[..., S:S + A], want=('log_prob', ))['log_prob'] if actor is not None else None
      res = disc._run(pol, want_logits=True, log_policy=lp)
      for r in range(R): outs[r][f's{s}_reward'], outs[r][f's{s}_logits'] = _np(res['reward'][r]), _np(res['logits'][r])
    m_all, v_all = opt.exp_avg, opt.exp_avg_sq
    for r in range(R):
      for name, mlp, un, vn in nets:
        off = 0 if name == 'g' else disc.h_mlp.flat.storage_offset() - disc.flat.storage_offset()
        _export(mlp, r, 0, name, outs[r])
        _export(mlp, r, 0, f'adam_{name}_m', outs[r], m_all[:, off:])
        _export(mlp, r, 0, f'adam_{name}_v', outs[r], v_all[:, off:])
        if c['spectral_norm']:
          uo = vo = 0
          for l in range(mlp.n_layers):
            od, idim = mlp.dims[l + 1], mlp.dims[l]
            outs[r][f'{name}u_{l}'], outs[r][f'{name}v_{l}'] = _np(getattr(disc, un)[r, uo:uo + od]), _np(getattr(disc, vn)[r, vo:vo + idim])
            uo, vo = uo + od, vo + idim
  elif k in ('red', 'dril'):  # SURVEY §8f row 4: the dropout MLP program (csrc/dropout_nets.cu) with every mask injected
    S, A, H, depth = c['S'], c['A'], c['H'], c['depth']
    n = 2 * (depth + 1)
    dcfg = Cfg(hidden_size=H, depth=depth, activation=c['activation'], input_dropout=c['input_dropout'], dropout=c['dropout'])
    def masks(prefix):
      out = [_stack(inps, f'{prefix}_in') if c['input_dropout'] > 0 else None]
      return out + [_stack(inps, f'{prefix}_h{l}') if c['dropout'] > 0 else None for l in range(depth)]
    if k == 'red':
      disc = il_b200.REDDiscriminator(S, A, Cfg(state_only=c['state_only'], reward_bandwidth_scale=None, discriminator=dcfg), replicas=R)
      _load_mlp(disc.predictor, inps, 'predictor', 0, n)
      _load_mlp(disc.target, inps, 'target', 0, n)
      opt = il_b200.AdamW(disc.parameters(), lr=c['lr'], weight_decay=c['wd'])
      for s in range(c['steps']):
        loss = torch.empty(R, device=DEV)
        il_b200.target_estimation_update(disc, _batch(inps, f'b{s}_', S, A, absorbing=False), opt, out_loss=loss, masks=masks(f'm{s}'))
        for r in range(R): outs[r][f's{s}_loss'] = _np(loss[r])
      disc.set_sigma_batch(_batch(inps, 'sig_', S, A, absorbing=False), masks=masks('msig'))
      disc.eval()
      rew = disc.predict_reward_batch(_batch(inps, 'p_', S, A, absorbing=False))
      for r in range(R):
        outs[r]['reward'], outs[r]['sigma'] = _np(rew[r]), _np(disc.sigma[r:r + 1])
        _export(disc.predictor, r, 0, 'predictor', outs[r])
        _export(disc.predictor, r, 0, 'adam_m', outs[r], opt.exp_avg)
        _export(disc.predictor, r, 0, 'adam_v', outs[r], opt.exp_avg_sq)
    else:
      actor = il_b200.SoftActor(S, A, dcfg, replicas=R)
      _load_mlp(actor.mlp, inps, 'actor', 0, n)
      opt = il_b200.AdamW(actor.parameters(), lr=c['lr'], weight_decay=c['wd'])
      for s in range(c['steps']):
        loss = torch.empty(R, device=DEV)
        il_b200.behavioural_cloning_update(actor, _batch(inps, f'b{s}_', S, A, absorbing=False), opt, out_loss=loss, masks=masks(f'm{s}'))
        for r in range(R): outs[r][f's{s}_loss'] = _np(loss[r])
      es, ea = _stack(inps, 'expert_states'), _stack(inps, 'expert_actions')
      ps, pa = _stack(inps, 'p_states'), _stack(inps, 'p_actions')
      ev = actor._get_action_uncertainty(es, ea, masks=masks('mthr')).reshape(R, -1)
      actor.set_uncertainty_threshold(es, ea, c['quantile'], masks=masks('mthr'))
      var = actor._get_action_uncertainty(ps, pa, masks=masks('mrew')).reshape(R, -1)
      rew = actor.predict_reward(ps, pa, masks=masks('mrew')).reshape(R, -1)
      for r in range(R):
        outs[r].update(expert_variance=_np(ev[r]), q=_np(actor._q[r:r + 1]), variance=_np(var[r]), reward=_np(rew[r]))
        _export(actor.mlp, r, 0, 'actor', outs[r])
        _export(actor.mlp, r, 0, 'adam_m', outs[r], opt.exp_avg)
        _export(actor.mlp, r, 0, 'adam_v', outs[r], opt.exp_avg_sq)
  elif k == 'gmmil':
    S, A = c['S'], c['A']
    d = il_b200.GMMILDiscriminator(S, A, Cfg(state_only=False), replicas=R)
    p, e, p2 = _batch(inps, 'p_', S, A), _batch(inps, 'e_', S, A), _batch(inps, 'p2_', S, A)
    r1 = d.predict_reward_batch(p, e).clone()
    r2 = d.predict_reward_batch(p2, e)
    for r in range(R): outs[r].update(reward_1=_np(r1[r]), gammas=_np(d.gamma[r]), reward_2=_np(r2[r]))
  elif k == 'pwil':
    S, A = c['S'], c['A']
    # one expert set for all replicas (atoms are shared); replicas differ in the agent trajectory
    n = c['N']
    z = torch.zeros
    mem = il_b200.ReplayMemory(n, S, A, True, transitions=dict(states=_t(inps[0]['expert_states']), actions=_t(inps[0]['expert_actions']), rewards=z(n), next_states=z(n, S),
                                                              terminals=z(n), timeouts=z(n), weights=torch.ones(n), num_trajectories=1), shared=True)
    d = il_b200.PWILDiscriminator(S, A, Cfg(state_only=False, reward_scale=5, reward_bandwidth_scale=5), mem, c['T'], replicas=R)
    rewards = []
    for i in range(c['steps']):
      rewards.append(d.compute_reward_batch(_t(np.stack([inp['states'][i] for inp in inps])), _t(np.stack([inp['actions'][i] for inp in inps]))).clone())
      if (i + 1) % c['T'] == 0: d.reset()
    rw = torch.stack(rewards, dim=1)
    for r in range(R): outs[r]['rewards'] = _np(rw[r])
  elif k == 'mix':  # memory.py:18-23 prefill, :46-48 transfer_transitions, :51-59 index rule, models.py:287-290 mix — R == 1 (the reference's numpy stream)
    assert R == 1
    S, A, inp = c['S'], c['A'], inps[0]
    tr = {key: _t(inp[f'e_{key}']) for key in ('states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights')}
    tr['num_trajectories'] = 3
    em = il_b200.ReplayMemory(c['Ne'], S, A, True, transitions=tr, shared=True)
    am = il_b200.ReplayMemory(c['size'], S, A, True)
    am.transfer_transitions(em)
    for i in range(c['extra']):
      am.append(float(100 + i), _t(inp['x_states'][i:i + 1]), _t(inp['x_actions'][i:i + 1]), float(inp['x_rewards'][i]), _t(inp['x_next_states'][i:i + 1]), float(bool(inp['x_terminals'][i])), 0.0)
    state = np.random.get_state()
    np.random.seed(int(inp['np_seed'][0]))
    try:
      ia, ie = am.draw_indices_host(c['B']), em.draw_indices_host(c['B'])
    finally:
      np.random.set_state(state)
    ta, te = am.gather(torch.from_numpy(ia)), em.gather(torch.from_numpy(ie))
    il_b200.mix_expert_agent_transitions(ta, te)
    outs[0]['idx_agent'], outs[0]['idx_expert'] = ia[0].astype(np.int64), ie[0].astype(np.int64)
    for key in ta.keys(): outs[0][f'mixed_{key}'] = _np(ta[key])
    outs[0]['meta'] = np.int64([int(am._idx[0]), int(am._full[0]), int(am._num_trajectories[0]), int(em._idx[0]), int(em._full[0]), int(em._num_trajectories[0])])
  elif k == 'replay':
    S, A = c['S'], c['A']
    mem = il_b200.ReplayMemory(c['size'], S, A, True, replicas=R)
    for i in range(c['appends']):
      ev = np.stack([int(inp['event'][i]) for inp in inps])
      mem.append(float(i + 1), _t(np.stack([inp['states'][i] for inp in inps])), _t(np.stack([inp['actions'][i] for inp in inps])),
                 _t(np.stack([inp['rewards'][i] for inp in inps])), _t(np.stack([inp['next_states'][i] for inp in inps])), _t((ev == 1).astype(np.float32)),
                 _t((ev == 2).astype(np.float32)), wrap=True)
    for r in range(R):
      for key in ('step', 'states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights'):
        outs[r][f'mem_{key}'] = _np(il_b200.memory._field_view(mem.rows, mem.off, S, A, key)[r])
      outs[r]['meta'] = np.int64([int(mem._idx[r]), int(mem._full[r]), int(mem._num_trajectories[r])])
    if R == 1:  # the reference's numpy index stream (memory.py:51-59)
      np.random.seed(c['seed'])
      t = mem.sample(c['B'])
      for key in t.keys(): outs[0][f'sample_{key}'] = _np(t[key])
  return outs
