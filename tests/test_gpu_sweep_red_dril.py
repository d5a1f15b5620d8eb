"""Per-replica dropout rates and activation of RED and DRIL, all product against product and bitwise unless noted: the mask fill with per-replica
rates against one scalar call per replica slice (keyed and unkeyed launches, eager and graph-replayed, with the scalar counter advance); the RED
and DRIL kernel entries with mixed relu / tanh / sigmoid replicas against uniform calls of each activation (and against the float64 port at the
single-call tolerances); `train.py -m` over the rate x activation grid crossed with a seed sweep, whose jobs equal their single runs; a uniform
group's blocks against the uniform runs of their jobs; and the six tuned RED / DRIL overlays, whose discriminator.pth loads into the reference's
nn.Sequential layout."""
import glob
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

RATES = [0.1, 0.5, 0.0999999, 0.75, 0.3]  # per replica; each rounded once to float32, as the scalar path's `float p` is
SEEDS = [0, 7, 123456789, 2**32 - 1, 42]
ACTS = ['relu', 'tanh', 'sigmoid', 'tanh', 'relu']


def _bits(t: torch.Tensor) -> torch.Tensor:
  return t.contiguous().view(torch.int32)


# ---- 1. the mask fill --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('n', [1, 6, 37, 64, 1003])
def test_unkeyed_mask_fill_with_rates_equals_one_scalar_call_per_replica(n):
  """Element i of the [R, n] draw takes replica i // n's rate; with n % 4 != 0 a quad straddles two replicas."""
  from il_b200 import _lib
  lib, h, st, R = _lib.lib(), _lib.handle(), _lib.stream(), len(RATES)
  p_r = torch.tensor(RATES, dtype=torch.float32, device='cuda')
  ctr = torch.tensor([13], dtype=torch.int64, device='cuda')
  out = torch.full((R, n), float('nan'), device='cuda')
  _lib.check(lib.il_fill_dropout_mask(h, out.data_ptr(), R * n, 0.2, 99, 31, ctr.data_ptr(), st, p_r.data_ptr(), R))
  for r, p in enumerate(RATES):
    ref = torch.full((R, n), float('nan'), device='cuda')
    _lib.check(lib.il_fill_dropout_mask(h, ref.data_ptr(), R * n, p, 99, 31, ctr.data_ptr(), st, None, 0))
    assert torch.equal(_bits(out[r]), _bits(ref[r])), f'replica {r} (p = {p})'
  keep = out[0][out[0] > 0]
  assert keep.numel() == 0 or torch.equal(keep, torch.full_like(keep, 1 / (1 - torch.tensor(RATES[0], dtype=torch.float32)).item()))


@pytest.mark.parametrize('n', [1, 6, 37, 1003])
def test_keyed_mask_fill_with_rates_equals_one_scalar_call_per_replica(n):
  from il_b200 import _lib
  lib, h, st, R = _lib.lib(), _lib.handle(), _lib.stream(), len(RATES)
  p_r, keys = torch.tensor(RATES, dtype=torch.float32, device='cuda'), _lib.seed_array(SEEDS, 'cuda')
  ctr = torch.tensor([5], dtype=torch.int64, device='cuda')
  out = torch.full((R, n), float('nan'), device='cuda')
  _lib.check(lib.il_fill_dropout_mask_r(h, out.data_ptr(), R, n, 0.2, keys.data_ptr(), 31, ctr.data_ptr(), st, p_r.data_ptr()))
  for r, (p, s) in enumerate(zip(RATES, SEEDS)):
    ref = torch.full((n, ), float('nan'), device='cuda')
    _lib.check(lib.il_fill_dropout_mask(h, ref.data_ptr(), n, p, s, 31, ctr.data_ptr(), st))
    assert torch.equal(_bits(out[r]), _bits(ref)), f'replica {r} (p = {p}, seed {s})'


@pytest.mark.parametrize('keyed', [False, True])
def test_mask_draws_with_rates_replay_from_a_graph_and_advance_the_counter_as_scalar_draws(keyed):
  from il_b200.models import _RNG
  R, shapes = len(RATES), [(7, 3), (5, 6), (9, 1)]
  p_r = torch.tensor(RATES, dtype=torch.float32, device='cuda')
  mk = lambda: _RNG(list(SEEDS) if keyed else 1979, 'cuda')
  eager = mk()
  want = [eager.dropout_mask(torch.empty(R, *s, device='cuda'), 0.2, 32, p_r) for s in shapes]
  cap = mk()
  cap._ctr('cuda')
  outs = [torch.full((R, *s), float('nan'), device='cuda') for s in shapes]
  side = torch.cuda.Stream()
  side.wait_stream(torch.cuda.current_stream())
  with torch.cuda.stream(side):
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=side):
      for o in outs: cap.dropout_mask(o, 0.2, 32, p_r)
  torch.cuda.current_stream().wait_stream(side)
  for _ in range(2):  # replayed from a reset counter, twice
    cap.counter.zero_()
    g.replay()
    torch.cuda.synchronize()
    for o, w in zip(outs, want): assert torch.equal(_bits(o), _bits(w))
    assert int(cap.counter) == int(eager.counter)
  for r, (p, s) in enumerate(zip(RATES, SEEDS)):  # replica r's slices are the scalar draws of its rate (and seed), counter included
    one = _RNG(s if keyed else 1979, 'cuda')
    for w, shp in zip(want, shapes):
      ref = one.dropout_mask(torch.empty(1 if keyed else R, *shp, device='cuda'), p, 32)
      assert torch.equal(_bits(w[r]), _bits(ref[0 if keyed else r])), f'replica {r}'
    assert int(one.counter) == int(eager.counter)


# ---- 2. kernel entries: mixed activations against uniform calls of each activation ------------------------------------------------------
def _imitation(alg, **disc):
  from il_b200.config import load_config
  cfg = load_config([f'algorithm={alg}', 'imitation.discriminator.hidden_size=24', 'imitation.discriminator.depth=2'] +
                    [f'imitation.discriminator.{k}={v}' for k, v in disc.items()])
  return cfg.imitation


def _port_params(mlp, r):
  return [p.double().cpu() for p in mlp.export_params(r, 0)]


def _masks(R, n, widths, seed):
  g = torch.Generator().manual_seed(seed)
  return [(torch.rand(R, n, w, generator=g) >= 0.3).float().div(0.7).cuda() for w in widths]


def test_red_entries_with_mixed_activations_equal_uniform_calls():
  from il_b200 import AdamW, REDDiscriminator
  from il_b200.training import target_estimation_update
  from oracle import port
  R, B, S, A = len(ACTS), 33, 11, 3
  cfg = _imitation('RED', input_dropout=0.2, dropout=0.4)
  torch.manual_seed(1)
  mixed = REDDiscriminator(S, A, cfg, replicas=R, device='cuda', activation=ACTS)
  assert mixed.activation_r == ACTS and mixed._choices.act_r is not None
  s, a = torch.randn(R, B, S, device='cuda'), torch.randn(R, B, A, device='cuda').clamp(-0.9, 0.9)
  din, H = S + A, 24
  mask_sets = [_masks(R, B, [din, H, H], seed) for seed in range(3)]

  def run(d):
    batch = d._batch_of(s, a)
    batch.rows[..., batch.off['weights']] = torch.rand(R, B, generator=torch.Generator().manual_seed(4)).cuda()
    opt, losses = AdamW(d.parameters(), lr=1e-3, weight_decay=0.1), []
    for m in mask_sets[:2]:
      loss = torch.zeros(R, device='cuda')
      target_estimation_update(d, batch, opt, out_loss=loss, masks=m)
      losses.append(loss)
    d.set_sigma_batch(batch, masks=mask_sets[2])
    d.eval()
    reward = d.predict_reward_batch(batch).clone()
    torch.cuda.synchronize()
    return dict(predictor=d.predictor.flat.clone(), target=d.target.flat.clone(), loss=torch.stack(losses, 1), sigma=d.sigma.clone(), reward=reward,
                m=opt.exp_avg.clone(), v=opt.exp_avg_sq.clone()), batch

  init_pred, init_targ = mixed.predictor.flat.clone(), mixed.target.flat.clone()
  got, batch = run(mixed)
  for act in sorted(set(ACTS)):
    uni = REDDiscriminator(S, A, cfg, replicas=R, device='cuda', activation=act)
    assert uni._choices.act_r is None
    uni.predictor.flat.copy_(init_pred)
    uni.target.flat.copy_(init_targ)
    ref, _ = run(uni)
    for r in (r for r in range(R) if ACTS[r] == act):
      for k in got: assert torch.equal(_bits(got[k][r]), _bits(ref[k][r])), f'replica {r} ({act}): {k}'
  # the float64 port: replica r's sigma and reward from the trained parameters, with its own activation
  for r in range(R):
    x = torch.cat([s[r], a[r]], 1).double().cpu()
    masks = [m[r].double().cpu() for m in mask_sets[2]]
    pp, tp = _port_params(mixed.predictor, r), _port_params(mixed.target, r)
    sig = 1 / port.squared_distance_mean(port.mlp_forward(pp, x, ACTS[r], 0.2, 0.4, True, list(masks)), port.mlp_forward(tp, x, ACTS[r])).median().item()
    assert abs(float(got['sigma'][r]) - sig) <= 2e-4 * abs(sig), f'replica {r}: sigma'
    rew = torch.exp(-float(got['sigma'][r]) * (port.mlp_forward(pp, x, ACTS[r]) - port.mlp_forward(tp, x, ACTS[r])).pow(2).mean(1))
    torch.testing.assert_close(got['reward'][r].double().cpu(), rew, rtol=2e-4, atol=2e-5, msg=f'replica {r}: reward')


def test_dril_entries_with_mixed_activations_equal_uniform_calls():
  from il_b200 import AdamW, SoftActor, _lib
  from il_b200.memory import TransitionBatch
  from il_b200.training import behavioural_cloning_update
  from oracle import port
  R, B, S, A, H, E = len(ACTS), 29, 11, 3, 24, SoftActor.ENSEMBLE
  cfg = _imitation('DRIL', input_dropout=0.2, dropout=0.4).discriminator
  torch.manual_seed(2)
  mixed = SoftActor(S, A, cfg, replicas=R, device='cuda', activation=ACTS)
  s, a = torch.randn(R, B, S, device='cuda'), torch.rand(R, B, A, device='cuda') * 1.8 - 0.9
  off, row = _lib.py_row_layout(S, A)
  rows = torch.zeros(R, B, row, device='cuda')
  rows[..., :S], rows[..., S:S + A], rows[..., off['weights']] = s, a, 1.0
  batch = TransitionBatch(rows, S, A, False)
  bc_masks = [_masks(R, B, [S, H, H], seed) for seed in range(2)]
  ens_masks = _masks(R, B * E, [S, H, H], 7)

  def run(d):
    opt, losses = AdamW(d.parameters(), lr=1e-3, weight_decay=0.01), []
    for m in bc_masks:
      loss = torch.zeros(R, device='cuda')
      behavioural_cloning_update(d, batch, opt, out_loss=loss, masks=m)
      losses.append(loss)
    lp = d._log_prob_dropout(s, a, repeat=E, masks=ens_masks).clone()
    torch.cuda.synchronize()
    return dict(params=d.mlp.flat.clone(), loss=torch.stack(losses, 1), log_prob=lp, m=opt.exp_avg.clone(), v=opt.exp_avg_sq.clone())

  init = mixed.mlp.flat.clone()
  got = run(mixed)
  for act in sorted(set(ACTS)):
    uni = SoftActor(S, A, cfg, replicas=R, device='cuda', activation=act)
    uni.mlp.flat.copy_(init)
    ref = run(uni)
    for r in (r for r in range(R) if ACTS[r] == act):
      for k in got: assert torch.equal(_bits(got[k][r]), _bits(ref[k][r])), f'replica {r} ({act}): {k}'
  for r in range(R):  # the float64 port: the ensemble log-density of the trained policy
    params = [p.double().cpu() for p in mixed.mlp.export_params(r, 0)]
    x, y = torch.repeat_interleave(s[r], E, 0).double().cpu(), torch.repeat_interleave(a[r], E, 0).double().cpu()
    want = port.actor_log_prob(params, x, y, ACTS[r], input_dropout=0.2, dropout=0.4, training=True, masks=[m[r].double().cpu() for m in ens_masks])
    torch.testing.assert_close(got['log_prob'][r].double().cpu(), want, rtol=1e-4, atol=1e-4, msg=f'replica {r}: log_prob')


def test_red_and_dril_init_with_each_replicas_gain_and_refuse_mixed_presence():
  from il_b200 import REDDiscriminator, SoftActor
  from il_b200.net import ReplicaRNG, init_fcnn_params
  S, A = 11, 3
  cfg = _imitation('RED', input_dropout=0.2, dropout=0.4)
  d = REDDiscriminator(S, A, cfg, replicas=3, device='cuda', rng=ReplicaRNG(5, 3), activation=['relu', 'tanh', 'sigmoid'], dropout=[0.1, 0.4, 0.6])
  for r, act in enumerate(['relu', 'tanh', 'sigmoid']):
    g = ReplicaRNG(5 + r, 1)
    with g.replica(0):
      dims = d.predictor.dims
      want_p, want_t = init_fcnn_params(dims, act), init_fcnn_params(dims, act)
    for got, want in zip(d.predictor.export_params(r, 0) + d.target.export_params(r, 0), want_p + want_t): assert torch.equal(got, want)
  assert set(d.state_dict()) == set(REDDiscriminator(S, A, cfg, device='cuda').state_dict())
  with pytest.raises(ValueError, match='presence'):
    REDDiscriminator(S, A, cfg, replicas=2, device='cuda', input_dropout=[0, 0.2])
  with pytest.raises(ValueError, match='need a dropout policy'):
    SoftActor(S, A, _imitation('DRIL', input_dropout=0, dropout=0).discriminator, replicas=2, device='cuda', activation=['relu', 'tanh'])


# ---- 3. loops ----------------------------------------------------------------------------------------------------------------------
SMALL = ['env=hopper', 'steps=30', 'training.start=10', 'evaluation.interval=15', 'evaluation.episodes=1', 'logging.interval=10', 'imitation.trajectories=2',
         'memory.size=60', 'training.batch_size=16', 'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'cuda_graphs=true',
         'imitation.pretraining.iterations=4', 'imitation.discriminator.hidden_size=16']
GRID = ['imitation.discriminator.input_dropout=0.1,0.3', 'imitation.discriminator.dropout=0.2,0.5', 'imitation.discriminator.activation=relu,tanh']
FILES = ('agent.pth', 'discriminator.pth', 'metrics.pth')


def _same(a, b, where=''):
  import numpy as np
  if isinstance(a, torch.Tensor):
    assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape, where
    assert torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8)), f'{where}: differs'
  elif isinstance(a, np.ndarray):
    assert isinstance(b, np.ndarray) and a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), f'{where}: differs'
  elif isinstance(a, dict):
    assert set(a) == set(b), f'{where}: keys {set(a) ^ set(b)}'
    for k in a: _same(a[k], b[k], f'{where}.{k}')
  elif isinstance(a, (list, tuple)):
    assert len(a) == len(b), f'{where}: length'
    for i, (x, y) in enumerate(zip(a, b)): _same(x, y, f'{where}[{i}]')
  elif isinstance(a, float):
    assert a == b or (a != a and b != b), f'{where}: {a} != {b}'
  else:
    assert a == b, f'{where}: {a!r} != {b!r}'


def _load(d):
  return {f: torch.load(os.path.join(d, f), weights_only=False) for f in FILES if os.path.exists(os.path.join(d, f))}


def _single(tmp_path, name, overrides):
  from il_b200.train import main
  out = str(tmp_path / name)
  main(overrides + [f'output_dir={out}'])
  (d, ) = glob.glob(os.path.join(out, '*', '*'))
  return _load(d)


@pytest.mark.parametrize('alg', ['DRIL', 'RED'])
def test_rate_activation_seed_sweep_jobs_equal_their_single_runs(alg, tmp_path, capsys):
  from il_b200.config import expand_sweep
  from il_b200.train import main
  base = [f'algorithm={alg}'] + SMALL + ['replicas=1']
  extra = ['imitation.quantile_cutoff=0.8,0.95'] if alg == 'DRIL' else []
  argv = base + GRID + extra + ['seed=1,2']
  out = str(tmp_path / 'sweep')
  main(['-m'] + argv + [f'output_dir={out}'])
  assert 'in 1 group(s)' in capsys.readouterr().out
  (run, ) = glob.glob(os.path.join(out, '*_sweeper', '*'))
  _, jobs = expand_sweep(['-m'] + argv)
  assert sorted(int(j) for j in os.listdir(run)) == list(range(len(jobs)))
  for job in jobs:
    got = _load(os.path.join(run, str(job.num)))
    ref = _single(tmp_path, f'job{job.num}', job.overrides)
    assert set(got) == set(FILES) == set(ref)
    _same(got, ref, f'{alg} job {job.num}: {job.overrides[-4:]}')


def _buffers(tr):
  d, o = tr.discriminator, tr.discriminator_optimiser
  out = dict(actor=tr.actor.mlp.flat, critic=tr.critic.mlp.flat, log_alpha=tr.log_alpha, rows=tr.batch.rows, disc=d.parameters()[0], disc_m=o.exp_avg, disc_v=o.exp_avg_sq,
             return_sum=tr.return_sum, state=tr.state, **tr.sac_out)
  if getattr(d, '_q', None) is not None: out['dril_q'] = d._q
  if getattr(d, 'sigma', None) is not None: out.update(sigma=d.sigma, target=d.target.flat)
  return {k: v.detach().reshape(tr.R, -1).clone() for k, v in out.items()}


@pytest.mark.parametrize('alg', ['DRIL', 'RED'])
def test_uniform_group_blocks_equal_the_uniform_runs_of_their_jobs(alg):
  """A group of J jobs x 2 replicas (one program seed) against, per job, the uniform program of the same J x 2 replicas at that job's values."""
  from il_b200.config import load_config
  from il_b200.train import Trainer
  per_job = {'imitation.discriminator.input_dropout': [0.1, 0.3, 0.3], 'imitation.discriminator.dropout': [0.5, 0.2, 0.5],
             'imitation.discriminator.activation': ['tanh', 'relu', 'sigmoid']}
  J, R, steps = 3, 2, 24
  base = [f'algorithm={alg}'] + SMALL + ['seed=5', f'replicas={J * R}']

  def drive(tr):
    tr.pretrain_discriminator()
    for _ in range(steps): tr.train_step()
    torch.cuda.synchronize()
    return _buffers(tr)
  got = drive(Trainer(load_config(base), per_replica={k: [v for v in vals for _ in range(R)] for k, vals in per_job.items()}))
  for j in range(J):
    uni = Trainer(load_config(base + [f'{k}={vals[j]}' for k, vals in per_job.items()]))
    assert not uni.per_replica
    ref = drive(uni)
    blk = slice(j * R, (j + 1) * R)
    for k, v in ref.items(): assert torch.equal(got[k][blk], v[blk]), f'job {j}: {k} differs'


@pytest.mark.parametrize('name', [f'{a}_{n}_trajectories' for a in ('RED', 'DRIL') for n in (5, 10, 25)])
def test_tuned_overlay_runs_and_its_discriminator_loads_into_the_reference_layout(name, tmp_path):
  """Each overlay runs briefly through train.py; discriminator.pth loads strictly into the reference's nn.Sequential (models.py:48-69: [Dropout],
  Linear, [Dropout], activation, ..., Linear) built from the overlay's own shape."""
  from torch import nn
  from il_b200.config import load_config
  alg = name.split('_')[0]
  short = ['env=hopper', 'steps=12', 'training.start=6', 'evaluation.interval=12', 'evaluation.episodes=1', 'memory.size=24', 'imitation.pretraining.iterations=2',
           'training.batch_size=16']
  ov = [f'algorithm={alg}', f'optimised_hyperparameters={name}'] + short
  sd = _single(tmp_path, name, ov)['discriminator.pth']
  cfg = load_config(ov)
  d = cfg.imitation.discriminator
  S, A = 11 + int(cfg.imitation.absorbing), 3  # hopper, plus the absorbing-state indicator
  acts = dict(relu=nn.ReLU, tanh=nn.Tanh, sigmoid=nn.Sigmoid)

  def fcnn(din, dout, dropout_layers):
    layers = [nn.Dropout(d.input_dropout)] if dropout_layers and d.input_dropout > 0 else []
    sizes = [din] + [d.hidden_size] * d.depth
    for l in range(d.depth):
      layers.append(nn.Linear(sizes[l], sizes[l + 1]))
      if dropout_layers and d.dropout > 0: layers.append(nn.Dropout(d.dropout))
      layers.append(acts[d.activation]())
    return nn.Sequential(*layers, nn.Linear(sizes[-1], dout))
  if alg == 'DRIL':
    want = nn.ModuleDict(dict(actor=fcnn(S, 2 * A, True)))
  else:
    din = S + A
    want = nn.ModuleDict(dict(predictor=nn.ModuleDict(dict(embedding=fcnn(din, din, True))), target=nn.ModuleDict(dict(embedding=fcnn(din, din, False)))))
  want.load_state_dict({k: v.cpu() for k, v in sd.items()}, strict=True)
