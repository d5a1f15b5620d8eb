"""Seed sweeps (per-replica seeds), all bitwise, product against product: each il_*_r RNG entry against one scalar call per replica with the same
stream id and counter (eager and graph-replayed, with the counter advance of a single-replica call), then `train.py -m ... seed=a,b,c` sweeps
whose job files equal the separate runs of each seed, a replicas=2 seed sweep whose replica k of job j is the run of seed s_j + k, and a seed
sweep crossed with a learning-rate sweep in one group."""
import glob
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SEEDS = [0, 7, 123456789, 2**32 - 1, 42]  # non-consecutive, both 32-bit halves of the key exercised
ALPHAS = [1.0, 0.4, 2.5, 1.0, 0.7]  # Beta(alpha, alpha) per replica; alpha 1 is the uniform draw


def _bits(t: torch.Tensor) -> torch.Tensor:
  return t.contiguous().view(torch.int32)


def _ctr(c0=13):
  return torch.tensor([c0], dtype=torch.int64, device='cuda')


# ---- 1. kernels -----------------------------------------------------------------------------------------------------------------
def _keyed_and_single(kind, n, stream_id=6, c0=13):
  """(the [R, n] keyed draw, the R single-replica draws) of one fill kind at counter c0."""
  from il_b200 import _lib
  lib, h, st = _lib.lib(), _lib.handle(), _lib.stream()
  R, keys = len(SEEDS), _lib.seed_array(SEEDS, 'cuda')
  alphas = torch.tensor(ALPHAS, device='cuda')
  out, ctr = torch.full((R, n), float('nan'), device='cuda'), _ctr(c0)
  if kind == 'normal': _lib.check(lib.il_fill_normal_r(h, out.data_ptr(), R, n, keys.data_ptr(), stream_id, ctr.data_ptr(), st))
  elif kind == 'uniform': _lib.check(lib.il_fill_uniform_r(h, out.data_ptr(), R, n, keys.data_ptr(), stream_id, ctr.data_ptr(), st))
  elif kind == 'beta': _lib.check(lib.il_fill_beta_r(h, out.data_ptr(), R, n, alphas.data_ptr(), keys.data_ptr(), stream_id, ctr.data_ptr(), st))
  else: _lib.check(lib.il_fill_dropout_mask_r(h, out.data_ptr(), R, n, 0.3, keys.data_ptr(), stream_id, ctr.data_ptr(), st))
  refs = []
  for r, s in enumerate(SEEDS):
    ref = torch.full((n, ), float('nan'), device='cuda')
    if kind == 'normal': _lib.check(lib.il_fill_normal(h, ref.data_ptr(), n, s, stream_id, ctr.data_ptr(), st))
    elif kind == 'uniform': _lib.check(lib.il_fill_uniform(h, ref.data_ptr(), n, s, stream_id, ctr.data_ptr(), st))
    elif kind == 'beta': _lib.check(lib.il_fill_beta(h, ref.data_ptr(), 1, n, alphas[r:r + 1].data_ptr(), s, stream_id, ctr.data_ptr(), st))
    else: _lib.check(lib.il_fill_dropout_mask(h, ref.data_ptr(), n, 0.3, s, stream_id, ctr.data_ptr(), st))
    refs.append(ref)
  torch.cuda.synchronize()
  return out, refs


@pytest.mark.parametrize('n', [1, 6, 37, 64, 1003])
@pytest.mark.parametrize('kind', ['normal', 'uniform', 'beta', 'dropout'])
def test_keyed_fill_equals_one_scalar_call_per_replica(kind, n):
  out, refs = _keyed_and_single(kind, n)
  for r, ref in enumerate(refs):
    assert not torch.isnan(ref).any()
    assert torch.equal(_bits(out[r]), _bits(ref)), f'{kind} n={n}: replica {r} (seed {SEEDS[r]})'
  if kind == 'beta':  # alpha == 1 replicas are the uniform draws
    uni, _ = _keyed_and_single('uniform', n)
    assert torch.equal(_bits(out[0]), _bits(uni[0])) and torch.equal(_bits(out[3]), _bits(uni[3]))


def _rng_draws(rng, alphas, n):
  """A sequence of [R, n] draws through _RNG (normal, uniform, beta, dropout mask, normal), R = len(alphas); returns them and the final counter."""
  R, a = len(alphas), torch.tensor(alphas, device='cuda')
  d = [rng.normal((R, n), 'cuda', stream_id=1), rng.uniform((R, n), 'cuda', stream_id=2), rng.beta((R, n), a, 'cuda', stream_id=8),
       rng.dropout_mask(torch.empty(R, n, device='cuda'), 0.25, 31), rng.normal((R, n + 2), 'cuda', stream_id=7)]
  return d, int(rng.counter)


def test_keyed_rng_advances_its_counter_like_a_single_replica_source():
  from il_b200.models import _RNG
  got, c = _rng_draws(_RNG(SEEDS, 'cuda'), ALPHAS, 11)
  assert c == 4 * 3 + 4  # ceil(11 / 4) per draw of 11 per replica, ceil(13 / 4) for the last: not the 5-replica totals
  for r, s in enumerate(SEEDS):
    ref, c1 = _rng_draws(_RNG(s, 'cuda'), ALPHAS[r:r + 1], 11)
    assert c1 == c
    for i, (a, b) in enumerate(zip(got, ref)): assert torch.equal(_bits(a[r]), _bits(b[0])), f'draw {i}, replica {r}'


def _rings(size=50):
  """A 5-replica memory with rings in different states (not full at several fill levels, full at several positions) and a shared memory."""
  from il_b200.memory import ReplayMemory
  S, A, R = 4, 2, len(SEEDS)
  per = ReplayMemory(size, S, A, False, replicas=R, device='cuda')
  per._idx.copy_(torch.tensor([5, 17, 0, 3, 40], dtype=torch.int32))
  per._full.copy_(torch.tensor([0, 1, 1, 0, 1], dtype=torch.int32))
  shared = ReplayMemory(size, S, A, False, replicas=R, shared=True, device='cuda')
  shared._idx.fill_(23); shared._full.fill_(1)
  return per, shared


def _single_ring(mem, r):
  from il_b200.memory import ReplayMemory
  one = ReplayMemory(mem.size, mem.state_size, mem.action_size, False, replicas=1, shared=mem.shared, device='cuda')
  m = 0 if mem.shared else r
  one._idx.copy_(mem._idx[m:m + 1]); one._full.copy_(mem._full[m:m + 1])
  return one


@pytest.mark.parametrize('n', [1, 37, 300])
@pytest.mark.parametrize('shared', [False, True])
def test_keyed_index_sampling_equals_one_scalar_call_per_replica(shared, n):
  per, sh = _rings()
  mem = sh if shared else per
  mem.seed = [s + 7919 for s in SEEDS]
  mem._rng_counter.fill_(101)
  got = mem.sample_indices_device(n, stream_id=4).clone()
  for r, s in enumerate(SEEDS):
    one = _single_ring(mem, r)
    one.seed = s + 7919
    one._rng_counter.fill_(101)
    ref = one.sample_indices_device(n, stream_id=4)
    assert torch.equal(got[r], ref[0]), f'replica {r}'
    assert int(one._rng_counter) == int(mem._rng_counter) == 101 + n


def test_keyed_calls_replay_from_a_cuda_graph():
  from il_b200.models import _RNG
  from il_b200 import _lib
  n = 37
  rng, (per, _) = _RNG(SEEDS, 'cuda'), _rings()
  per.seed = SEEDS
  alphas = torch.tensor(ALPHAS, device='cuda')
  outs = [torch.empty(len(SEEDS), n, device='cuda') for _ in range(4)]
  idx = torch.empty(len(SEEDS), n, dtype=torch.int32, device='cuda')

  def body():
    rng.normal(None, 'cuda', stream_id=1, out=outs[0])
    rng.uniform(None, 'cuda', stream_id=2, out=outs[1])
    rng.beta(None, alphas, 'cuda', stream_id=8, out=outs[2])
    rng.dropout_mask(outs[3], 0.5, 31)
    per.sample_indices_device(n, out=idx, stream_id=3)

  rng._ctr('cuda').fill_(9); per._rng_counter.fill_(9)
  body()
  torch.cuda.synchronize()
  eager, eager_idx, counters = [o.clone() for o in outs], idx.clone(), (int(rng.counter), int(per._rng_counter))
  for o in outs: o.fill_(float('nan'))
  idx.fill_(-1)
  rng.counter.fill_(9); per._rng_counter.fill_(9)
  torch.cuda.synchronize()
  before = _lib.launch_count()
  g = torch.cuda.CUDAGraph()
  with torch.cuda.graph(g):
    body()
  assert _lib.launch_count() - before == 10  # one launch per draw plus its counter advance: what the scalar path launches
  g.replay()
  torch.cuda.synchronize()
  for a, b in zip(outs, eager): assert torch.equal(_bits(a), _bits(b))
  assert torch.equal(idx, eager_idx) and (int(rng.counter), int(per._rng_counter)) == counters


def test_keyed_entries_refuse_a_null_key_array():
  from il_b200 import _lib
  out = torch.empty(2, 8, device='cuda')
  with pytest.raises(RuntimeError, match='il_fill_normal_r: bad argument'):
    _lib.check(_lib.lib().il_fill_normal_r(_lib.handle(), out.data_ptr(), 2, 8, None, 1, None, _lib.stream()))


# ---- 2. loops: a seed sweep's job files equal the separate runs of its seeds -------------------------------------------------------
SMALL = ['env=hopper', 'steps=60', 'training.start=20', 'evaluation.interval=30', 'evaluation.episodes=1', 'logging.interval=20', 'imitation.trajectories=2',
         'memory.size=100', 'training.batch_size=32', 'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'cuda_graphs=true']
CASES = {
    'gail_tf32x3_gp_mixup': ['algorithm=GAIL', 'gemm_mode=tf32x3', 'imitation.grad_penalty=1', 'imitation.loss_function=Mixup', 'imitation.mixup_alpha=0.5'],
    'gail_general': ['algorithm=GAIL', 'imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh'],
    'sac': ['algorithm=SAC'],
    'adril': ['algorithm=AdRIL', 'imitation.update_freq=25'],
    'pwil_prefill': ['algorithm=PWIL', 'imitation.mix_expert_data=prefill_memory'],
    'gmmil': ['algorithm=GMMIL'],
    'red': ['algorithm=RED', 'imitation.pretraining.iterations=5', 'imitation.discriminator.dropout=0.2'],
    'dril': ['algorithm=DRIL', 'imitation.pretraining.iterations=5'],
    'bc': ['algorithm=BC', 'bc_pretraining.iterations=12'],
}
FILES = ('agent.pth', 'discriminator.pth', 'metrics.pth')


def _same(a, b, where=''):
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


def _sweep(tmp_path, overrides, capsys):
  from il_b200.train import main
  out = str(tmp_path / 'sweep')
  main(['-m'] + overrides + [f'output_dir={out}'])
  assert 'in 1 group(s)' in capsys.readouterr().out
  (run, ) = glob.glob(os.path.join(out, '*_sweeper', '*'))
  return {int(j): _load(os.path.join(run, j)) for j in os.listdir(run)}


@pytest.mark.parametrize('case', list(CASES))
def test_seed_sweep_jobs_equal_the_runs_of_their_seeds(case, tmp_path, capsys):
  seeds = [2, 9, 123456789]
  base = CASES[case] + SMALL
  jobs = _sweep(tmp_path, base + ['seed=' + ','.join(map(str, seeds))], capsys)
  assert sorted(jobs) == [0, 1, 2]
  for j, s in enumerate(seeds):
    ref = _single(tmp_path, f'seed{s}', base + [f'seed={s}'])
    assert set(jobs[j]) == set(ref) and 'agent.pth' in ref and 'metrics.pth' in ref
    assert ('discriminator.pth' in ref) == (case in ('gail_tf32x3_gp_mixup', 'gail_general', 'red', 'dril'))
    _same(jobs[j], ref, f'{case} seed {s}')
  # different seeds train differently (the keyed streams are not one stream)
  assert not torch.equal(jobs[0]['agent.pth']['actor']['actor.0.weight'], jobs[1]['agent.pth']['actor']['actor.0.weight'])


def test_replica_k_of_a_seed_sweep_job_is_the_run_of_seed_plus_k(tmp_path, capsys):
  base = CASES['gail_tf32x3_gp_mixup'] + SMALL
  jobs = _sweep(tmp_path, base + ['replicas=2', 'seed=4,20'], capsys)
  for j, s in enumerate((4, 20)):
    got = jobs[j]
    for k in range(2):
      ref = _single(tmp_path, f'seed{s + k}', base + [f'seed={s + k}'])
      for part in ('actor', 'critic'):
        _same({n: v[k] for n, v in got['agent.pth'][part].items()}, ref['agent.pth'][part], f'job {j} replica {k} {part}')
      _same(got['agent.pth']['log_alpha'][k:k + 1], ref['agent.pth']['log_alpha'], f'job {j} replica {k} log_alpha')
      _same({n: v[k] for n, v in got['discriminator.pth'].items()}, ref['discriminator.pth'], f'job {j} replica {k} discriminator')
      m, mr = got['metrics.pth'], ref['metrics.pth']
      _same([t[k] for t in m['test_returns']], mr['test_returns'], f'job {j} replica {k} test_returns')
      _same(m['train_returns'][k:k + 1], mr['train_returns'], f'job {j} replica {k} train_returns')


def test_seed_sweep_crossed_with_a_learning_rate_sweep_is_one_group_of_single_runs(tmp_path, capsys):
  base = CASES['sac'] + SMALL
  jobs = _sweep(tmp_path, base + ['seed=3,8', 'training.learning_rate=1e-4,3e-4'], capsys)
  assert sorted(jobs) == [0, 1, 2, 3]
  for j, (s, lr) in enumerate((s, lr) for s in (3, 8) for lr in ('1e-4', '3e-4')):
    _same(jobs[j], _single(tmp_path, f'seed{s}_lr{lr}', base + [f'seed={s}', f'training.learning_rate={lr}']), f'job {j}')
