"""Checkpoint and resume on the GPU (checkpoint.interval, `train.py resume=`, `train_all.py resume=`): a run interrupted right after its
checkpoint at step t and resumed in a fresh process writes the files of the run that was never interrupted, bit for bit (every tensor equal,
every list exactly, all but the training_time value); the same for a multirun interrupted in its second group and a search interrupted in its
second round; and a census that every device tensor a Trainer holds is either checkpointed or named here as scratch or set-up."""
import fnmatch
import glob
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FILES = ('agent.pth', 'discriminator.pth', 'metrics.pth', 'trajectories.pth')
# 48 steps, updates from step 16, an evaluation every 16 steps and a checkpoint every 8
BASE = ['env=hopper', 'steps=48', 'training.start=16', 'training.batch_size=32', 'imitation.trajectories=2', 'reinforcement.actor.hidden_size=32',
        'reinforcement.critic.hidden_size=32', 'replicas=3', 'seed=5', 'evaluation.interval=16', 'evaluation.episodes=2', 'logging.interval=8', 'gemm_mode=fp32',
        'save_trajectories=true', 'imitation.pretraining.iterations=20']
CASES = [('SAC', ['algorithm=SAC'], 24),
         ('GAIL-fused', ['algorithm=GAIL'], 24),
         ('GAIL-general', ['algorithm=GAIL', 'imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh', 'imitation.loss_function=Mixup'], 24),
         ('GMMIL', ['algorithm=GMMIL'], 24),
         ('PWIL-none', ['algorithm=PWIL', 'imitation.mix_expert_data=none'], 24),
         ('PWIL-prefill', ['algorithm=PWIL', 'imitation.mix_expert_data=prefill_memory'], 24),
         ('AdRIL-balanced', ['algorithm=AdRIL', 'imitation.balanced=true', 'imitation.update_freq=20'], 24),
         ('RED', ['algorithm=RED'], 24),
         ('DRIL', ['algorithm=DRIL'], 24),
         ('SAC-bc', ['algorithm=SAC', 'bc_pretraining.iterations=10', 'imitation.bc_aux_loss=true'], 24),
         ('host-rng', ['algorithm=GAIL', 'device_rng=false'], 24),
         ('ring-wrapped', ['algorithm=GMMIL', 'memory.size=20'], 24),
         ('before-start', ['algorithm=GAIL'], 8),
         ('at-evaluation', ['algorithm=GAIL'], 32),
         ('time-usage', ['algorithm=SAC', 'check_time_usage=true'], 24)]


def _same(x, y, path):
  if isinstance(x, dict):
    assert set(x) == set(y), f'{path}: keys {sorted(set(x) ^ set(y))}'
    for k in x:
      if k != 'training_time': _same(x[k], y[k], f'{path}.{k}')
  elif isinstance(x, (list, tuple)):
    assert type(x) is type(y) and len(x) == len(y), f'{path}: length {len(x)} vs {len(y)}'
    for i, (a, b) in enumerate(zip(x, y)): _same(a, b, f'{path}[{i}]')
  elif torch.is_tensor(x):
    assert torch.is_tensor(y) and x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y), f'{path}: tensors differ'
  elif isinstance(x, np.ndarray):
    assert isinstance(y, np.ndarray) and x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y, equal_nan=True), f'{path}: arrays differ'
  elif isinstance(x, float) and math.isnan(x):
    assert isinstance(y, float) and math.isnan(y), f'{path}: {x} vs {y}'
  else:
    assert type(x) is type(y) and x == y, f'{path}: {x!r} vs {y!r}'


def _same_files(a, b, outputs=None):
  """outputs: (a's output_dir, b's): the command lines recorded in overrides.yaml differ in it and nothing else."""
  for name in FILES:
    fa, fb = os.path.join(a, name), os.path.join(b, name)
    assert os.path.exists(fa) == os.path.exists(fb), name
    if os.path.exists(fa): _same(torch.load(fa, weights_only=False), torch.load(fb, weights_only=False), name)
  if os.path.exists(os.path.join(a, 'overrides.yaml')):
    text_b = open(os.path.join(b, 'overrides.yaml')).read()
    assert open(os.path.join(a, 'overrides.yaml')).read() == (text_b.replace(outputs[1], outputs[0]) if outputs else text_b)


def _python(args, timeout=900):
  r = subprocess.run([sys.executable, *args], cwd=ROOT, capture_output=True, text=True, timeout=timeout)
  assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
  return r.stdout


@pytest.mark.parametrize('name,extra,t', CASES, ids=[c[0] for c in CASES])
def test_resumed_run_writes_the_files_of_the_uninterrupted_run(tmp_path, name, extra, t):
  from il_b200 import checkpoint
  from il_b200.config import load_config
  from il_b200.train import _train
  args = BASE + extra
  a, b = tmp_path / 'a', tmp_path / 'b'
  a.mkdir()
  b.mkdir()
  _train(load_config(args), [(str(a) + os.sep, '', None, None)])  # never interrupted, no checkpoints
  assert _train(load_config(args + ['checkpoint.interval=8']), [(str(b) + os.sep, '', None, None)], checkpoint_dir=str(b / 'checkpoint'), overrides=args, stop_at=t) is None
  assert checkpoint.latest(str(b / 'checkpoint')) == str(b / 'checkpoint' / f'step{t}') and not (b / 'metrics.pth').exists()
  assert sorted(os.listdir(b / 'checkpoint')) == ['LATEST', f'step{t}']
  out = _python(['train.py', f'resume={b}'])  # a fresh process
  assert f'resuming at step {t + 1}' in out
  _same_files(str(a), str(b))


# ---- census ------------------------------------------------------------------------------------------------------------------------
# Device tensors that need no checkpoint, by what they are: rewritten before every read, or rebuilt by the constructor
SCRATCH = {
    'workspaces': ['*._ws', '*._ws_cache.*', '*._ws_retired.*', 'trainer.actor_ws', '*._drop_ws'],
    'sampled batches': ['trainer.batch.rows', 'trainer.expert_batch.rows'],
    'noise buffers': ['trainer.' + n for n in ('eps_act', 'u_reset', 'u_pol', 'u_exp', 'eps_gp', 'eps_mix', 'eps_next', 'eps_new')],
    'index buffers': ['trainer.idx_pol', 'trainer.idx_exp'],
    'step outputs': ['trainer.' + n for n in ('action', 'env_reward', 'store_reward', 'done', 'timeout', 'terminal_f', 'timeout_f', 'gail_losses')] + ['trainer.sac_out.*'],
    'eval buffers': ['*._eval_states.*', '*._eval_batches.*', '*.env._state', '*.env._reward', '*.env._done', '*.eval_env.*'],
    'set-up constants': ['*.params.*', '*.batch.p.*', '*expert_memory.rows', '*expert_memory._idx', '*expert_memory._full', '*expert_memory._num_trajectories', '*._seed_r',
                         '*.seed_r', '*.lr_r', '*.weight_decay_r', 'trainer.discount', 'trainer.polyak_factor', 'trainer.entropy_target', 'trainer.mixup_alpha',
                         'trainer.gail_penalty_pass', 'trainer.imitation_cfg.*', '*._choice_cache.*', '*._choices.*', '*._reward_function_r', '*._spectral_norm_r',
                         '*._replica_order', '*._update_freq_r', '*._balanced_r', 'trainer.discriminator.atoms', 'trainer.discriminator.data_scale',
                         'trainer.discriminator.data_offset', 'trainer.discriminator.reward_scale_r', 'trainer.discriminator.reward_bandwidth_r',
                         'trainer.discriminator.discount'],
}


def _walk(obj, path, seen, out):
  if id(obj) in seen: return
  seen.add(id(obj))
  if torch.is_tensor(obj):
    if obj.is_cuda: out.append((path, obj))
  elif isinstance(obj, dict):
    for k, v in obj.items(): _walk(v, f'{path}.{k}', seen, out)
  elif isinstance(obj, (list, tuple)):
    for i, v in enumerate(obj): _walk(v, f'{path}.{i}', seen, out)
  elif type(obj).__module__.startswith('il_b200') and hasattr(obj, '__dict__'):
    for k, v in vars(obj).items(): _walk(v, f'{path}.{k}', seen, out)


@pytest.mark.parametrize('algorithm,extra', [('SAC', ['imitation.bc_aux_loss=true']), ('GAIL', []), ('GAIL', ['imitation.discriminator.depth=2', 'imitation.spectral_norm=true']),
                                             ('GAIL', ['imitation.discriminator.reward_shaping=true']), ('GMMIL', []), ('PWIL', []), ('AdRIL', []),
                                             ('RED', ['imitation.discriminator.dropout=0.2']), ('DRIL', []), ('SAC', ['device_rng=false'])])
def test_every_device_tensor_is_checkpointed_or_named_scratch(algorithm, extra):
  from il_b200.config import load_config
  from il_b200.train import Trainer
  tr = Trainer(load_config(BASE + [f'algorithm={algorithm}'] + extra))
  if algorithm in ('RED', 'DRIL'): tr.pretrain_discriminator()
  for _ in range(20): tr.train_step()
  tr.evaluate()
  state = {t.untyped_storage().data_ptr() for t in tr._state_tensors().values()}
  found = []
  _walk(tr, 'trainer', set(), found)
  patterns = [p for ps in SCRATCH.values() for p in ps]
  loose = [p for p, t in found if t.untyped_storage().data_ptr() not in state and not any(fnmatch.fnmatchcase(p, q) for q in patterns)]
  assert not loose, f'device tensors neither in checkpoint_state() nor named scratch: {loose}'
  assert len(found) > len(state)


# ---- multirun and search --------------------------------------------------------------------------------------------------------
STOPPER = r"""
import sys
sys.path.insert(0, {root!r})
import il_b200, il_b200.train as T
real, calls = T._train, []
def stop_in(*a, **k):  # the {nth}th program whose checkpoint directory names {where!r} stops after its checkpoint at step {t}
  if {where!r} in (k.get('checkpoint_dir') or ''): calls.append(1)
  if len(calls) == {nth}:
    assert real(*a, stop_at={t}, **k) is None
    raise SystemExit(3)
  return real(*a, **k)
T._train = stop_in
from il_b200 import hpo
(hpo.main if {search} else T.main)(sys.argv[1:])
"""


def _interrupted(tmp_path, argv, where, nth, t, search=False):
  script = tmp_path / 'stop.py'
  script.write_text(STOPPER.format(root=ROOT, where=where, nth=nth, t=t, search=search))
  r = subprocess.run([sys.executable, str(script), *argv], cwd=ROOT, capture_output=True, text=True, timeout=900)
  assert r.returncode == 3, r.stdout[-3000:] + r.stderr[-3000:]


def _scores(text, outputs=None):
  """The closing per-job score lines; outputs: (a's output_dir, this sweep's), the one override the two sweeps' command lines differ in."""
  lines = [l for l in text.splitlines() if l.startswith('job ') and ': score ' in l]
  return [l.replace(outputs[1], outputs[0]) for l in lines] if outputs else lines


def test_resumed_sweep_equals_the_uninterrupted_sweep(tmp_path):
  argv = ['-m', 'algorithm=SAC', 'env=hopper,walker2d', 'seed=1,2', 'training.learning_rate=0.001,0.0003'] + [a for a in BASE if not a.startswith(('env=', 'seed='))] + \
         ['checkpoint.interval=8']
  a, b = tmp_path / 'a', tmp_path / 'b'
  full = _python(['train.py', *argv, f'output_dir={a}'])
  _interrupted(tmp_path, argv + [f'output_dir={b}'], 'group1', 1, 16)
  (run_a, ), (run_b, ) = glob.glob(str(a / '*_sweeper' / '*')), glob.glob(str(b / '*_sweeper' / '*'))
  assert os.path.isfile(os.path.join(run_b, 'checkpoint', 'group1', 'step16', 'rank0.pt'))
  resumed = _python(['train.py', f'resume={run_b}'])
  assert 'finished before the resume' in resumed and 'resuming at step 17' in resumed
  jobs = sorted(d for d in os.listdir(run_a) if d.isdigit())
  assert jobs == sorted(d for d in os.listdir(run_b) if d.isdigit()) and len(jobs) == 8
  for j in jobs: _same_files(os.path.join(run_a, j), os.path.join(run_b, j), (str(a), str(b)))
  assert _scores(full) == _scores(resumed, (str(a), str(b))) and len(_scores(full)) == 8
  assert not os.path.exists(os.path.join(run_b, 'checkpoint', 'group1')), 'a finished group leaves no checkpoint behind'


def test_resumed_search_equals_the_uninterrupted_search(tmp_path):
  short = ['steps=32', 'evaluation.interval=16', 'evaluation.episodes=1', 'logging.interval=8', 'imitation.trajectories=2', 'memory.size=100',
           'reinforcement.actor.hidden_size=32', 'reinforcement.critic.hidden_size=32', 'training.start=8', 'training.batch_size=32', 'gemm_mode=fp32']
  argv = ['-m', 'algorithm=SAC'] + short + ['hpo.max_trials=4', 'hpo.initial=2', 'hpo.batch=2', 'hpo.candidates=1024', 'checkpoint.interval=8']
  a, b = tmp_path / 'a', tmp_path / 'b'
  _python(['train_all.py', *argv, f'output_dir={a}'])
  _interrupted(tmp_path, argv + [f'output_dir={b}'], 'round1', 2, 24, search=True)
  (run_a, ), (run_b, ) = glob.glob(str(a / '*_all_sweeper' / '*')), glob.glob(str(b / '*_all_sweeper' / '*'))
  with open(os.path.join(run_b, 'hpo.json')) as f: assert len(json.load(f)['rounds']) == 1
  _python(['train_all.py', f'resume={run_b}'])
  with open(os.path.join(run_a, 'hpo.json')) as f: want = json.load(f)
  with open(os.path.join(run_b, 'hpo.json')) as f: got = json.loads(f.read().replace(str(b), str(a)))  # the output_dir override
  _same(want, got, 'hpo.json')  # the record holds no wall-clock field
  for trial in range(4):
    for env in want['envs']: _same_files(os.path.join(run_a, str(trial), env), os.path.join(run_b, str(trial), env))


# ---- two ranks ----------------------------------------------------------------------------------------------------------------------
TWO_RANK = r"""
import os, sys
sys.path.insert(0, {root!r})
import il_b200
from il_b200 import distributed
from il_b200.config import load_config
from il_b200.train import _train
args = {args!r}
out = sys.argv[1]
if sys.argv[2] == 'full': _train(load_config(args), [(out + os.sep, '', None, None)])
else: assert _train(load_config(args + ['checkpoint.interval=8']), [(out + os.sep, '', None, None)], checkpoint_dir=os.path.join(out, 'checkpoint'), overrides=args, stop_at=24) is None
distributed.shutdown()
"""


@pytest.mark.timeout(900)
def test_two_rank_resume(tmp_path):
  if torch.cuda.device_count() < 2: pytest.skip('needs 2 GPUs')
  script = tmp_path / 'two.py'
  script.write_text(TWO_RANK.format(root=ROOT, args=BASE + ['algorithm=GAIL', 'replicas=4']))
  run = lambda *a: _python(['-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr', '127.0.0.1', '--master-port', '29733', *a])
  a, b = tmp_path / 'a', tmp_path / 'b'
  a.mkdir()
  b.mkdir()
  run(str(script), str(a), 'full')
  run(str(script), str(b), 'stop')
  assert sorted(os.listdir(b / 'checkpoint' / 'step24')) == ['meta.json', 'rank0.pt', 'rank1.pt']
  run('train.py', f'resume={b}')
  _same_files(str(a), str(b))
  for k in (1, ):
    _same(torch.load(a / f'trajectories.rank{k}.pth', weights_only=False), torch.load(b / f'trajectories.rank{k}.pth', weights_only=False), f'trajectories.rank{k}')
