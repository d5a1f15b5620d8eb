"""Checkpoint files and resume plans without a GPU (il_b200/checkpoint.py): checkpoint.interval validation, the refusals of `resume=`,
atomic saves, and the per-group plan of a resumed multirun and the per-env plan of a resumed search."""
import json
import os

import pytest
import torch
import yaml

import il_b200
from il_b200 import checkpoint, hpo
from il_b200.checkpoint import CheckpointError
from il_b200.config import load_config
from il_b200.train import resume

V = 100  # a library version for the files these tests write


def _save(d, step, value, version=V, meta=None):
  checkpoint.save(d, step, dict(x=torch.full((4, ), float(value))), meta or dict(config=dict(seed=0), overrides=[]), version=version)


@pytest.mark.parametrize('value,want', [(None, 0), (0, 0), (1, 1), (250, 250)])
def test_interval_accepts_integers_from_zero(value, want):
  cfg = load_config(['algorithm=SAC'] + ([] if value is None else [f'checkpoint.interval={value}']))
  assert checkpoint.interval_of(cfg) == want


@pytest.mark.parametrize('value', ['-1', '2.5', 'true', 'abc', '[1,2]'])
def test_interval_refuses_anything_else(value):
  with pytest.raises(CheckpointError, match='checkpoint.interval'):
    checkpoint.interval_of(load_config(['algorithm=SAC', f'checkpoint.interval={value}']))


def test_interval_leaves_the_loaded_config_as_it_was():
  """checkpoint.interval is read with cfg.get: it is not in conf/train_config.yaml, so load_config returns the same tree as before for any
  command line without it."""
  assert 'checkpoint' not in load_config(['algorithm=GAIL', 'env=hopper'])


def test_save_then_load_round_trips(tmp_path):
  d = str(tmp_path / 'ck')
  _save(d, 8, 1.0, meta=dict(config=dict(seed=3), overrides=['seed=3'], replicas=2))
  meta, state = checkpoint.load(d, version=V)
  assert meta['step'] == 8 and meta['world_size'] == 1 and meta['il_version'] == V and meta['config'] == dict(seed=3) and meta['replicas'] == 2
  assert set(meta['files']) == {'rank0.pt'} and meta['files']['rank0.pt']['bytes'] == os.path.getsize(os.path.join(d, 'step8', 'rank0.pt'))
  assert torch.equal(state['x'], torch.full((4, ), 1.0))
  _save(d, 16, 2.0)
  assert sorted(os.listdir(d)) == ['LATEST', 'step16'], 'the older step directory is deleted once LATEST names the new one'
  assert float(checkpoint.load(d, version=V)[1]['x'][0]) == 2.0


def test_two_rank_checkpoint_keeps_one_file_per_rank(tmp_path):
  import threading
  d, barrier = str(tmp_path / 'ck'), threading.Barrier(2)
  ranks = [threading.Thread(target=checkpoint.save, args=(d, 4, dict(x=torch.full((4, ), 5.0 + k)), dict(config={}, overrides=[]), k, 2, V, barrier.wait)) for k in (0, 1)]
  for t in ranks: t.start()
  for t in ranks: t.join()
  meta, s1 = checkpoint.load(d, rank=1, world=2, version=V)
  assert set(meta['files']) == {'rank0.pt', 'rank1.pt'} and float(s1['x'][0]) == 6.0
  with pytest.raises(CheckpointError, match='2 rank'):
    checkpoint.load(d, rank=0, world=1, version=V)


def test_a_save_killed_halfway_leaves_the_previous_checkpoint(tmp_path, monkeypatch):
  d = str(tmp_path / 'ck')
  _save(d, 8, 1.0)
  real = torch.save

  def half(obj, f, *a, **k):  # writes part of the file, then dies
    f.write(b'\x80\x02partial')
    raise KeyboardInterrupt('killed')
  monkeypatch.setattr(torch, 'save', half)
  with pytest.raises(KeyboardInterrupt):
    _save(d, 16, 2.0)
  monkeypatch.setattr(torch, 'save', real)
  assert os.path.isdir(os.path.join(d, 'step16')), 'the half-written directory is there ...'
  assert checkpoint.latest(d) == os.path.join(d, 'step8'), '... but LATEST still names the complete one'
  meta, state = checkpoint.load(d, version=V)
  assert meta['step'] == 8 and float(state['x'][0]) == 1.0
  _save(d, 16, 2.0)  # the next save replaces the half-written directory
  assert checkpoint.load(d, version=V)[0]['step'] == 16 and sorted(os.listdir(d)) == ['LATEST', 'step16']


def test_a_step_directory_without_latest_is_not_a_checkpoint(tmp_path):
  d = tmp_path / 'ck'
  (d / 'step8').mkdir(parents=True)
  (d / 'step8' / 'rank0.pt').write_bytes(b'x')
  assert checkpoint.latest(str(d)) is None
  with pytest.raises(CheckpointError, match='no checkpoint'):
    checkpoint.load(str(d), version=V)


def _run_dir(tmp_path, version=V):
  run = tmp_path / 'run'
  _save(str(run / 'checkpoint'), 8, 1.0, version=version, meta=dict(config=dict(load_config(['algorithm=SAC'])), overrides=['algorithm=SAC']))
  return str(run)


def test_resume_refuses_other_overrides(tmp_path):
  with pytest.raises(CheckpointError, match='no other override'):
    checkpoint.resume_run_meta(_run_dir(tmp_path), ['steps=10'], version=V)
  with pytest.raises(CheckpointError, match='no other override'):
    resume(_run_dir(tmp_path), ['seed=1'])


def test_resume_refuses_a_missing_directory_or_checkpoint(tmp_path):
  with pytest.raises(CheckpointError, match='no run directory'):
    checkpoint.resume_run_meta(str(tmp_path / 'absent'), [], version=V)
  (tmp_path / 'empty').mkdir()
  with pytest.raises(CheckpointError, match='no checkpoint'):
    checkpoint.resume_run_meta(str(tmp_path / 'empty'), [], version=V)


def test_resume_refuses_another_library_version_or_world_size(tmp_path):
  run = _run_dir(tmp_path, version=V)
  assert checkpoint.resume_run_meta(run, [], version=V)['overrides'] == ['algorithm=SAC']
  with pytest.raises(CheckpointError, match='il_version 100; this build is 101'):
    checkpoint.resume_run_meta(run, [], version=V + 1)
  with pytest.raises(CheckpointError, match='1 rank'):
    checkpoint.resume_run_meta(run, [], world=2, version=V)


def test_resume_refuses_a_corrupted_file(tmp_path):
  run = _run_dir(tmp_path)
  f = os.path.join(run, 'checkpoint', 'step8', 'rank0.pt')
  data = bytearray(open(f, 'rb').read())
  data[len(data) // 2] ^= 0xFF  # same size, one byte flipped
  open(f, 'wb').write(bytes(data))
  with pytest.raises(CheckpointError, match='sha256'):
    checkpoint.load(os.path.join(run, 'checkpoint'), version=V)
  open(f, 'ab').write(b'tail')
  with pytest.raises(CheckpointError, match='size'):
    checkpoint.load(os.path.join(run, 'checkpoint'), version=V)


def test_resume_refusals_are_one_line_on_the_command_line(tmp_path):
  from il_b200.train import main
  with pytest.raises(SystemExit) as e:
    main([f'resume={tmp_path / "absent"}'])
  assert str(e.value).startswith('resume refused: ') and '\n' not in str(e.value)


def _fabricate_sweep(tmp_path, groups, finished, scored, running):
  """A sweep directory: `finished` jobs have metrics.pth, `scored` jobs a score in checkpoint/scores.json, groups in `running` a checkpoint."""
  base = tmp_path / 'sweep'
  for g in groups:
    for j in g:
      (base / str(j)).mkdir(parents=True, exist_ok=True)
      if j in finished: (base / str(j) / 'metrics.pth').write_bytes(b'm')
  checkpoint.write_scores(str(base / 'checkpoint'), {str(j): 0.5 for j in scored})
  for k in running: _save(str(base / 'checkpoint' / f'group{k}'), 8, 1.0)
  return str(base)


def test_sweep_plan_skips_finished_groups_continues_the_interrupted_one_and_runs_the_rest(tmp_path):
  groups = [[0, 1], [2, 3], [4, 5]]
  base = _fabricate_sweep(tmp_path, groups, finished={0, 1}, scored={0, 1}, running=[1])
  assert checkpoint.sweep_plan(base, groups) == ['skip', 'continue', 'run']


def test_sweep_plan_reruns_a_group_whose_outputs_or_scores_are_incomplete(tmp_path):
  # group 0: one job's metrics.pth missing; group 1: files written but killed before its scores were recorded (its checkpoint is still there)
  groups = [[0, 1], [2, 3]]
  base = _fabricate_sweep(tmp_path, groups, finished={0, 2, 3}, scored={0, 1}, running=[1])
  assert checkpoint.sweep_plan(base, groups) == ['run', 'continue']


def test_resume_of_a_sweep_reads_its_command_line(tmp_path, monkeypatch):
  base = tmp_path / 'sweep'
  base.mkdir()
  argv = ['-m', 'algorithm=SAC', 'env=hopper,walker2d', 'checkpoint.interval=8']
  (base / 'multirun.yaml').write_text(yaml.safe_dump(argv))
  seen = {}
  monkeypatch.setattr(il_b200.train, 'run_sweep', lambda jobs, a, resume_dir: seen.update(jobs=jobs, argv=a, dir=resume_dir) or [])
  resume(str(base))
  assert seen['argv'] == argv and seen['dir'] == str(base) and [j.overrides for j in seen['jobs']] == [['algorithm=SAC', f'env={e}', 'checkpoint.interval=8'] for e in ('hopper', 'walker2d')]


def _fabricate_search(tmp_path, finished, scored, running):
  """A search directory in round 1 whose trials 0, 1 run as one program per env: `finished` envs have the trials' metrics.pth, `scored` envs
  their scores in checkpoint/round1/scores.json, `running` a checkpoint."""
  d = tmp_path / 'search'
  root = d / 'checkpoint' / 'round1'
  for env in finished:
    for j in (0, 1):
      (d / str(j) / env).mkdir(parents=True, exist_ok=True)
      (d / str(j) / env / 'metrics.pth').write_bytes(b'm')
  checkpoint.write_scores(str(root), {e: {'0': 0.25, '1': 0.5} for e in scored})
  for env in running: _save(str(root / env / 'group0'), 8, 1.0)
  return str(d)


def test_search_plan_finishes_the_interrupted_round(tmp_path):
  d = _fabricate_search(tmp_path, finished=['ant', 'halfcheetah'], scored=['ant'], running=['halfcheetah'])
  plan = hpo.round_plan(d, 1, {e: [[0, 1]] for e in ('ant', 'halfcheetah', 'hopper', 'walker2d')})
  assert plan == {'ant': ['skip'], 'halfcheetah': ['continue'], 'hopper': ['run'], 'walker2d': ['run']}


def test_search_resume_keeps_the_finished_rounds_of_hpo_json(tmp_path):
  """The completed rounds come back from hpo.json with the best objective after each round and the Sobol points they consumed, so the next
  round is proposed as in the uninterrupted search."""
  base = ['algorithm=SAC']
  h = hpo.load_hpo(['hpo.initial=2', 'hpo.batch=2', 'hpo.max_trials=6'])
  space = hpo.Space.of('SAC', base)
  fresh = dict(algorithm='SAC', overrides=base, hpo=h, envs=['ant', 'halfcheetah', 'hopper', 'walker2d'], searched=[p.key for p in space.params],
               group_keys=[p.key for p in space.group_params], d=space.d, trials=[], rounds=[])
  xs, used = hpo.sobol_round(space, 2, h['seed'], 0, h['max_groups'])
  trials = [dict(trial=i, round=0, x=x.tolist(), objective=o, failed=False) for i, (x, o) in enumerate(zip(xs, (0.25, 0.75)))]
  trials.append(dict(trial=2, round=1, x=xs[0].tolist(), objective=float('nan'), failed=True))
  d = tmp_path / 'search'
  d.mkdir()
  (d / 'hpo.json').write_text(json.dumps(dict(fresh, trials=trials, rounds=[dict(kind='sobol'), dict(kind='gp')])))
  record, best_after, n_sobol = hpo.completed_rounds(str(d), fresh, space, h, 1.0)
  assert record['trials'] == json.loads(json.dumps(trials)) and best_after == [0.75, 0.75] and n_sobol == used
  assert hpo.completed_rounds(str(tmp_path), fresh, space, h, 1.0) == (fresh, [], 0), 'killed in round 0: nothing finished'
  with pytest.raises(CheckpointError, match='hpo'):
    hpo.completed_rounds(str(d), dict(fresh, hpo=dict(h, seed=1)), space, h, 1.0)
