"""RED's and DRIL's dropout rates and activation in multirun sweeps, without a GPU: in the programs a multirun runs (config.sweep_groups) they are
per-replica keys, grouped only on whether each dropout site exists; config.group_jobs keeps them as grouping keys; values the reference refuses,
and a mix of present and absent sites, are refused. The six tuned RED / DRIL overlays load with the reference's values."""
import os

import pytest
import yaml

from il_b200.config import (PER_REPLICA_DROPOUT, SweepError, expand_sweep, group_jobs, load_config, per_replica_keys, replica_values, split_per_replica, sweep_groups,
                            vectorised_keys)
from oracle import ref_overlays

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GRID = ['imitation.discriminator.input_dropout=0.1,0.3', 'imitation.discriminator.dropout=0.2,0.5', 'imitation.discriminator.activation=relu,tanh']
IN, DROP, ACT = PER_REPLICA_DROPOUT


@pytest.mark.parametrize('alg', ['DRIL', 'RED'])
def test_rate_activation_grid_is_one_group_in_hydra_order(alg):
  extra = ['imitation.quantile_cutoff=0.8,0.95'] if alg == 'DRIL' else []
  _, jobs = expand_sweep(['-m', f'algorithm={alg}', *GRID, *extra])
  J = 16 if alg == 'DRIL' else 8
  assert len(jobs) == J
  (g, ) = sweep_groups(jobs)
  assert [j.num for j in g.jobs] == list(range(J))
  assert set(g.per_job) == set(PER_REPLICA_DROPOUT) | ({'imitation.quantile_cutoff'} if alg == 'DRIL' else set())
  rep = J // 8  # the last key varies fastest (Hydra's basic sweeper)
  assert g.per_job[IN] == [x for x in (0.1, 0.3) for _ in range(4 * rep)]
  assert g.per_job[DROP] == [x for _ in range(2) for x in (0.2, 0.5) for _ in range(2 * rep)]
  assert g.per_job[ACT] == [x for _ in range(4) for x in ('relu', 'tanh') for _ in range(rep)]
  if alg == 'DRIL': assert g.per_job['imitation.quantile_cutoff'] == [0.8, 0.95] * 8


@pytest.mark.parametrize('alg', ['DRIL', 'RED'])
def test_group_jobs_still_splits_on_the_dropout_keys(alg):
  _, jobs = expand_sweep(['-m', f'algorithm={alg}', *GRID])
  groups = group_jobs(jobs)
  assert len(groups) == 8 and all(len(g.jobs) == 1 and g.per_job == {} for g in groups)
  assert not set(PER_REPLICA_DROPOUT) & set(vectorised_keys(load_config([f'algorithm={alg}'])))


@pytest.mark.parametrize('alg', ['DRIL', 'RED'])
def test_presence_of_a_dropout_site_splits_groups(alg):
  _, jobs = expand_sweep(['-m', f'algorithm={alg}', 'imitation.discriminator.input_dropout=0,0.3', 'imitation.learning_rate=1e-4,3e-4'])
  groups = sweep_groups(jobs)
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1], [2, 3]]
  # the rate stays a per-job value (equal within each group: the scalar path)
  assert [g.per_job for g in groups] == [{IN: [0, 0], 'imitation.learning_rate': [1e-4, 3e-4]}, {IN: [0.3, 0.3], 'imitation.learning_rate': [1e-4, 3e-4]}]
  _, jobs = expand_sweep(['-m', f'algorithm={alg}', 'imitation.discriminator.dropout=0,0.2,0.5'])
  groups = sweep_groups(jobs)
  assert [[j.num for j in g.jobs] for g in groups] == [[0], [1, 2]]
  assert [g.per_job for g in groups] == [{DROP: [0]}, {DROP: [0.2, 0.5]}]


def test_dril_activation_needs_a_dropout_site():
  no_drop = ['algorithm=DRIL', 'imitation.discriminator.input_dropout=0', 'imitation.discriminator.dropout=0']
  assert ACT not in per_replica_keys(load_config(no_drop)) and ACT in per_replica_keys(load_config(['algorithm=DRIL']))
  assert ACT in per_replica_keys(load_config(['algorithm=RED']))  # RED always runs on the dropout program
  _, jobs = expand_sweep(['-m', *no_drop, 'imitation.discriminator.activation=relu,tanh'])
  assert len(sweep_groups(jobs)) == 2


def test_gail_ignores_the_dropout_keys_and_refuses_per_replica_activation():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.input_dropout=0,0.5', 'imitation.discriminator.dropout=0.25,0.75'])
  (g, ) = sweep_groups(jobs)
  assert len(g.jobs) == 4 and g.per_job == {}
  assert not set(PER_REPLICA_DROPOUT) & set(per_replica_keys(load_config(['algorithm=GAIL'])))
  with pytest.raises(SweepError, match='cannot take per-replica values'):
    split_per_replica(load_config(['algorithm=GAIL']), {ACT: ['relu', 'tanh']}, 2)


def test_per_job_values_expand_to_replica_blocks_and_equal_values_collapse():
  assert replica_values(DROP, [0.2, 0.5], 3) == [0.2, 0.2, 0.2, 0.5, 0.5, 0.5]
  assert replica_values(ACT, ['relu', 'tanh'], 2) == ['relu', 'relu', 'tanh', 'tanh']
  cfg, arrays = split_per_replica(load_config(['algorithm=RED']), {IN: [0.3, 0.3], DROP: [0.2, 0.5], ACT: ['tanh', 'tanh']}, 2)
  assert arrays == {DROP: [0.2, 0.5]}
  assert cfg.imitation.discriminator.input_dropout == 0.3 and cfg.imitation.discriminator.activation == 'tanh'
  _, arrays = split_per_replica(load_config(['algorithm=DRIL']), {ACT: ['relu', 'sigmoid', 'tanh'], IN: [0.1, 0.25, 0.499]}, 3)
  assert arrays == {ACT: ['relu', 'sigmoid', 'tanh'], IN: [0.1, 0.25, 0.499]}


@pytest.mark.parametrize('alg,key,vals,match', [
    ('RED', IN, [0, 0.3], r'mix rate 0 and rate > 0'),
    ('DRIL', DROP, [0.2, 0], r'mix rate 0 and rate > 0'),
    ('RED', DROP, [0.2, 1], r'replica 1: .*=1: not in \[0, 1\)'),
    ('DRIL', IN, [1.5, 0.1], r'replica 0: .*=1.5: not in \[0, 1\)'),
    ('RED', IN, [-0.1, 0.1], r'replica 0: .*not in \[0, 1\)'),
    ('DRIL', DROP, [0.2, 'x'], r'replica 1: .*not a number'),
    ('RED', DROP, [True, 0.2], r'replica 0: .*not a number'),
    ('RED', ACT, ['relu', 'elu'], r'replica 1: .*elu.*not one of relu, sigmoid, tanh'),
    ('DRIL', ACT, ['gelu', 'tanh'], r'replica 0: .*not one of'),
])
def test_refusals(alg, key, vals, match):
  with pytest.raises(SweepError, match=match):
    split_per_replica(load_config([f'algorithm={alg}']), {key: vals}, len(vals))


def test_every_sweep_group_passes_split_per_replica():
  _, jobs = expand_sweep(['-m', 'algorithm=RED', 'imitation.discriminator.input_dropout=0,0.3,0.4', 'imitation.discriminator.activation=relu,sigmoid'])
  for g in sweep_groups(jobs):  # each group is homogeneous in presence, so split_per_replica accepts it
    split_per_replica(load_config(g.overrides), {k: replica_values(k, v, 1) for k, v in g.per_job.items()}, len(g.jobs))


@pytest.mark.parametrize('name', ref_overlays.NAMES)
def test_tuned_overlay_loads_with_the_reference_values(name):
  theirs = {k: v for k, v in ref_overlays.load()[name].items() if not k.startswith(('defaults', 'hydra'))}
  with open(os.path.join(ROOT, 'conf', 'optimised_hyperparameters', f'{name}.yaml')) as f: raw = yaml.safe_load(f)

  def flat(d, prefix=''):
    out = {}
    for k, v in d.items():
      if isinstance(v, dict): out.update(flat(v, f'{prefix}{k}.'))
      else: out[prefix + k] = v
    return out
  assert flat(raw) == theirs
  alg = name.split('_')[0]
  cfg = load_config([f'algorithm={alg}', f'optimised_hyperparameters={name}'])
  for k, v in theirs.items():
    node = cfg
    for p in k.split('.'): node = node[p]
    assert node == v and type(node) is type(v), (k, node, v)
