"""Seed sweeps without a GPU: in the programs a multirun runs (config.sweep_groups) `seed` is a per-replica key, except with device_rng false and
with an expert memory subsampled from the seeded numpy stream; group_jobs keeps its one-seed-per-program partition; job j's replica k takes
seed s_j + k; equal seeds collapse to the scalar config; seeds that are not non-negative integers, and per-replica seeds with fast_init, are
refused."""
import pytest

from il_b200.config import (PER_REPLICA_SEED, SweepError, expand_sweep, group_jobs, load_config, per_replica_keys, replica_values, seed_per_replica, split_per_replica,
                            sweep_groups, vectorised_keys)


def test_seed_splits_group_jobs_but_not_the_sweep_programs():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'seed=1,2', 'env=hopper,walker2d', 'training.learning_rate=1e-4,3e-4'])
  groups = group_jobs(jobs)  # one seed per program
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1], [2, 3], [4, 5], [6, 7]]
  assert all(g.per_job == {'training.learning_rate': [1e-4, 3e-4]} for g in groups)
  groups = sweep_groups(jobs)  # env groups, seed and learning rate per replica
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1, 4, 5], [2, 3, 6, 7]]
  assert all(g.per_job == {'seed': [1, 1, 2, 2], 'training.learning_rate': [1e-4, 3e-4] * 2} for g in groups)
  assert 'seed' not in vectorised_keys(load_config(['algorithm=GAIL'])) and 'seed' in per_replica_keys(load_config(['algorithm=GAIL']))


@pytest.mark.parametrize('alg', ['GAIL', 'SAC', 'AdRIL', 'PWIL', 'GMMIL', 'RED', 'DRIL', 'BC'])
def test_seed_sweep_is_one_group(alg):
  _, jobs = expand_sweep(['-m', f'algorithm={alg}', 'seed=1,2,3'])
  (g, ) = sweep_groups(jobs)
  assert [j.num for j in g.jobs] == [0, 1, 2] and g.per_job == {'seed': [1, 2, 3]}


def test_seed_crossed_with_a_hyper_parameter_grid_is_one_group():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'optimised_hyperparameters=GAIL_5_trajectories', 'seed=1,2,3,4,5', 'imitation.learning_rate=1e-5,3e-5'])
  (g, ) = sweep_groups(jobs)
  assert len(g.jobs) == 10
  assert g.per_job == {'seed': [s for s in (1, 2, 3, 4, 5) for _ in range(2)], 'imitation.learning_rate': [1e-5, 3e-5] * 5}


def test_seed_stays_a_grouping_key_with_host_index_draws():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'device_rng=false', 'seed=1,2'])
  groups = sweep_groups(jobs)
  assert len(groups) == 2 and all(g.per_job == {} for g in groups)
  assert 'seed' not in per_replica_keys(load_config(['algorithm=GAIL', 'device_rng=false']))


def test_seed_stays_a_grouping_key_with_a_subsampled_expert_memory():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.subsample=2', 'seed=1,2'])
  assert len(sweep_groups(jobs)) == 2
  # SAC builds no expert memory unless it pre-trains or uses the BC auxiliary loss: subsampling draws nothing there
  assert seed_per_replica(load_config(['algorithm=SAC', 'imitation.subsample=2']))
  assert not seed_per_replica(load_config(['algorithm=SAC', 'imitation.subsample=2', 'bc_pretraining.iterations=10']))
  assert not seed_per_replica(load_config(['algorithm=SAC', 'imitation.subsample=2', 'imitation.bc_aux_loss=true']))
  with pytest.raises(SweepError, match='cannot take per-replica values'):
    split_per_replica(load_config(['algorithm=GAIL', 'imitation.subsample=2']), {'seed': [1, 2]}, 2)


def test_seeds_expand_to_s_plus_k_per_replica():
  assert replica_values('seed', [10, 20], 2) == [10, 11, 20, 21]
  assert replica_values('seed', [3, 7, 5], 1) == [3, 7, 5]
  assert replica_values('training.learning_rate', [1e-4, 3e-4], 2) == [1e-4, 1e-4, 3e-4, 3e-4]  # other keys repeat per replica


def test_equal_seeds_fall_back_to_the_scalar_config():
  cfg = load_config(['algorithm=GAIL'])
  out, arrays = split_per_replica(cfg, {'seed': [4, 4, 4]}, 3)
  assert arrays == {} and out.seed == 4 and cfg.seed == 0
  out, arrays = split_per_replica(cfg, {'seed': [4, 5, 9]}, 3)
  assert arrays == {'seed': [4, 5, 9]} and all(type(s) is int for s in arrays['seed'])
  assert PER_REPLICA_SEED == ('seed', )


@pytest.mark.parametrize('vals,match', [([1, 2.5], r'seed=2.5'), ([-1, 2], r'seed=-1'), ([True, 2], r'seed=True'), ([1, 'x'], r"seed='x'"), ([1, 2**32], r'seed=4294967296')])
def test_split_per_replica_refuses_seeds_that_are_not_non_negative_integers(vals, match):
  with pytest.raises(SweepError, match=match):
    split_per_replica(load_config(['algorithm=GAIL']), {'seed': vals}, 2)


@pytest.mark.parametrize('value', ['1.5', '-3', 'true'])
def test_sweep_refuses_bad_seeds_before_expanding_them(value):
  _, jobs = expand_sweep(['-m', 'algorithm=SAC', f'seed=1,{value}'])
  (g, ) = sweep_groups(jobs)
  with pytest.raises(SweepError, match='seed='):
    replica_values('seed', g.per_job['seed'], 2)


def test_fast_init_refuses_per_replica_seeds():
  from il_b200.train import Trainer
  with pytest.raises(SweepError, match='fast_init'):
    Trainer(load_config(['algorithm=SAC', 'replicas=2']), replicas=2, fast_init=True, per_replica={'seed': [1, 2]})
