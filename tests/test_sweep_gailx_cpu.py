"""Multirun sweeps over the general GAIL discriminator's choices without a GPU: on a configuration that runs the general discriminator (depth 2,
tanh, reward shaping with the log-policy term), loss function, reward function, spectral norm, prior, margin and grad_penalty are per-replica
keys of sweep_groups (one program), while group_jobs keeps its partition and hidden size, depth and activation still split groups."""
import pytest

from il_b200.config import (PER_REPLICA_GENERAL_DISCRIMINATOR, SweepError, expand_sweep, general_discriminator_keys, group_jobs, load_config, per_replica_keys,
                            split_per_replica, sweep_groups, vectorised_keys)

GRID = ['imitation.loss_function=BCE,Mixup,PUGAIL', 'imitation.discriminator.reward_function=GAIL,AIRL,FAIRL', 'imitation.spectral_norm=true,false',
        'imitation.grad_penalty=0,0.5']
GENERAL = {'depth 2': ['imitation.discriminator.depth=2'], 'tanh': ['imitation.discriminator.activation=tanh'],
           'shaping + log-policy': ['imitation.discriminator.reward_shaping=true', 'imitation.discriminator.subtract_log_policy=true']}


@pytest.mark.parametrize('which', list(GENERAL))
def test_general_choice_grid_is_one_program_in_hydra_order(which):
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', *GENERAL[which], *GRID])
  assert len(jobs) == 36
  (g, ) = sweep_groups(jobs)
  assert [j.num for j in g.jobs] == list(range(36))
  assert set(g.per_job) == {'imitation.loss_function', 'imitation.discriminator.reward_function', 'imitation.spectral_norm', 'imitation.grad_penalty'}
  # the last key varies fastest (Hydra's basic sweeper)
  assert g.per_job['imitation.loss_function'] == [x for x in ('BCE', 'Mixup', 'PUGAIL') for _ in range(12)]
  assert g.per_job['imitation.discriminator.reward_function'] == [x for _ in range(3) for x in ('GAIL', 'AIRL', 'FAIRL') for _ in range(4)]
  assert g.per_job['imitation.spectral_norm'] == [x for _ in range(9) for x in (True, False) for _ in range(2)]
  assert g.per_job['imitation.grad_penalty'] == [0, 0.5] * 18
  # group_jobs keeps today's partition: every choice but mixup_alpha is a grouping key of the general discriminator
  groups = group_jobs(jobs)
  assert len(groups) == 36 and all(len(x.jobs) == 1 and x.per_job == {} for x in groups)


def test_prior_and_margin_are_per_replica_on_the_general_discriminator():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.depth=2', 'imitation.loss_function=PUGAIL', 'imitation.pos_class_prior=0.3,0.7',
                          'imitation.nonnegative_margin=0,0.5', 'imitation.mixup_alpha=0.4,1'])
  (g, ) = sweep_groups(jobs)
  assert g.per_job == {'imitation.pos_class_prior': [0.3, 0.3, 0.3, 0.3, 0.7, 0.7, 0.7, 0.7], 'imitation.nonnegative_margin': [0, 0, 0.5, 0.5] * 2,
                       'imitation.mixup_alpha': [0.4, 1] * 4}


@pytest.mark.parametrize('split', ['imitation.discriminator.hidden_size=64,128', 'imitation.discriminator.depth=2,3', 'imitation.discriminator.activation=tanh,sigmoid'])
def test_shape_and_activation_still_split_general_groups(split):
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.reward_shaping=true', split, 'imitation.loss_function=BCE,Mixup'])
  groups = sweep_groups(jobs)
  assert len(groups) == 2
  for g in groups:
    assert len({j.overrides[2] for j in g.jobs}) == 1 and g.per_job == {'imitation.loss_function': ['BCE', 'Mixup']}


def test_general_and_fused_jobs_are_never_one_program():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.depth=1,2', 'imitation.loss_function=BCE,Mixup'])
  groups = sweep_groups(jobs)
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1], [2, 3]]


def test_fused_per_replica_keys_are_unchanged():
  cfg = load_config(['algorithm=GAIL'])
  assert general_discriminator_keys(cfg) == ()
  assert per_replica_keys(cfg) == vectorised_keys(cfg) + ('seed', )
  assert general_discriminator_keys(load_config(['algorithm=RED', 'imitation.discriminator.depth=2'])) == ()


def test_general_keys_enter_per_replica_keys_only():
  cfg = load_config(['algorithm=GAIL', 'imitation.discriminator.depth=2'])
  assert set(PER_REPLICA_GENERAL_DISCRIMINATOR) <= set(per_replica_keys(cfg))
  assert 'imitation.grad_penalty' not in vectorised_keys(cfg) and 'imitation.loss_function' not in vectorised_keys(cfg)
  assert len(set(per_replica_keys(cfg))) == len(per_replica_keys(cfg))


def test_split_per_replica_refuses_invalid_general_values():
  cfg = load_config(['algorithm=GAIL', 'imitation.discriminator.activation=tanh'])
  with pytest.raises(SweepError, match='pos_class_prior'):
    split_per_replica(cfg, {'imitation.loss_function': ['PUGAIL', 'BCE'], 'imitation.pos_class_prior': [1.5, 0.5]}, 2)
  with pytest.raises(SweepError, match='nonnegative_margin'):
    split_per_replica(cfg, {'imitation.loss_function': ['PUGAIL', 'PUGAIL'], 'imitation.nonnegative_margin': [-1.0, 0.0]}, 2)
  with pytest.raises(SweepError, match='mixup_alpha'):
    split_per_replica(cfg, {'imitation.loss_function': ['Mixup', 'BCE'], 'imitation.mixup_alpha': [0, 1]}, 2)
  with pytest.raises(SweepError, match='Foo'):
    split_per_replica(cfg, {'imitation.loss_function': ['Foo', 'BCE']}, 2)
  with pytest.raises(SweepError, match='Foo'):
    split_per_replica(cfg, {'imitation.discriminator.reward_function': ['Foo', 'GAIL']}, 2)
  with pytest.raises(SweepError, match='true / false'):
    split_per_replica(cfg, {'imitation.spectral_norm': ['yes', True]}, 2)
  with pytest.raises(SweepError, match='not a number'):
    split_per_replica(cfg, {'imitation.grad_penalty': ['a', 0.5]}, 2)
  with pytest.raises(SweepError, match='hidden_size'):
    split_per_replica(cfg, {'imitation.discriminator.hidden_size': [64, 128]}, 2)
  _, arrays = split_per_replica(cfg, {'imitation.loss_function': ['BCE', 'PUGAIL'], 'imitation.grad_penalty': [0, 0.5], 'imitation.spectral_norm': [True, True]}, 2)
  assert arrays == {'imitation.loss_function': ['BCE', 'PUGAIL'], 'imitation.grad_penalty': [0.0, 0.5]}
