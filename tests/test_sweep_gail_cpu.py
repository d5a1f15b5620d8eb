"""Multirun sweeps over the GAIL discriminator's choices without a GPU: loss function, reward function, spectral norm and the Mixup / PUGAIL
parameters are per-replica keys of the fused discriminator (one group), grouping keys of the general one (except mixup_alpha), and the
discriminator dropout that GAIL never reads does not split a sweep."""
import pytest

from il_b200.config import PER_REPLICA_DISCRIMINATOR, VECTORISED, SweepError, expand_sweep, group_jobs, load_config, split_per_replica, vectorised_keys


def test_discriminator_choice_grid_is_one_group_in_hydra_order():
  argv = ['-m', 'algorithm=GAIL', 'imitation.loss_function=BCE,Mixup,PUGAIL', 'imitation.discriminator.reward_function=GAIL,AIRL,FAIRL', 'imitation.spectral_norm=true,false',
          'imitation.mixup_alpha=0.4,1', 'imitation.pos_class_prior=0.5,0.7']
  _, jobs = expand_sweep(argv)
  assert len(jobs) == 3 * 3 * 2 * 2 * 2
  (g, ) = group_jobs(jobs)
  assert [j.num for j in g.jobs] == list(range(72))
  assert set(g.per_job) == set(PER_REPLICA_DISCRIMINATOR) - {'imitation.nonnegative_margin'}
  # the last key varies fastest (Hydra's basic sweeper)
  assert g.per_job['imitation.loss_function'] == [x for x in ('BCE', 'Mixup', 'PUGAIL') for _ in range(24)]
  assert g.per_job['imitation.discriminator.reward_function'] == [x for _ in range(3) for x in ('GAIL', 'AIRL', 'FAIRL') for _ in range(8)]
  assert g.per_job['imitation.spectral_norm'] == [x for _ in range(9) for x in (True, False) for _ in range(4)]
  assert g.per_job['imitation.mixup_alpha'] == [x for _ in range(18) for x in (0.4, 1) for _ in range(2)]
  assert g.per_job['imitation.pos_class_prior'] == [0.5, 0.7] * 36


def test_gail_ignores_discriminator_dropout_but_red_does_not():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.input_dropout=0,0.5', 'imitation.discriminator.dropout=0.25,0.75'])
  (g, ) = group_jobs(jobs)
  assert len(g.jobs) == 4 and g.per_job == {}
  _, jobs = expand_sweep(['-m', 'algorithm=RED', 'imitation.discriminator.input_dropout=0,0.5', 'imitation.discriminator.dropout=0.25,0.75'])
  assert len(group_jobs(jobs)) == 4


def test_general_discriminator_groups_on_choices_but_not_on_mixup_alpha():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.reward_shaping=true', 'imitation.loss_function=BCE,Mixup',
                          'imitation.discriminator.reward_function=AIRL,GAIL', 'imitation.spectral_norm=true,false', 'imitation.mixup_alpha=0.4,1'])
  groups = group_jobs(jobs)
  assert len(groups) == 8
  assert all(len(g.jobs) == 2 and set(g.per_job) == {'imitation.mixup_alpha'} for g in groups)
  cfg = load_config(['algorithm=GAIL', 'imitation.discriminator.reward_shaping=true'])
  assert 'imitation.loss_function' not in vectorised_keys(cfg) and 'imitation.mixup_alpha' in vectorised_keys(cfg)


def test_choice_keys_are_not_per_replica_outside_gail():
  cfg = load_config(['algorithm=RED'])
  assert not set(PER_REPLICA_DISCRIMINATOR) & set(vectorised_keys(cfg))
  assert set(VECTORISED) <= set(vectorised_keys(load_config(['algorithm=GAIL'])))


def test_split_per_replica_refuses_values_the_reference_asserts_against():
  cfg = load_config(['algorithm=GAIL'])
  with pytest.raises(SweepError, match='pos_class_prior'):
    split_per_replica(cfg, {'imitation.loss_function': ['PUGAIL', 'BCE'], 'imitation.pos_class_prior': [1.5, 0.5]}, 2)
  with pytest.raises(SweepError, match='mixup_alpha'):
    split_per_replica(cfg, {'imitation.loss_function': ['Mixup', 'BCE'], 'imitation.mixup_alpha': [0, 1]}, 2)
  with pytest.raises(SweepError, match='nonnegative_margin'):
    split_per_replica(cfg, {'imitation.loss_function': ['PUGAIL', 'PUGAIL'], 'imitation.nonnegative_margin': [-1.0, 0.0]}, 2)
  with pytest.raises(SweepError, match='Foo'):
    split_per_replica(cfg, {'imitation.loss_function': ['Foo', 'BCE']}, 2)
  with pytest.raises(SweepError, match='Foo'):
    split_per_replica(cfg, {'imitation.discriminator.reward_function': ['Foo', 'Foo']}, 2)
  with pytest.raises(SweepError, match='true / false'):
    split_per_replica(cfg, {'imitation.spectral_norm': ['yes', True]}, 2)
  # a prior outside [0, 1] is only refused for PUGAIL replicas (the reference asserts it under loss_function == 'PUGAIL')
  _, arrays = split_per_replica(cfg, {'imitation.loss_function': ['BCE', 'PUGAIL'], 'imitation.pos_class_prior': [1.5, 0.5]}, 2)
  assert arrays['imitation.pos_class_prior'] == [1.5, 0.5]


def test_split_per_replica_collapses_equal_strings_and_bools():
  cfg = load_config(['algorithm=GAIL'])
  out, arrays = split_per_replica(cfg, {'imitation.loss_function': ['Mixup'] * 3, 'imitation.spectral_norm': [False] * 3, 'imitation.discriminator.reward_function': ['GAIL', 'AIRL', 'GAIL'],
                                        'imitation.mixup_alpha': [0.4, 0.4, 0.4]}, 3)
  assert arrays == {'imitation.discriminator.reward_function': ['GAIL', 'AIRL', 'GAIL']}
  assert out.imitation.loss_function == 'Mixup' and out.imitation.spectral_norm is False and out.imitation.mixup_alpha == 0.4
  assert cfg.imitation.loss_function == 'BCE'  # the caller's config is untouched
