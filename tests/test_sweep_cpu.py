"""Multirun command lines (Hydra's basic sweeper, `train.py -m key=a,b,...`) without a GPU: job expansion and numbering, the split of swept keys
into per-replica (vectorised) and grouping keys, the collapse of equal per-replica values, and the refusals of sweep syntax outside -m."""
import pytest

from il_b200.config import VECTORISED, SweepError, expand_sweep, group_jobs, load_config, split_per_replica


def _ov(jobs):
  return [j.overrides for j in jobs]


def test_one_swept_key_in_order():
  multirun, jobs = expand_sweep(['-m', 'algorithm=PWIL', 'env=walker2d', 'reinforcement.discount=0.97,0.98,0.99'])
  assert multirun and [j.num for j in jobs] == [0, 1, 2]
  assert _ov(jobs) == [['algorithm=PWIL', 'env=walker2d', f'reinforcement.discount={d}'] for d in ('0.97', '0.98', '0.99')]


def test_two_and_three_swept_keys_last_varies_fastest():
  _, jobs = expand_sweep(['--multirun', 'seed=1,2', 'env=hopper', 'training.learning_rate=1e-4,3e-4'])
  assert _ov(jobs) == [['seed=1', 'env=hopper', 'training.learning_rate=1e-4'], ['seed=1', 'env=hopper', 'training.learning_rate=3e-4'],
                       ['seed=2', 'env=hopper', 'training.learning_rate=1e-4'], ['seed=2', 'env=hopper', 'training.learning_rate=3e-4']]
  _, jobs = expand_sweep(['-m', 'a=1,2', 'b=x,y', 'c=5,6,7'])
  assert len(jobs) == 12 and [j.num for j in jobs] == list(range(12))
  assert jobs[0].overrides == ['a=1', 'b=x', 'c=5'] and jobs[1].overrides == ['a=1', 'b=x', 'c=6'] and jobs[3].overrides == ['a=1', 'b=y', 'c=5']
  assert jobs[11].overrides == ['a=2', 'b=y', 'c=7']


def test_non_swept_overrides_are_carried_into_every_job():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'steps=100', 'imitation.grad_penalty=0,1', 'training.batch_size=32'])
  assert all(j.overrides[0] == 'algorithm=GAIL' and j.overrides[1] == 'steps=100' and j.overrides[3] == 'training.batch_size=32' for j in jobs)


def test_without_multirun_is_one_job():
  multirun, jobs = expand_sweep(['algorithm=GAIL', 'training.batch_size=32'])
  assert not multirun and len(jobs) == 1 and jobs[0].overrides == ['algorithm=GAIL', 'training.batch_size=32']


def test_vectorised_and_grouping_keys_partition_the_jobs():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'training.batch_size=32,64', 'training.learning_rate=1e-4,3e-4'])
  groups = group_jobs(jobs)
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1], [2, 3]]
  for g in groups: assert g.per_job == {'training.learning_rate': [1e-4, 3e-4]}
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'reinforcement.discount=0.97,0.99', 'imitation.grad_penalty=0,1', 'imitation.entropy_bonus=0,0.1'])
  (g, ) = group_jobs(jobs)
  assert len(g.jobs) == 8 and g.per_job['imitation.grad_penalty'] == [0, 0, 1, 1, 0, 0, 1, 1]
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'seed=1,2', 'env=hopper,walker2d'])  # seed and env are grouping keys
  assert len(group_jobs(jobs)) == 4


def test_general_discriminator_keeps_grad_penalty_a_grouping_key():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.reward_shaping=true', 'imitation.grad_penalty=0,1', 'reinforcement.discount=0.9,0.99'])
  groups = group_jobs(jobs)
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1], [2, 3]]
  assert all(set(g.per_job) == {'reinforcement.discount'} for g in groups)


def test_every_vectorised_key_exists_in_the_config():
  cfg = load_config(['algorithm=GAIL'])
  for k in VECTORISED:
    node = cfg
    for p in k.split('.'): node = node[p]
    assert isinstance(node, (int, float)), k


def test_equal_values_collapse_to_a_scalar():
  cfg = load_config(['algorithm=GAIL'])
  out, arrays = split_per_replica(cfg, {'training.learning_rate': [1e-4] * 4, 'reinforcement.discount': [0.9, 0.9, 0.99, 0.99]}, 4)
  assert arrays == {'reinforcement.discount': [0.9, 0.9, 0.99, 0.99]}
  assert out.training.learning_rate == 1e-4 and cfg.training.learning_rate == load_config(['algorithm=GAIL']).training.learning_rate  # the caller's config is untouched
  with pytest.raises(SweepError): split_per_replica(cfg, {'training.batch_size': [32, 64]}, 2)
  with pytest.raises(SweepError): split_per_replica(cfg, {'training.learning_rate': [1e-4, 3e-4]}, 3)


@pytest.mark.parametrize('argv', [['-m', 'training.learning_rate=range(1,3)'], ['-m', 'seed=choice(1,2)'], ['-m', 'training.learning_rate=interval(0,1)'],
                                  ['-m', 'env=glob(*)']])
def test_other_sweep_syntaxes_raise(argv):
  with pytest.raises(SweepError, match='only comma-separated'):
    expand_sweep(argv)


def test_comma_list_without_multirun_raises():
  with pytest.raises(SweepError, match='multirun'):
    expand_sweep(['training.learning_rate=1e-4,3e-4'])
  with pytest.raises(SweepError, match='multirun'):
    load_config(['reinforcement.discount=0.97,0.98,0.99'])
  with pytest.raises(SweepError):
    load_config(['-m', 'algorithm=PWIL'])


def test_quoted_comma_value_stays_a_string():
  assert load_config(["imitation.loss_function='BCE,Mixup'"]).imitation.loss_function == 'BCE,Mixup'
  _, jobs = expand_sweep(['-m', "imitation.loss_function='BCE,Mixup'", 'seed=1,2'])
  assert len(jobs) == 2 and jobs[0].overrides[0] == "imitation.loss_function='BCE,Mixup'"


def test_load_config_unchanged_for_existing_override_forms():
  cfg = load_config(['algorithm=GAIL', 'env=walker2d', 'training.batch_size=512', 'training.learning_rate=3e-4', 'reinforcement.discount=0.97', 'imitation.absorbing=false',
                     'output_dir=null', '+extra.key=5', 'imitation.discriminator.hidden_size=32', "name='x y'", 'lst=[1,2]', 'optimised_hyperparameters=GAIL_5_trajectories'])
  assert cfg.algorithm == 'GAIL' and cfg.env == 'walker2d' and cfg.training.batch_size == 512 and cfg.training.learning_rate == 3e-4
  assert cfg.reinforcement.discount == 0.97 and cfg.imitation.absorbing is False and cfg.output_dir is None and cfg.extra.key == 5
  assert cfg.imitation.discriminator.hidden_size == 32 and cfg.name == 'x y' and cfg.lst == [1, 2]
