"""Which keys take per-replica values, without a GPU: for one configuration of each kind, the keys per replica in both multirun partitions
(vectorised_keys) and those per replica in the programs a multirun runs (per_replica_keys), pinned as literal sets; and the group_jobs /
sweep_groups partitions of three multiruns that cross per-replica keys with grouping keys."""
import pytest

from il_b200.config import expand_sweep, group_jobs, load_config, per_replica_keys, sweep_groups, vectorised_keys

SCALARS = {'training.learning_rate', 'training.weight_decay', 'reinforcement.discount', 'reinforcement.target_temperature', 'reinforcement.polyak_factor',
           'imitation.learning_rate', 'imitation.weight_decay', 'imitation.grad_penalty', 'imitation.entropy_bonus', 'bc_pretraining.learning_rate',
           'bc_pretraining.weight_decay'}
GP, LOSS, RF, SN, ALPHA, PRIOR, MARGIN, WIDTH = ('imitation.grad_penalty', 'imitation.loss_function', 'imitation.discriminator.reward_function', 'imitation.spectral_norm',
                                                 'imitation.mixup_alpha', 'imitation.pos_class_prior', 'imitation.nonnegative_margin', 'imitation.discriminator.hidden_size')
IN, DROP, ACT = 'imitation.discriminator.input_dropout', 'imitation.discriminator.dropout', 'imitation.discriminator.activation'
CUTOFF, SCALE, BANDWIDTH = 'imitation.quantile_cutoff', 'imitation.reward_scale', 'imitation.reward_bandwidth_scale'
FUSED = SCALARS | {LOSS, RF, SN, ALPHA, PRIOR, MARGIN, WIDTH}
GENERAL = (SCALARS - {GP} | {ALPHA}, {GP, LOSS, RF, SN, PRIOR, MARGIN, 'seed'})

# name: (overrides, set(vectorised_keys), set(per_replica_keys) - set(vectorised_keys))
KEYS = {
    'AdRIL': (['algorithm=AdRIL'], SCALARS | {'imitation.balanced', 'imitation.update_freq'}, {'seed'}),
    'BC': (['algorithm=BC'], SCALARS, {'seed'}),
    'DRIL': (['algorithm=DRIL'], SCALARS | {CUTOFF}, {IN, DROP, ACT, 'seed'}),
    'GAIL': (['algorithm=GAIL'], FUSED, {'seed'}),
    'GMMIL': (['algorithm=GMMIL'], SCALARS, {'seed'}),
    'PWIL': (['algorithm=PWIL'], SCALARS | {SCALE, BANDWIDTH}, {'seed'}),
    'RED': (['algorithm=RED'], SCALARS, {IN, DROP, ACT, 'seed'}),
    'SAC': (['algorithm=SAC'], SCALARS, {'seed'}),
    'GAIL general depth 2': (['algorithm=GAIL', 'imitation.discriminator.depth=2'], *GENERAL),
    'GAIL general tanh': (['algorithm=GAIL', 'imitation.discriminator.activation=tanh'], *GENERAL),
    'GAIL general shaping + log-policy': (['algorithm=GAIL', 'imitation.discriminator.reward_shaping=true', 'imitation.discriminator.subtract_log_policy=true'], *GENERAL),
    'PWIL none': (['algorithm=PWIL', 'imitation.mix_expert_data=none'], SCALARS | {SCALE, BANDWIDTH}, {'seed'}),
    'PWIL mixed_batch': (['algorithm=PWIL', 'imitation.mix_expert_data=mixed_batch'], SCALARS, {'seed'}),
    'PWIL prefill_memory': (['algorithm=PWIL', 'imitation.mix_expert_data=prefill_memory'], SCALARS, {'seed'}),
    'DRIL without a dropout site': (['algorithm=DRIL', f'{IN}=0', f'{DROP}=0'], SCALARS | {CUTOFF}, {IN, DROP, 'seed'}),
    'GAIL device_rng=false': (['algorithm=GAIL', 'device_rng=false'], FUSED, set()),
    'GAIL subsample=2 (expert memory)': (['algorithm=GAIL', 'imitation.subsample=2'], FUSED, set()),
    'SAC subsample=2 (no expert memory)': (['algorithm=SAC', 'imitation.subsample=2'], SCALARS, {'seed'}),
}


@pytest.mark.parametrize('name', list(KEYS))
def test_per_replica_keys_of_each_kind_of_configuration(name):
  overrides, vectorised, sweep_only = KEYS[name]
  cfg = load_config(overrides)
  assert set(vectorised_keys(cfg)) == vectorised
  assert set(per_replica_keys(cfg)) == vectorised | sweep_only
  assert per_replica_keys(cfg)[:len(vectorised_keys(cfg))] == vectorised_keys(cfg)


# name: (argv, group_jobs partition, sweep_groups partition); a partition is [(job numbers, swept keys with per-job values)] in group order
PARTITIONS = {
    # seed and (on the general discriminator) the loss function are per replica in sweep_groups only, env and depth group, GAIL ignores dropout
    'GAIL': (['-m', 'algorithm=GAIL', 'seed=1,2', 'env=hopper,walker2d', f'{LOSS}=BCE,PUGAIL', 'imitation.discriminator.depth=1,2', f'{DROP}=0.25,0.75'],
             [([0, 1, 4, 5], {LOSS}), ([2, 3], set()), ([6, 7], set()), ([8, 9, 12, 13], {LOSS}), ([10, 11], set()), ([14, 15], set()),
              ([16, 17, 20, 21], {LOSS}), ([18, 19], set()), ([22, 23], set()), ([24, 25, 28, 29], {LOSS}), ([26, 27], set()), ([30, 31], set())],
             [([0, 1, 4, 5, 16, 17, 20, 21], {LOSS, 'seed'}), ([2, 3, 6, 7, 18, 19, 22, 23], {LOSS, 'seed'}), ([8, 9, 12, 13, 24, 25, 28, 29], {LOSS, 'seed'}),
              ([10, 11, 14, 15, 26, 27, 30, 31], {LOSS, 'seed'})]),
    # the dropout rates group on their presence, the activation groups without a dropout site, the width groups, the cutoff is per replica
    'DRIL': (['-m', 'algorithm=DRIL', f'{IN}=0,0.1', f'{DROP}=0,0.2', f'{ACT}=relu,tanh', f'{WIDTH}=32,64', f'{CUTOFF}=0.9,0.98'],
             [([2 * i, 2 * i + 1], {CUTOFF}) for i in range(16)],
             [([0, 1], {IN, DROP, CUTOFF}), ([2, 3], {IN, DROP, CUTOFF}), ([4, 5], {IN, DROP, CUTOFF}), ([6, 7], {IN, DROP, CUTOFF}),
              ([8, 9, 12, 13], {IN, DROP, ACT, CUTOFF}), ([10, 11, 14, 15], {IN, DROP, ACT, CUTOFF}), ([16, 17, 20, 21], {IN, DROP, ACT, CUTOFF}),
              ([18, 19, 22, 23], {IN, DROP, ACT, CUTOFF}), ([24, 25, 28, 29], {IN, DROP, ACT, CUTOFF}), ([26, 27, 30, 31], {IN, DROP, ACT, CUTOFF})]),
    # the scales are per replica without expert-data mixing only, the seed only without a subsampled expert memory
    'PWIL': (['-m', 'algorithm=PWIL', 'imitation.mix_expert_data=none,mixed_batch', f'{SCALE}=1,10', 'imitation.subsample=1,2', 'seed=1,2'],
             [([0, 4], {SCALE}), ([1, 5], {SCALE}), ([2, 6], {SCALE}), ([3, 7], {SCALE}), *(([j], set()) for j in range(8, 16))],
             [([0, 1, 4, 5], {SCALE, 'seed'}), ([2, 6], {SCALE}), ([3, 7], {SCALE}), ([8, 9], {'seed'}), ([10], set()), ([11], set()), ([12, 13], {'seed'}),
              ([14], set()), ([15], set())]),
}


@pytest.mark.parametrize('name', list(PARTITIONS))
def test_partitions_of_mixed_multiruns(name):
  argv, by_group_jobs, by_sweep_groups = PARTITIONS[name]
  _, jobs = expand_sweep(argv)
  for partition, want in ((group_jobs(jobs), by_group_jobs), (sweep_groups(jobs), by_sweep_groups)):
    assert [([j.num for j in g.jobs], set(g.per_job)) for g in partition] == want
    for g in partition:  # each per-job value is that job's value of the key
      for k, vals in g.per_job.items(): assert vals == [_value(j.overrides, k) for j in g.jobs]


def _value(overrides, k):
  node = load_config(overrides)
  for p in k.split('.'): node = node[p]
  return node
