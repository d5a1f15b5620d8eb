"""Multirun sweeps over AdRIL's, PWIL's and DRIL's own search-space keys without a GPU: AdRIL's update frequency and balanced sampling, PWIL's
reward scales (without expert-data mixing) and DRIL's quantile cutoff are per-replica keys (one group); PWIL's scales with mixed_batch /
prefill_memory and RED / DRIL width and dropout still split; values the reference asserts against are refused."""
import ctypes as C

import pytest

from il_b200 import _lib
from il_b200.config import PER_REPLICA_ALGORITHM, SweepError, expand_sweep, group_jobs, load_config, split_per_replica, vectorised_keys

ADRIL_FREQS = (0, 1250, 2500, 5000, 12500, 25000, 50000)


def test_adril_grid_is_one_group_in_hydra_order():
  _, jobs = expand_sweep(['-m', 'algorithm=AdRIL', 'imitation.balanced=true,false', 'imitation.update_freq=' + ','.join(map(str, ADRIL_FREQS))])
  assert len(jobs) == 14
  (g, ) = group_jobs(jobs)
  assert [j.num for j in g.jobs] == list(range(14))
  assert set(g.per_job) == {'imitation.update_freq', 'imitation.balanced'}
  assert g.per_job['imitation.balanced'] == [x for x in (True, False) for _ in range(7)]
  assert g.per_job['imitation.update_freq'] == list(ADRIL_FREQS) * 2


def test_pwil_scale_grid_is_one_group_without_expert_mixing():
  swept = ['imitation.reward_scale=1,5,10', 'imitation.reward_bandwidth_scale=1,5,10']
  _, jobs = expand_sweep(['-m', 'algorithm=PWIL', 'imitation.mix_expert_data=none', *swept])
  (g, ) = group_jobs(jobs)
  assert len(g.jobs) == 9
  assert g.per_job == {'imitation.reward_scale': [x for x in (1, 5, 10) for _ in range(3)], 'imitation.reward_bandwidth_scale': [1, 5, 10] * 3}
  for mix in ('mixed_batch', 'prefill_memory'):  # the relabelling walk writes scale-dependent rewards into the shared expert memory
    _, jobs = expand_sweep(['-m', 'algorithm=PWIL', f'imitation.mix_expert_data={mix}', *swept])
    groups = group_jobs(jobs)
    assert len(groups) == 9 and all(len(g.jobs) == 1 and g.per_job == {} for g in groups), mix
    assert not set(PER_REPLICA_ALGORITHM['PWIL']) & set(vectorised_keys(load_config(['algorithm=PWIL', f'imitation.mix_expert_data={mix}'])))


def test_pwil_mix_expert_data_sweep_groups_the_scales_per_mixing_mode():
  _, jobs = expand_sweep(['-m', 'algorithm=PWIL', 'imitation.mix_expert_data=none,mixed_batch', 'imitation.reward_scale=1,10'])
  groups = group_jobs(jobs)
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1], [2], [3]]
  assert groups[0].per_job == {'imitation.reward_scale': [1, 10]}


def test_dril_cutoff_sweep_is_one_group_but_width_and_dropout_split():
  _, jobs = expand_sweep(['-m', 'algorithm=DRIL', 'imitation.quantile_cutoff=0.8,0.9,0.98'])
  (g, ) = group_jobs(jobs)
  assert g.per_job == {'imitation.quantile_cutoff': [0.8, 0.9, 0.98]}
  _, jobs = expand_sweep(['-m', 'algorithm=DRIL', 'imitation.quantile_cutoff=0.8,0.98', 'imitation.discriminator.hidden_size=32,64'])
  groups = group_jobs(jobs)
  assert len(groups) == 2 and all(g.per_job == {'imitation.quantile_cutoff': [0.8, 0.98]} for g in groups)
  _, jobs = expand_sweep(['-m', 'algorithm=DRIL', 'imitation.quantile_cutoff=0.8,0.98', 'imitation.discriminator.dropout=0.1,0.2'])
  assert len(group_jobs(jobs)) == 2
  _, jobs = expand_sweep(['-m', 'algorithm=RED', 'imitation.discriminator.hidden_size=32,64', 'imitation.discriminator.input_dropout=0,0.5'])
  assert len(group_jobs(jobs)) == 4


def test_algorithm_keys_are_not_per_replica_for_other_algorithms():
  for alg in ('GAIL', 'RED', 'GMMIL', 'SAC'):
    keys = set(vectorised_keys(load_config([f'algorithm={alg}'])))
    assert not keys & {k for ks in PER_REPLICA_ALGORITHM.values() for k in ks}, alg
  with pytest.raises(SweepError, match='cannot take per-replica values'):
    split_per_replica(load_config(['algorithm=DRIL']), {'imitation.update_freq': [0, 1250]}, 2)


@pytest.mark.parametrize('alg,key,vals,match', [
    ('AdRIL', 'imitation.update_freq', [1250, -1], r'replica 1: imitation.update_freq=-1'),
    ('AdRIL', 'imitation.update_freq', [12.5, 1250], r'replica 0: imitation.update_freq=12.5'),
    ('AdRIL', 'imitation.update_freq', [0, True], r'replica 1: imitation.update_freq=True'),
    ('AdRIL', 'imitation.balanced', [True, 1], r'replica 1: imitation.balanced=1'),
    ('AdRIL', 'imitation.balanced', ['yes', False], r'replica 0: imitation.balanced'),
    ('DRIL', 'imitation.quantile_cutoff', [0.9, 1.5], r'replica 1: imitation.quantile_cutoff=1.5'),
    ('DRIL', 'imitation.quantile_cutoff', [-0.1, 0.9], r'replica 0: imitation.quantile_cutoff=-0.1'),
    ('DRIL', 'imitation.quantile_cutoff', [0.9, 'high'], r'replica 1: imitation.quantile_cutoff'),
    ('PWIL', 'imitation.reward_scale', [5, 'x'], r'replica 1: imitation.reward_scale'),
    ('PWIL', 'imitation.reward_bandwidth_scale', [False, 5], r'replica 0: imitation.reward_bandwidth_scale')])
def test_split_per_replica_refuses_values_the_reference_asserts_against(alg, key, vals, match):
  with pytest.raises(SweepError, match=match):
    split_per_replica(load_config([f'algorithm={alg}']), {key: vals}, 2)


def test_split_per_replica_keeps_types_and_collapses_equal_values():
  cfg = load_config(['algorithm=AdRIL'])
  out, arrays = split_per_replica(cfg, {'imitation.update_freq': [0, 1250, 0], 'imitation.balanced': [False] * 3}, 3)
  assert arrays == {'imitation.update_freq': [0, 1250, 0]} and all(type(x) is int for x in arrays['imitation.update_freq'])
  assert out.imitation.balanced is False and cfg.imitation.balanced is True
  out, arrays = split_per_replica(load_config(['algorithm=DRIL']), {'imitation.quantile_cutoff': [0.8, 1, 0]}, 3)
  assert arrays == {'imitation.quantile_cutoff': [0.8, 1.0, 0.0]}
  out, arrays = split_per_replica(load_config(['algorithm=PWIL']), {'imitation.reward_scale': [1, 10], 'imitation.reward_bandwidth_scale': [5, 5]}, 2)
  assert arrays == {'imitation.reward_scale': [1.0, 10.0]} and out.imitation.reward_bandwidth_scale == 5.0


def test_pwil_struct_size_matches_c():
  out = (C.c_int32 * 15)()
  assert _lib.lib().il_struct_sizes(out) == 0
  assert out[7] == C.sizeof(_lib.Pwil) == 80
  assert _lib.Pwil.reward_scale_r.offset == 64 and _lib.Pwil.reward_bandwidth_r.offset == 72
