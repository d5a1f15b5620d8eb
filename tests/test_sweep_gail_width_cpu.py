"""Multirun sweeps over the GAIL discriminator's hidden size without a GPU: a per-replica shape of the fused discriminator (one group), a grouping
key of the general one and of RED / DRIL, with its values validated and the number of distinct widths in one program capped."""
import pytest

from il_b200 import _lib
from il_b200.config import MAX_WIDTH_CLASSES, PER_REPLICA_WIDTH, SweepError, expand_sweep, group_jobs, load_config, split_per_replica, vectorised_keys

W = 'imitation.discriminator.hidden_size'


def test_width_by_loss_sweep_is_one_group_on_the_fused_discriminator():
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', f'{W}=32,64,128', 'imitation.loss_function=BCE,Mixup,PUGAIL'])
  (g, ) = group_jobs(jobs)
  assert [j.num for j in g.jobs] == list(range(9))
  assert g.per_job[W] == [x for x in (32, 64, 128) for _ in range(3)]
  assert g.per_job['imitation.loss_function'] == ['BCE', 'Mixup', 'PUGAIL'] * 3
  assert W in vectorised_keys(load_config(['algorithm=GAIL'])) and PER_REPLICA_WIDTH == (W, )


@pytest.mark.parametrize('general', ['imitation.discriminator.depth=2', 'imitation.discriminator.activation=tanh', 'imitation.discriminator.reward_shaping=true'])
def test_width_splits_groups_on_the_general_discriminator(general):
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', general, f'{W}=32,64,128', 'reinforcement.discount=0.97,0.99'])
  groups = group_jobs(jobs)
  assert [[j.num for j in g.jobs] for g in groups] == [[0, 1], [2, 3], [4, 5]]
  assert all(set(g.per_job) == {'reinforcement.discount'} for g in groups)
  assert W not in vectorised_keys(load_config(['algorithm=GAIL', general]))


@pytest.mark.parametrize('alg', ['RED', 'DRIL'])
def test_width_splits_groups_for_red_and_dril(alg):
  _, jobs = expand_sweep(['-m', f'algorithm={alg}', f'{W}=32,64'])
  assert len(group_jobs(jobs)) == 2
  assert W not in vectorised_keys(load_config([f'algorithm={alg}']))


def test_width_values_are_positive_ints():
  cfg = load_config(['algorithm=GAIL'])
  for bad in (True, '64', 64.0, 48.5, 0, -32):
    with pytest.raises(SweepError, match='positive integer'):
      split_per_replica(cfg, {W: [64, bad]}, 2)
  out, arrays = split_per_replica(cfg, {W: [64, 64]}, 2)
  assert arrays == {} and out.imitation.discriminator.hidden_size == 64
  out, arrays = split_per_replica(cfg, {W: [32, 128, 48]}, 3)
  assert arrays == {W: [32, 128, 48]}


def test_width_class_cap():
  assert MAX_WIDTH_CLASSES == _lib.MAX_WIDTH_CLASSES == 8
  cfg = load_config(['algorithm=GAIL'])
  widths = [16 * (i + 1) for i in range(MAX_WIDTH_CLASSES)]
  _, arrays = split_per_replica(cfg, {W: widths + widths}, 2 * MAX_WIDTH_CLASSES)  # at the cap
  assert arrays[W] == widths + widths
  with pytest.raises(SweepError, match=f'at most {MAX_WIDTH_CLASSES}'):
    split_per_replica(cfg, {W: widths + [200]}, MAX_WIDTH_CLASSES + 1)
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', f'{W}=' + ','.join(str(x) for x in widths + [200])])
  with pytest.raises(SweepError, match=f'at most {MAX_WIDTH_CLASSES}'):
    group_jobs(jobs)
  # on the general discriminator the widths are separate programs: no cap
  _, jobs = expand_sweep(['-m', 'algorithm=GAIL', 'imitation.discriminator.depth=2', f'{W}=' + ','.join(str(x) for x in widths + [200])])
  assert len(group_jobs(jobs)) == MAX_WIDTH_CLASSES + 1


def test_struct_mirror_has_the_width_class_table():
  g = _lib.Gail()
  assert len(g.width_class_H) == len(g.width_class_begin) == MAX_WIDTH_CLASSES
  assert _lib.Gail.replica_order.offset % 8 == 0 and _lib.Gail.n_width_classes.offset == _lib.Gail.spectral_norm_r.offset + 8
