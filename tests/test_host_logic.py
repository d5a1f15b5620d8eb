"""CPU-only checks of the host-side logic of the drop-in: expert-data ingest (environments.py:63-125), the Hydra-free
configuration surface (train.py:21-23, conf/) and the replica sharding helpers. No CUDA call is made here."""
import os

import numpy as np
import pytest
import torch
import yaml

from il_b200 import config, environments
from oracle import cases, port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INGEST = [n for n, c in cases.CASES.items() if c['kind'] == 'ingest']


@pytest.mark.parametrize('name', INGEST)
def test_expert_ingest_equals_oracle_bit_for_bit(name):
  """il_b200.environments.build_expert_transitions (the product's get_dataset preprocessing, global numpy RNG for the
  subsampling offsets like environments.py:113) == the oracle port, which tests/golden pins against the reference."""
  c, inp = cases.CASES[name], cases.make_inputs(name)
  raw = {k: torch.from_numpy(inp[k].copy()) for k in ('observations', 'next_observations', 'actions', 'terminals', 'timeouts')}
  seed = int(inp['np_seed'][0])
  state = np.random.get_state()
  np.random.seed(seed)
  try:
    got = environments.build_expert_transitions(raw, c['trajectories'], c['subsample'], c['absorbing'])
  finally:
    np.random.set_state(state)
  want = port.build_expert_transitions(raw, c['trajectories'], c['subsample'], c['absorbing'], rng=np.random.RandomState(seed))
  assert got['num_trajectories'] == want['num_trajectories']
  for k in ('states', 'actions', 'next_states', 'terminals', 'timeouts', 'weights', 'rewards'):
    assert got[k].shape == want[k].shape, k
    assert torch.equal(got[k], want[k]), k
  assert inp['terminals'].tobytes() == raw['terminals'].numpy().tobytes(), 'the raw buffer must not be modified'


def test_expert_ingest_edge_cases():
  """Ragged input: a single one-step episode, an episode that ends by time limit (no absorbing row), subsample larger
  than an episode (the absorbing pair is always kept, environments.py:115)."""
  obs, A = 3, 2
  raw = dict(observations=torch.arange(18, dtype=torch.float32).view(6, obs), next_observations=torch.ones(6, obs), actions=torch.zeros(6, A),
             terminals=torch.tensor([1., 0, 0, 0, 0, 1]), timeouts=torch.tensor([0., 0, 0, 1, 0, 0]))
  tr = environments.build_expert_transitions(raw, 0, 1, True)
  assert tr['num_trajectories'] == 3
  # episode 0: 1 row + absorbing row; episode 1: 3 rows, timeout, no absorbing row; episode 2: 2 rows + absorbing row
  assert tr['states'].shape == (1 + 1 + 3 + 2 + 1, obs + 1)
  assert tr['states'][:, -1].tolist() == [0, 1, 0, 0, 0, 0, 0, 1]
  assert tr['terminals'].sum() == 0 and tr['timeouts'].tolist() == [0, 0, 0, 0, 1, 0, 0, 0]
  assert torch.all(tr['rewards'] == 0)
  state = np.random.get_state()
  np.random.seed(0)
  try:
    sub = environments.build_expert_transitions(raw, 1, 20, True)  # first episode only, subsample 20 > length
  finally:
    np.random.set_state(state)
  assert sub['states'].shape[0] == 2 and torch.equal(sub['weights'], torch.full((2,), 1 / 20))


def _reference_conf(*parts):
  """The reference's conf/<parts> flattened, as stored by oracle/ref_golden.py."""
  from oracle import ref_golden
  return ref_golden.load_conf()['/'.join(parts)]


def _flat(d, prefix=''):
  out = {}
  for k, v in d.items():
    if isinstance(v, dict): out.update(_flat(v, f'{prefix}{k}.'))
    else: out[prefix + k] = v
  return out


def test_config_defaults_and_overrides():
  cfg = config.load_config(['algorithm=GAIL', 'env=hopper', 'training.batch_size=512', 'imitation.discriminator.reward_function=FAIRL', 'replicas=8', 'cuda_graphs=false'])
  assert cfg.algorithm == 'GAIL' and cfg.env == 'hopper'
  assert cfg.training.batch_size == 512 and isinstance(cfg.training.batch_size, int)
  assert cfg.imitation.discriminator.reward_function == 'FAIRL'
  assert cfg.replicas == 8 and cfg.cuda_graphs is False
  # GAIL.yaml:5-7 overlays (discount / target temperature / polyak) on top of train_config.yaml:36-38
  assert cfg.reinforcement.discount == 0.97 and cfg.reinforcement.polyak_factor == 0.99 and cfg.reinforcement.target_temperature == -0.5
  assert cfg.imitation.weight_decay == 10 and cfg.imitation.learning_rate == 3e-5 and cfg.imitation.spectral_norm is True
  sac = config.load_config(['algorithm=SAC'])
  assert sac.reinforcement.discount == 0.99 and sac.reinforcement.polyak_factor == 0.995
  tuned = config.load_config(['algorithm=GAIL', 'optimised_hyperparameters=GAIL_5_trajectories'])
  assert tuned.training.batch_size == 1024 and tuned.imitation.loss_function == 'Mixup'
  with pytest.raises(FileNotFoundError): config.load_config(['algorithm=NOPE'])
  assert config.load_config(['algorithm=RED']).imitation.pretraining.iterations == 100000 and config.load_config(['algorithm=DRIL']).imitation.quantile_cutoff == 0.98
  assert config.load_config(['algorithm=AdRIL']).imitation.update_freq == 1250
  with pytest.raises(AttributeError): _ = cfg.training.no_such_key


def test_conf_tree_carries_the_reference_values():
  """Every key of the reference's train_config.yaml / algorithm overlays / tuned overlays that this repo ships has
  the reference's value (this repo adds keys — replicas, device_rng, cuda_graphs, gemm_mode, output_dir — never changes one)."""
  ours = _flat(config.load_config([]))
  for k, v in _reference_conf('train_config.yaml').items():
    if k.startswith(('hydra', 'defaults')): continue
    assert k in ours, f'train_config.yaml: {k} missing'
    assert ours[k] == v, (k, ours[k], v)
  for alg in ('SAC', 'GAIL', 'GMMIL', 'PWIL', 'BC'):
    with open(os.path.join(ROOT, 'conf', 'algorithm', f'{alg}.yaml')) as f: mine = _flat(yaml.safe_load(f) or {})
    theirs = {k: v for k, v in _reference_conf('algorithm', f'{alg}.yaml').items() if not k.startswith(('defaults', 'hydra'))}
    assert mine == theirs, (alg, set(mine.items()) ^ set(theirs.items()))
  for alg in ('BC', 'GAIL', 'GMMIL', 'PWIL'):
    for n in (5, 10, 25):
      name = f'{alg}_{n}_trajectories.yaml'
      with open(os.path.join(ROOT, 'conf', 'optimised_hyperparameters', name)) as f: mine = _flat(yaml.safe_load(f) or {})
      theirs = {k: v for k, v in _reference_conf('optimised_hyperparameters', name).items() if not k.startswith(('defaults', 'hydra'))}
      assert mine == theirs, (name, set(mine.items()) ^ set(theirs.items()))


def test_parameter_initialisation_consumes_the_reference_rng_stream():
  """train.py:51-66 seeds torch once and builds actor, then the twin critic; replica r of this build must initialise
  like a reference run with seed + r (net.ReplicaRNG + net.init_fcnn_params, CPU side of ReplicaMLP). The reference's
  parameters are stored as a fixed sample of entries and the SHA-256 of every tensor's bytes (oracle/ref_golden.py)."""
  from il_b200 import net
  from oracle import ref_golden
  ref = ref_golden.load_init()
  S, A, H = 12, 3, 256
  rng = net.ReplicaRNG(seed=7, replicas=3)
  for r in range(3):
    with rng.replica(r):
      mine_actor = net.init_fcnn_params([S, H, H, 2 * A], 'relu')
      mine_c1, mine_c2 = net.init_fcnn_params([S + A, H, H, 1], 'relu'), net.init_fcnn_params([S + A, H, H, 1], 'relu')
    for name, mine in (('actor', mine_actor), ('critic_1', mine_c1), ('critic_2', mine_c2)):
      assert sum(k.startswith(f'{r}|{name}|') for k in ref) == len(mine)
      for i, t in enumerate(mine):
        tag = f"{r}|{name}|{i // 2}|{'bias' if i % 2 else 'weight'}"
        # bit equality of every entry: tensors of up to 8 entries are stored whole, larger ones as sampled entries + SHA-256 of their bytes
        if isinstance(ref[tag], np.ndarray): assert np.array_equal(t.numpy(), ref[tag]), tag
        else: ref[tag].check_equal(tag, t)
  # the global stream is left untouched by the per-replica streams
  torch.manual_seed(123)
  a = torch.rand(3)
  torch.manual_seed(123)
  with rng.replica(0): net.init_fcnn_params([4, 4], 'relu')
  assert torch.equal(a, torch.rand(3))


def test_shard_and_statistics_helpers():
  from il_b200 import distributed
  for total, world in ((1024, 1), (1024, 8), (10, 4), (7, 8)):
    spans = [distributed.shard(total, rank, world) for rank in range(world)]
    assert spans[0][0] == 0 and spans[-1][1] == total
    assert all(a[1] == b[0] for a, b in zip(spans[:-1], spans[1:]))
    sizes = [hi - lo for lo, hi in spans]
    assert max(sizes) - min(sizes) <= 1


def test_cli_overrides_parse_like_hydra():
  """ADVICE r1: `training.learning_rate=3e-4` and `imitation.nonnegative_margin=inf` must arrive as floats (YAML 1.1 reads them as strings)."""
  from il_b200.config import load_config
  cfg = load_config(['algorithm=GAIL', 'env=hopper', 'training.learning_rate=3e-4', 'imitation.nonnegative_margin=inf', 'steps=1e5', 'training.batch_size=512',
                     'imitation.spectral_norm=false', 'imitation.loss_function=PUGAIL', 'imitation.discriminator.reward_function=FAIRL'])
  assert isinstance(cfg.training.learning_rate, float) and cfg.training.learning_rate == 3e-4
  assert cfg.imitation.nonnegative_margin == float('inf')
  assert cfg.steps == 1e5 and cfg.training.batch_size == 512 and isinstance(cfg.training.batch_size, int)
  assert cfg.imitation.spectral_norm is False and cfg.imitation.loss_function == 'PUGAIL' and cfg.imitation.discriminator.reward_function == 'FAIRL'
