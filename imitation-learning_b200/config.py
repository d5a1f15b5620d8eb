"""Hydra-free loader for the reference's configuration surface (train.py:21-23, conf/): a base YAML, an
`algorithm=<ALG>` global overlay (`# @package _global_`), an optional `optimised_hyperparameters=<name>` overlay and
dotted `key=value` overrides — `python train.py algorithm=GAIL env=hopper training.batch_size=512` — and Hydra's basic multirun
sweeps (`-m key=a,b,...`, expand_sweep)."""
from __future__ import annotations

import copy
import itertools
import os
import re
from dataclasses import dataclass, field
from typing import Any, Dict, List, Optional, Sequence, Tuple

import yaml

from ._lib import MAX_WIDTH_CLASSES

CONF_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'conf')


class Config(dict):
  """Attribute-style nested dict (the subset of omegaconf.DictConfig the reference uses: attribute access, .get)."""

  def __getattr__(self, k):
    try:
      v = self[k]
    except KeyError:
      raise AttributeError(k)
    if isinstance(v, dict) and not isinstance(v, Config):
      v = Config(v)
      self[k] = v
    return v

  def __setattr__(self, k, v): self[k] = v

  def get(self, k, default=None):
    return getattr(self, k) if k in self else default


def _merge(dst: Dict[str, Any], src: Dict[str, Any]) -> Dict[str, Any]:
  for k, v in src.items():
    if isinstance(v, dict) and isinstance(dst.get(k), dict): _merge(dst[k], v)
    else: dst[k] = v
  return dst


def _parse(v: str) -> Any:
  """Override values the way Hydra's grammar reads them: ints, then floats (3e-4, 1e6, inf, nan — YAML 1.1 would hand
  these back as strings), then YAML for the rest (true / false / null / lists / quoted strings)."""
  t = v.strip()
  try:
    return int(t)
  except ValueError:
    pass
  try:
    return float(t)
  except ValueError:
    pass
  return yaml.safe_load(v)


def load_config(overrides: Optional[List[str]] = None, conf_dir: str = CONF_DIR) -> Config:
  overrides = list(overrides or [])
  for o in overrides:
    if o in MULTIRUN_FLAGS: raise SweepError(f'{o}: a multirun command line is expanded by expand_sweep(), one load_config() per job')
    _reject_sweep(o)
  with open(os.path.join(conf_dir, 'train_config.yaml')) as f: cfg = yaml.safe_load(f)
  groups = {'algorithm': cfg.get('algorithm', 'SAC'), 'optimised_hyperparameters': None}
  rest = []
  for o in overrides:
    k, _, v = o.partition('=')
    if k in groups: groups[k] = v
    else: rest.append((k, v))
  for g in ('algorithm', 'optimised_hyperparameters'):
    if groups[g] in (None, 'null', ''): continue
    path = os.path.join(conf_dir, g, f'{groups[g]}.yaml')
    if not os.path.exists(path):
      raise FileNotFoundError(f'no {g} config {groups[g]!r} under {conf_dir}')
    with open(path) as f: _merge(cfg, yaml.safe_load(f) or {})
  for k, v in rest:
    node = cfg
    parts = k.lstrip('+').split('.')
    for p in parts[:-1]: node = node.setdefault(p, {})
    node[parts[-1]] = _parse(v)
  return Config(cfg)


# ---- multirun (Hydra's basic sweeper) ------------------------------------------------------------------------------------------
MULTIRUN_FLAGS = ('-m', '--multirun')
# Scalars that leave every tensor shape unchanged: a sweep over them runs as per-replica values of one program (Trainer(per_replica=...)).
# Every other swept key is a grouping key: jobs that differ in one run as separate programs.
VECTORISED = ('training.learning_rate', 'training.weight_decay', 'reinforcement.discount', 'reinforcement.target_temperature', 'reinforcement.polyak_factor',
              'imitation.learning_rate', 'imitation.weight_decay', 'imitation.grad_penalty', 'imitation.entropy_bonus', 'bc_pretraining.learning_rate',
              'bc_pretraining.weight_decay')
# The GAIL discriminator's choices that leave every shape unchanged: per-replica values of the fused discriminator (csrc/gail.cu: one CTA per
# replica branches on them). The general discriminator (csrc/gail_general.cu) takes only the Mixup alpha per replica.
PER_REPLICA_DISCRIMINATOR = ('imitation.loss_function', 'imitation.discriminator.reward_function', 'imitation.spectral_norm', 'imitation.mixup_alpha',
                             'imitation.pos_class_prior', 'imitation.nonnegative_margin')
# The fused GAIL discriminator's hidden size: a per-replica shape (each replica keeps a single run's layout inside the stride of the widest; one
# launch per width class), with at most MAX_WIDTH_CLASSES distinct widths in one program. The general discriminator groups on it.
PER_REPLICA_WIDTH = ('imitation.discriminator.hidden_size', )
# Keys an algorithm never reads: jobs that differ only in them are the same run (GAILDiscriminator never passes its dropout to _create_fcnn,
# models.py:157-162), so they neither split groups nor become per-replica values.
UNUSED_KEYS = {'GAIL': ('imitation.discriminator.input_dropout', 'imitation.discriminator.dropout')}
# Other algorithms' own search-space keys that change no shape and no random draw: AdRIL's update frequency and balanced sampling
# (adril_relabel_kernel reads them per replica), PWIL's reward scale and bandwidth scale (pwil_reward_kernel), DRIL's quantile cutoff (the
# per-replica threshold q, computed once after pre-training). PWIL's scales are per replica only with imitation.mix_expert_data == 'none':
# with mixed_batch / prefill_memory the relabelling walk of train.py:136-140 writes scale-dependent rewards into the expert memory, which all
# replicas share, so there they stay grouping keys.
PER_REPLICA_ALGORITHM = {'AdRIL': ('imitation.update_freq', 'imitation.balanced'), 'PWIL': ('imitation.reward_scale', 'imitation.reward_bandwidth_scale'),
                         'DRIL': ('imitation.quantile_cutoff', )}
# The run's seed: per replica, every random stream of replica r is keyed by its own seed at replica-local indices (Trainer(per_replica={'seed': ...})),
# so replica r is the single run with that seed. It stays a grouping key where a stream cannot be split per replica: with device_rng false
# (the host numpy index stream is one per rank), and with imitation.subsample > 1 when the run builds an expert memory (get_dataset draws the
# subsampling offsets from the seeded numpy stream, and all replicas share that memory).
PER_REPLICA_SEED = ('seed', )
# RED's and DRIL's dropout rates and activation: per-replica values of the dropout program (csrc/dropout_nets.cu: the mask fill reads each replica's
# rate, the activation passes each replica's activation). Only whether a rate is 0 is structural (the nn.Sequential indices and state_dict keys,
# which mask draws happen, and for DRIL whether the dropout program runs at all), so sweep_groups groups on that presence (_dropout_presence) and
# Trainer(per_replica=...) refuses a mix of 0 and > 0 for one site. DRIL's activation is per replica only with a dropout site: without one the
# policy runs on the fused MLP kernels, which take one activation. Like `seed`, these keys are per replica in sweep_groups only (per_replica_keys).
PER_REPLICA_DROPOUT = ('imitation.discriminator.input_dropout', 'imitation.discriminator.dropout', 'imitation.discriminator.activation')
_ACTIVATIONS = ('relu', 'sigmoid', 'tanh')  # models.py:17 ACTIVATION_FUNCTIONS
_CHOICES = {'imitation.loss_function': ('BCE', 'Mixup', 'PUGAIL'), 'imitation.discriminator.reward_function': ('AIRL', 'FAIRL', 'GAIL')}
_SWEEP_FUNCTIONS = re.compile(r'^(range|choice|interval|glob|sort|shuffle|tag)\s*\(')


class SweepError(ValueError):
  pass


def _top_level_split(v: str) -> List[str]:
  """Splits an override value on the commas outside quotes, brackets and parentheses (Hydra's sweep syntax `a,b,c`)."""
  parts, depth, quote, cur = [], 0, None, ''
  for ch in v:
    if quote:
      quote = None if ch == quote else quote
    elif ch in '\'"':
      quote = ch
    elif ch in '[({':
      depth += 1
    elif ch in '])}':
      depth -= 1
    elif ch == ',' and depth == 0:
      parts.append(cur)
      cur = ''
      continue
    cur += ch
  return parts + [cur]


def _reject_sweep(o: str):
  """Outside a multirun, a sweep value is the ambiguity Hydra refuses."""
  k, _, v = o.partition('=')
  if _SWEEP_FUNCTIONS.match(v.strip()) or len(_top_level_split(v)) > 1:
    raise SweepError(f"Ambiguous value for argument '{o}'\n1. To use it as a list, use key=[value1,value2]\n2. To use it as string, quote the value: key=\'value1,value2\'\n"
                     '3. To sweep over it, add --multirun (-m) to your command line')


@dataclass
class SweepJob:
  num: int                          # job number (Hydra's hydra.job.num), from 0
  overrides: List[str]              # the job's full override list (swept keys with this job's value)


@dataclass
class SweepGroup:
  """Jobs that agree on every grouping key: one program with len(jobs) x `replicas` replicas, job j owning block j."""
  jobs: List[SweepJob]
  per_job: Dict[str, List[Any]] = field(default_factory=dict)  # vectorised swept key -> one parsed value per job

  @property
  def overrides(self) -> List[str]:
    return self.jobs[0].overrides


def expand_sweep(argv: Sequence[str]) -> Tuple[bool, List[SweepJob]]:
  """(multirun, jobs) of a command line. Without -m / --multirun: one job with the overrides as given (a comma list raises, as in Hydra).
  With it: the Cartesian product of the comma lists in Hydra's basic-sweeper order (overrides in the order given, the last varying
  fastest). range() / choice() / interval() / glob() sweeps are not supported; quoted values ('a,b') stay strings."""
  argv = list(argv)
  multirun = any(a in MULTIRUN_FLAGS for a in argv)
  overrides = [a for a in argv if a not in MULTIRUN_FLAGS]
  if not multirun:
    for o in overrides: _reject_sweep(o)
    return False, [SweepJob(0, overrides)]
  choices = []
  for o in overrides:
    k, eq, v = o.partition('=')
    if not eq: raise SweepError(f'override {o!r} is not key=value')
    if _SWEEP_FUNCTIONS.match(v.strip()):
      raise SweepError(f'{o}: only comma-separated sweeps (key=a,b,c) are supported, not {v.strip().split("(")[0]}()')
    vals = _top_level_split(v)
    if any(x.strip() == '' for x in vals) and len(vals) > 1: raise SweepError(f'{o}: empty sweep value')
    choices.append([f'{k}={x}' for x in vals])
  return True, [SweepJob(i, list(c)) for i, c in enumerate(itertools.product(*choices))]


def vectorised_keys(cfg: Config) -> Tuple[str, ...]:
  """VECTORISED minus the keys a path of this configuration cannot take per replica, plus the discriminator choices for GAIL and the
  algorithm's own keys of PER_REPLICA_ALGORITHM: the general GAIL discriminator (csrc/gail_general.cu) batches its gradient-penalty pass over
  replicas, so a replica with grad_penalty 0 would still take that pass's power iteration, and it takes only mixup_alpha of
  PER_REPLICA_DISCRIMINATOR; PWIL takes its scales per replica only without expert-data mixing (the expert memory's relabelled rewards
  depend on them and are shared)."""
  d = cfg.imitation.get('discriminator') or {}
  gail = cfg.get('algorithm') == 'GAIL'
  general = gail and bool(d.get('reward_shaping') or d.get('subtract_log_policy') or d.get('depth', 1) != 1 or d.get('activation', 'relu') != 'relu')
  keys = tuple(k for k in VECTORISED if not (general and k == 'imitation.grad_penalty'))
  if gail: keys += ('imitation.mixup_alpha', ) if general else PER_REPLICA_DISCRIMINATOR + PER_REPLICA_WIDTH
  alg = cfg.get('algorithm')
  if alg in PER_REPLICA_ALGORITHM and not (alg == 'PWIL' and cfg.imitation.get('mix_expert_data', 'none') != 'none'): keys += PER_REPLICA_ALGORITHM[alg]
  return keys


def per_replica_keys(cfg: Config) -> Tuple[str, ...]:
  """Every key Trainer(per_replica=...) takes in this configuration: vectorised_keys plus `seed` where it can be per replica (seed_per_replica)
  and RED's / DRIL's dropout keys (dropout_keys)."""
  return vectorised_keys(cfg) + (PER_REPLICA_SEED if seed_per_replica(cfg) else ()) + dropout_keys(cfg)


def dropout_keys(cfg: Config) -> Tuple[str, ...]:
  """The keys of PER_REPLICA_DROPOUT this configuration takes per replica: all three for RED; for DRIL the rates, and the activation when the
  policy has a dropout site."""
  alg = cfg.get('algorithm')
  if alg == 'RED': return PER_REPLICA_DROPOUT
  if alg != 'DRIL': return ()
  d = cfg.imitation.get('discriminator') or {}
  return PER_REPLICA_DROPOUT if any(_positive(d.get(k)) for k in ('input_dropout', 'dropout')) else PER_REPLICA_DROPOUT[:2]


def _positive(x: Any) -> bool:
  return isinstance(x, (int, float)) and not isinstance(x, bool) and x > 0


def _dropout_presence(cfg: Config, keys) -> Tuple:
  """Whether each dropout site whose rate is a per-replica key is present (rate > 0): the structural part of a rate, a grouping key."""
  d = cfg.imitation.get('discriminator') or {}
  return tuple((k, _positive(d.get(k.rsplit('.', 1)[1]))) for k in PER_REPLICA_DROPOUT[:2] if k in keys)


def needs_expert_memory(cfg: Config) -> bool:
  """Whether the run builds the expert memory (train.py:55-61; SAC only for BC pre-training or the BC auxiliary loss)."""
  return cfg.get('algorithm') != 'SAC' or cfg.bc_pretraining.get('iterations', 0) > 0 or bool(cfg.imitation.get('bc_aux_loss', False))


def seed_per_replica(cfg: Config) -> bool:
  """Whether `seed` can take per-replica values in this configuration (PER_REPLICA_SEED)."""
  return bool(cfg.get('device_rng', True)) and not (cfg.imitation.get('subsample', 1) > 1 and needs_expert_memory(cfg))


def group_jobs(jobs: List[SweepJob], conf_dir: str = CONF_DIR) -> List[SweepGroup]:
  """Partitions the jobs of a sweep: swept vectorised keys become per-job values, every other swept key (`seed` included) separates groups.
  Groups are ordered by their first job. Each group is one program with one seed, replica jR + k initialised from seed + jR + k."""
  return _partition(jobs, conf_dir, vectorised_keys)


def sweep_groups(jobs: List[SweepJob], conf_dir: str = CONF_DIR) -> List[SweepGroup]:
  """The programs a multirun runs (train.run_sweep): group_jobs' partition with `seed` a per-replica key where seed_per_replica holds, so
  groups that differ only in their seed are one program whose replicas draw their random numbers by their own seeds (per_replica_keys)."""
  return _partition(jobs, conf_dir, per_replica_keys)


def _partition(jobs: List[SweepJob], conf_dir: str, keys_of) -> List[SweepGroup]:
  """Jobs that agree on every swept key outside keys_of(config) form one group, in the order of their first job; the swept keys inside it
  become per-job values."""
  swept = {}
  for j in jobs:
    for o in j.overrides:
      k, _, v = o.partition('=')
      swept.setdefault(k, set()).add(v)
  swept = [k for k, vs in swept.items() if len(vs) > 1]
  groups: Dict[Tuple, SweepGroup] = {}
  for j in jobs:
    ov = dict(o.partition('=')[::2] for o in j.overrides)
    cfg = load_config(j.overrides, conf_dir)
    keys = keys_of(cfg)
    vec = set(keys) | set(UNUSED_KEYS.get(cfg.get('algorithm'), ()))
    key = tuple((k, ov.get(k)) for k in swept if k not in vec) + _dropout_presence(cfg, [k for k in swept if k in keys])
    g = groups.setdefault(key, SweepGroup([]))
    g.jobs.append(j)
  for g in groups.values():
    cfgs = [load_config(j.overrides, conf_dir) for j in g.jobs]
    vec = keys_of(cfgs[0])
    for k in swept:
      if k in vec: g.per_job[k] = [get_key(c, k) for c in cfgs]
    for k in PER_REPLICA_WIDTH: _check_width_classes(k, g.per_job.get(k, []))
  return list(groups.values())


def get_key(cfg: Dict[str, Any], dotted: str) -> Any:
  node = cfg
  for p in dotted.split('.'): node = node[p]
  return node


def set_key(cfg: Dict[str, Any], dotted: str, value: Any):
  parts = dotted.split('.')
  node = cfg
  for p in parts[:-1]: node = node[p]
  node[parts[-1]] = value


def _check_width_classes(k: str, vals: Sequence[Any]):
  n = len(set(vals))
  if n > MAX_WIDTH_CLASSES: raise SweepError(f'{k}: {n} distinct widths in one program; the fused discriminator takes at most {MAX_WIDTH_CLASSES}')


def _per_replica_value(k: str, x: Any) -> Any:
  """A per-replica value as the config holds it: a name of _CHOICES[k], a bool for spectral_norm, a positive int for a width, a non-negative
  int for a seed, a float otherwise."""
  if k in PER_REPLICA_WIDTH:
    if isinstance(x, bool) or not isinstance(x, int) or x <= 0: raise SweepError(f'{k}={x!r}: not a positive integer')
    return x
  if k in PER_REPLICA_SEED:  # np.random.seed (train.py:51) takes 0 <= seed < 2**32
    if isinstance(x, bool) or not isinstance(x, int) or not 0 <= x < 2**32: raise SweepError(f'{k}={x!r}: not an integer in [0, 2**32)')
    return x
  if k in _CHOICES:
    if x not in _CHOICES[k]: raise SweepError(f'{k}={x!r}: not one of {", ".join(_CHOICES[k])}')  # train.py:42,44
    return x
  if k == 'imitation.spectral_norm':
    if not isinstance(x, bool): raise SweepError(f'{k}={x!r}: not true / false')
    return x
  if isinstance(x, (bool, str)): raise SweepError(f'{k}={x!r}: not a number')
  return float(x)


def replica_values(k: str, per_job: Sequence[Any], R: int) -> List[Any]:
  """The J * R replica values of a group from its J job values: job j's value for each of its R replicas, except a seed, where replica i of
  job j takes s_j + i (a seed sweep with replicas=R runs each job as the replicas=R run of its seed)."""
  if k not in PER_REPLICA_SEED: return [v for v in per_job for _ in range(R)]
  return [_per_replica_value(k, s) + i for s in per_job for i in range(R)]


def _algorithm_value(k: str, x: Any, r: int) -> Any:
  """A value of PER_REPLICA_ALGORITHM for replica r, as the reference types or asserts it: update_freq an int >= 0 (train.py:37), balanced a
  bool, quantile_cutoff in [0, 1] (train.py:39), the PWIL scales numbers."""
  if k == 'imitation.update_freq':
    if isinstance(x, bool) or not isinstance(x, int) or x < 0: raise SweepError(f'replica {r}: {k}={x!r}: not an integer >= 0')
    return x
  if k == 'imitation.balanced':
    if not isinstance(x, bool): raise SweepError(f'replica {r}: {k}={x!r}: not true / false')
    return x
  if isinstance(x, bool) or not isinstance(x, (int, float)): raise SweepError(f'replica {r}: {k}={x!r}: not a number')
  if k == 'imitation.quantile_cutoff' and not 0 <= x <= 1: raise SweepError(f'replica {r}: {k}={x!r}: not in [0, 1]')
  return float(x)


def _dropout_value(k: str, x: Any, r: int) -> Any:
  """A value of PER_REPLICA_DROPOUT for replica r: an activation of models.py:17, or a rate in [0, 1) (nn.Dropout refuses p outside [0, 1], and
  p = 1 scales by 1 / 0; the scalar path refuses it too)."""
  if k == 'imitation.discriminator.activation':
    if x not in _ACTIVATIONS: raise SweepError(f'replica {r}: {k}={x!r}: not one of {", ".join(_ACTIVATIONS)}')
    return x
  if isinstance(x, bool) or not isinstance(x, (int, float)): raise SweepError(f'replica {r}: {k}={x!r}: not a number')
  if not 0 <= x < 1: raise SweepError(f'replica {r}: {k}={x!r}: not in [0, 1)')
  return float(x)


def _check_gail_replicas(cfg: Config, arrays: Dict[str, List[Any]], R: int):
  """The reference's GAIL asserts (train.py:42-47) for every replica: alpha > 0 for Mixup replicas, 0 <= prior <= 1 and margin >= 0 for PUGAIL ones."""
  val = lambda k, r: arrays[k][r] if k in arrays else get_key(cfg, k)
  for r in range(R):
    loss = val('imitation.loss_function', r)
    if loss == 'Mixup' and not val('imitation.mixup_alpha', r) > 0: raise SweepError(f'replica {r}: Mixup needs imitation.mixup_alpha > 0')
    if loss == 'PUGAIL':
      if not 0 <= val('imitation.pos_class_prior', r) <= 1: raise SweepError(f'replica {r}: PUGAIL needs 0 <= imitation.pos_class_prior <= 1')
      if not val('imitation.nonnegative_margin', r) >= 0: raise SweepError(f'replica {r}: PUGAIL needs imitation.nonnegative_margin >= 0')


def split_per_replica(cfg: Config, per_replica: Optional[Dict[str, Sequence[Any]]], R: int) -> Tuple[Config, Dict[str, List[Any]]]:
  """(config, arrays) for Trainer(per_replica=...): a key whose R values are all equal becomes that scalar in a copy of the config (the
  uniform path, bit for bit); the others stay per-replica lists. Keys outside per_replica_keys(cfg) and values the reference's asserts refuse
  (train.py:37-49, per replica) are refused."""
  cfg = copy.deepcopy(cfg)
  arrays = {}
  allowed = per_replica_keys(cfg)
  for k, vals in (per_replica or {}).items():
    if k not in allowed: raise SweepError(f'{k} cannot take per-replica values in this configuration (per-replica keys: {", ".join(allowed)})')
    per_alg = k in PER_REPLICA_ALGORITHM.get(cfg.get('algorithm'), ())
    vals = [_dropout_value(k, x, r) if k in PER_REPLICA_DROPOUT else _algorithm_value(k, x, r) if per_alg else _per_replica_value(k, x) for r, x in enumerate(vals)]
    if len(vals) != R: raise SweepError(f'{k}: {len(vals)} values for {R} replicas')
    if k in PER_REPLICA_WIDTH: _check_width_classes(k, vals)
    if k in PER_REPLICA_DROPOUT[:2] and len({x > 0 for x in vals}) > 1:
      raise SweepError(f'{k}: replicas mix rate 0 and rate > 0 ({vals}); whether a dropout site exists is a grouping key, only its rate is per replica')
    if all(x == vals[0] for x in vals): set_key(cfg, k, vals[0])
    else: arrays[k] = vals
  if cfg.get('algorithm') == 'GAIL': _check_gail_replicas(cfg, arrays, R)
  return cfg, arrays
