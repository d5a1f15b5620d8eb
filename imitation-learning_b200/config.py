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
  """VECTORISED minus the keys a path of this configuration cannot take per replica, plus the discriminator choices for GAIL: the general GAIL
  discriminator (csrc/gail_general.cu) batches its gradient-penalty pass over replicas, so a replica with grad_penalty 0 would still take that
  pass's power iteration, and it takes only mixup_alpha of PER_REPLICA_DISCRIMINATOR."""
  d = cfg.imitation.get('discriminator') or {}
  gail = cfg.get('algorithm') == 'GAIL'
  general = gail and bool(d.get('reward_shaping') or d.get('subtract_log_policy') or d.get('depth', 1) != 1 or d.get('activation', 'relu') != 'relu')
  keys = tuple(k for k in VECTORISED if not (general and k == 'imitation.grad_penalty'))
  if gail: keys += ('imitation.mixup_alpha', ) if general else PER_REPLICA_DISCRIMINATOR + PER_REPLICA_WIDTH
  return keys


def group_jobs(jobs: List[SweepJob], conf_dir: str = CONF_DIR) -> List[SweepGroup]:
  """Partitions the jobs of a sweep: swept vectorised keys become per-job values, every other swept key separates groups. Groups are
  ordered by their first job."""
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
    vec = set(vectorised_keys(cfg)) | set(UNUSED_KEYS.get(cfg.get('algorithm'), ()))
    key = tuple((k, ov.get(k)) for k in swept if k not in vec)
    g = groups.setdefault(key, SweepGroup([]))
    g.jobs.append(j)
  for g in groups.values():
    cfgs = [load_config(j.overrides, conf_dir) for j in g.jobs]
    vec = vectorised_keys(cfgs[0])
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
  """A per-replica value as the config holds it: a name of _CHOICES[k], a bool for spectral_norm, a positive int for a width, a float otherwise."""
  if k in PER_REPLICA_WIDTH:
    if isinstance(x, bool) or not isinstance(x, int) or x <= 0: raise SweepError(f'{k}={x!r}: not a positive integer')
    return x
  if k in _CHOICES:
    if x not in _CHOICES[k]: raise SweepError(f'{k}={x!r}: not one of {", ".join(_CHOICES[k])}')  # train.py:42,44
    return x
  if k == 'imitation.spectral_norm':
    if not isinstance(x, bool): raise SweepError(f'{k}={x!r}: not true / false')
    return x
  if isinstance(x, (bool, str)): raise SweepError(f'{k}={x!r}: not a number')
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
  uniform path, bit for bit); the others stay per-replica lists. Keys outside vectorised_keys(cfg) and values the reference's asserts refuse
  (train.py:42-49, per replica for GAIL) are refused."""
  cfg = copy.deepcopy(cfg)
  arrays = {}
  allowed = vectorised_keys(cfg)
  for k, vals in (per_replica or {}).items():
    if k not in allowed: raise SweepError(f'{k} cannot take per-replica values in this configuration (per-replica keys: {", ".join(allowed)})')
    vals = [_per_replica_value(k, x) for x in vals]
    if len(vals) != R: raise SweepError(f'{k}: {len(vals)} values for {R} replicas')
    if k in PER_REPLICA_WIDTH: _check_width_classes(k, vals)
    if all(x == vals[0] for x in vals): set_key(cfg, k, vals[0])
    else: arrays[k] = vals
  if cfg.get('algorithm') == 'GAIL': _check_gail_replicas(cfg, arrays, R)
  return cfg, arrays
