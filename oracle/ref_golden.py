"""TEST INFRASTRUCTURE ONLY — stored results of the UNMODIFIED reference that the CPU tests compare against.

`python -m oracle.ref_golden` (needs the reference tree, see oracle/refstub.py) runs the reference's `train.train(cfg)` for every
configuration of tests/test_oracle_loop_pinned.py, its parameter initialisation for tests/test_host_logic.py and reads its conf tree, and
writes tests/golden/reference.npz. The tests only read that file. Everything train() wrote is stored whole. The 256-wide
initialisation tensors (630 k floats of random numbers) are stored as a fixed, seeded sample of entries plus the SHA-256 of their
bytes (`Sampled`): the test asks for bit equality, which the digest decides for every entry.
"""
import hashlib
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATH = os.path.join(ROOT, 'tests', 'golden', 'reference.npz')
INIT_SAMPLES = 8


def _np(v):
  return torch.as_tensor(v).detach().cpu().numpy()


def _hash(s):
  h = 0
  for ch in s: h = (h * 131 + ord(ch)) % (2 ** 61 - 1)
  return h


def sample_index(numel, n, tag):
  """Fixed sample of n flat indices of a tensor, seeded by its name."""
  return np.sort(np.random.default_rng(_hash(tag) % (2 ** 32)).choice(numel, n, replace=False))


def digest(arr):
  return hashlib.sha256(np.ascontiguousarray(arr, dtype='<f4').tobytes()).hexdigest()


class Sampled:
  """A reference float32 tensor known through `values` at the flat indices `idx`, the SHA-256 `sha` of its bytes and its `shape`."""

  def __init__(self, shape, idx, values, sha):
    self.shape, self.idx, self.values, self.sha = tuple(shape), idx, values, sha

  def check_equal(self, name, mine):
    mine = torch.as_tensor(mine).detach().cpu().numpy()
    assert tuple(mine.shape) == self.shape, (name, self.shape, tuple(mine.shape))
    assert np.array_equal(mine.reshape(-1)[self.idx], self.values), f'{name}: sampled entries differ'
    assert digest(mine) == self.sha, f'{name}: some entry differs (SHA-256 of the tensor)'


class _Writer:
  def __init__(self): self.f32, self.f64, self.index = [], [], {}

  def put(self, group, key, arr, samples=0):
    arr = np.asarray(arr)
    flat = arr.reshape(-1)
    if samples and flat.size > samples:
      assert arr.dtype == np.float32
      self.index.setdefault(group, []).append([key, list(arr.shape), 'float32', samples, digest(arr)])
      self.f32.append(flat[sample_index(flat.size, samples, key)])
    else:
      self.index.setdefault(group, []).append([key, list(arr.shape), str(arr.dtype), 0, ''])
      (self.f32 if arr.dtype == np.float32 else self.f64).append(flat.astype(np.float32 if arr.dtype == np.float32 else np.float64))

  def save(self, conf):
    blob = json.dumps(dict(index=list(self.index.items()), conf=conf), sort_keys=True, separators=(',', ':')).encode()
    np.savez_compressed(PATH, f32=np.concatenate(self.f32), f64=np.concatenate(self.f64), meta=np.frombuffer(blob, np.uint8))


_loaded = {}


def _load():
  if not _loaded:
    with np.load(PATH) as z:
      meta = json.loads(z['meta'].tobytes().decode())
      f32, f64 = z['f32'], z['f64']
    p32 = p64 = 0
    groups = {}
    for group, entries in meta['index']:  # write order = order of the values in the two pools
      out = groups.setdefault(group, {})
      for key, shape, dtype, samples, sha in entries:
        numel = int(np.prod(shape)) if shape else 1
        n = samples or numel
        if dtype == 'float32': vals, p32 = f32[p32:p32 + n], p32 + n
        else: vals, p64 = f64[p64:p64 + n], p64 + n
        out[key] = Sampled(shape, sample_index(numel, samples, key), vals, sha) if samples else vals.astype(dtype).reshape(shape)
    _loaded.update(groups=groups, conf=meta['conf'])
  return _loaded


def flatten_train_result(out):
  """run_reference_train()'s nested result as a flat, ordered dict of arrays (the pieces the loop tests compare)."""
  flat = {}
  for net, sd in out['agent'].items():
    if isinstance(sd, dict):
      for k, v in sd.items(): flat[f'agent|{net}|{k}'] = _np(v)
    else:
      flat[f'agent|{net}'] = _np(sd)
  for k, v in out.get('discriminator', {}).items(): flat[f'discriminator|{k}'] = _np(v)
  m = out['metrics']
  flat['metrics|train_returns'] = np.asarray([r[0] for r in m['train_returns']], dtype=np.float64)
  flat['metrics|update_steps'] = np.asarray(m['update_steps'], dtype=np.int64)
  for k in ('predicted_rewards', 'Q_values', 'entropies'):
    if len(m.get(k, [])): flat[f'metrics|{k}|last'] = _np(m[k][-1])
  if len(m.get('test_returns', [])): flat['metrics|test_returns|first'] = np.asarray(m['test_returns'][0], dtype=np.float64)
  flat['score'] = np.asarray(out['score'], dtype=np.float64)
  return flat


def load_train_result(case_id):
  """The stored result of the reference's train() for one test id, in the nested shape run_reference_train() returns (metrics: last /
  first entries only)."""
  flat = dict(_load()['groups'][f'train|{case_id}'])
  out = dict(agent={}, metrics={}, score=float(flat.pop('score')))
  tensor = lambda v: torch.from_numpy(np.asarray(v))
  for key, v in flat.items():
    parts = key.split('|')
    if parts[0] == 'agent' and len(parts) == 3: out['agent'].setdefault(parts[1], {})[parts[2]] = tensor(v)
    elif parts[0] == 'agent': out['agent'][parts[1]] = tensor(v)
    elif parts[0] == 'discriminator': out.setdefault('discriminator', {})[parts[1]] = tensor(v)
    elif key == 'metrics|train_returns': out['metrics']['train_returns'] = [[float(x)] for x in v]
    elif key == 'metrics|update_steps': out['metrics']['update_steps'] = [int(x) for x in v]
    elif key == 'metrics|test_returns|first': out['metrics']['test_returns'] = [v]
    else: out['metrics'][parts[1]] = [tensor(v)]
  return out


def load_init():
  """{'<replica>|<net>|<layer>|<weight or bias>': Sampled} of the reference's SoftActor / TwinCritic initialisation."""
  return _load()['groups']['init']


def load_conf():
  """{'<file under conf/>': flattened values} of the reference's conf tree."""
  return _load()['conf']


def _flat_conf(d, prefix=''):
  out = {}
  for k, v in d.items():
    if isinstance(v, dict): out.update(_flat_conf(v, f'{prefix}{k}.'))
    else: out[prefix + k] = v
  return out


def main():
  import yaml
  from . import loop, ref_train, refstub
  if not refstub.available(): sys.exit('reference tree not available; the fixtures can only be regenerated next to it')
  sys.path.insert(0, os.path.join(ROOT, 'tests'))
  import test_oracle_loop_pinned as T
  w = _Writer()
  runs = [(cid, T._cfg(alg, env, T.LOOP_SEED, extra), env) for cid, (alg, env, extra, _) in zip(T.CONFIG_IDS, T.CONFIGS)]
  runs += [(f'bc-{alg}-{it}', T._bc_cfg(alg, it), T.BC_ENV) for alg, it in T.BC_CONFIGS]
  for cid, cfg, env in runs:
    raw = loop.synthesize_raw_dataset(env, True, 5, T.MAX_EPISODE_STEPS)
    for key, arr in flatten_train_result(ref_train.run_reference_train(cfg, raw, T.MAX_EPISODE_STEPS)).items():
      w.put(f'train|{cid}', key, arr)
    print(cid)

  # parameter initialisation of the reference's SoftActor / TwinCritic (tests/test_host_logic.py)
  ref = refstub.load()
  S, A, H = 12, 3, 256
  mc = ref.DictConfig(hidden_size=H, depth=2, activation='relu')
  for r in range(3):
    torch.manual_seed(7 + r)
    actor, critic = ref.models.SoftActor(S, A, mc), ref.models.TwinCritic(S, A, mc)
    for net, seq in (('actor', actor.actor), ('critic_1', critic.critic_1.critic), ('critic_2', critic.critic_2.critic)):
      for l, lin in enumerate(m for m in seq if isinstance(m, torch.nn.Linear)):
        for kind, t in (('weight', lin.weight), ('bias', lin.bias)): w.put('init', f'{r}|{net}|{l}|{kind}', _np(t), INIT_SAMPLES)

  # the reference's conf tree, flattened (tests/test_host_logic.py)
  conf = {}
  def read(*parts):
    with open(os.path.join(refstub.REFERENCE_DIR, 'conf', *parts)) as f: return yaml.safe_load(f) or {}
  conf['train_config.yaml'] = _flat_conf(read('train_config.yaml'))
  for alg in ('SAC', 'GAIL', 'GMMIL', 'PWIL', 'BC'): conf[f'algorithm/{alg}.yaml'] = _flat_conf(read('algorithm', f'{alg}.yaml'))
  for alg in ('BC', 'GAIL', 'GMMIL', 'PWIL'):
    for n in (5, 10, 25): conf[f'optimised_hyperparameters/{alg}_{n}_trajectories.yaml'] = _flat_conf(read('optimised_hyperparameters', f'{alg}_{n}_trajectories.yaml'))
  w.save(conf)


if __name__ == '__main__':
  main()
