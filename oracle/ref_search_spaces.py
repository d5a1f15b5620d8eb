"""TEST INFRASTRUCTURE ONLY — the reference's hyper-parameter search spaces as data.

`python -m oracle.ref_search_spaces` (needs the reference tree, see oracle/refstub.py) reads the reference's
conf/hyperparameter_search_space/<ALG>.yaml, resolves each file's `defaults: [SAC]` the way Hydra composes it (the listed file's params
first, then the file's own) and writes tests/golden/hp_search_spaces.json: {ALG: {key: {type, bounds | values, value_type}}} in the composed
key order. tests/test_hpo_cpu.py compares the shipped conf/hyperparameter_search_space files against it. The tests only read that file.
"""
import json
import os

import yaml

from . import refstub

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATH = os.path.join(ROOT, 'tests', 'golden', 'hp_search_spaces.json')
ALGORITHMS = ('AdRIL', 'BC', 'DRIL', 'GAIL', 'GMMIL', 'PWIL', 'RED', 'SAC')


def load():
  """{algorithm: {key: spec}} as stored."""
  with open(PATH) as f: return json.load(f)


def _composed(alg):
  with open(os.path.join(refstub.REFERENCE_DIR, 'conf', 'hyperparameter_search_space', f'{alg}.yaml')) as f: d = yaml.safe_load(f) or {}
  params = {}
  for base in d.get('defaults', []): params.update(_composed(base))
  params.update(d.get('params', {}))
  return params


def main():
  out = {'_provenance': 'written by oracle/ref_search_spaces.py from the reference\'s conf/hyperparameter_search_space/*.yaml (defaults composed, '
                        'values unchanged)'}
  for alg in ALGORITHMS: out[alg] = _composed(alg)
  with open(PATH, 'w') as f:
    json.dump(out, f, indent=1)
    f.write('\n')
  print(PATH)


if __name__ == '__main__':
  main()
