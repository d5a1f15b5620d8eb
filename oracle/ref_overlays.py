"""TEST INFRASTRUCTURE ONLY — the reference's tuned RED / DRIL overlays as data.

`python -m oracle.ref_overlays` (needs the reference tree, see oracle/refstub.py) reads the reference's
conf/optimised_hyperparameters/{RED,DRIL}_{5,10,25}_trajectories.yaml, flattens each to dotted keys and writes
tests/golden/red_dril_overlays.json, which tests/test_sweep_red_dril_cpu.py compares the shipped overlays against. The tests only read that file.
"""
import json
import os

import yaml

from . import refstub
from .ref_golden import _flat_conf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PATH = os.path.join(ROOT, 'tests', 'golden', 'red_dril_overlays.json')
NAMES = [f'{alg}_{n}_trajectories' for alg in ('RED', 'DRIL') for n in (5, 10, 25)]


def load():
  """{overlay name: {dotted key: value}} as stored."""
  with open(PATH) as f: return json.load(f)


def main():
  out = {'_provenance': 'written by oracle/ref_overlays.py from the reference\'s conf/optimised_hyperparameters/{RED,DRIL}_{5,10,25}_trajectories.yaml '
                        '(flattened to dotted keys, values unchanged)'}
  for name in NAMES:
    with open(os.path.join(refstub.REFERENCE_DIR, 'conf', 'optimised_hyperparameters', f'{name}.yaml')) as f: out[name] = _flat_conf(yaml.safe_load(f) or {})
  with open(PATH, 'w') as f:
    json.dump(out, f, indent=1, sort_keys=True)
    f.write('\n')
  print(PATH)


if __name__ == '__main__':
  main()
