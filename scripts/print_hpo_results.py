"""Prints a hyper-parameter search's trials sorted by objective: the printing half of the reference's scripts/print_plot_hp_opt_results.py.

`python scripts/print_hpo_results.py --path <output_dir>/<ALG>_all_sweeper/<timestamp> [--out results.json] [--write-overlay best.yaml]`

For every trial directory <n>/ (overrides.yaml, <env>/metrics.pth for each env): min_avg_test_return = the minimum over envs of the mean of
test_returns_normalized over evaluations x (replicas x) episodes. Override keys that never vary (and `algorithm`) are dropped, as in the
reference. A trial with a non-finite mean on any env (a diverged run) scores NaN (numpy's min propagates it) and is listed last. --write-overlay
writes the best finite trial's values of every searched key (hpo.json's `searched` list, whether or not the key varied across trials) as a
conf/optimised_hyperparameters-style YAML, which `train.py optimised_hyperparameters=<name>` (with the file under
conf/optimised_hyperparameters/) or load_config reads.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import yaml

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import il_b200  # noqa: E402,F401
from il_b200.config import _parse  # noqa: E402
from il_b200.environments import ENVS  # noqa: E402


def min_avg_test_return(trial_dir):
  """The minimum over envs of the mean normalised test return (metrics.pth of a replicas=1 run: [T][episodes]; of R replicas: [T][R][episodes])."""
  m = np.min([np.mean(np.asarray(torch.load(os.path.join(trial_dir, env, 'metrics.pth'), weights_only=False)['test_returns_normalized'], dtype=np.float64)) for env in ENVS])
  return float(m) if np.isfinite(m) else float('nan')


def load(path):
  """[(trial number, {key: value string}, min_avg_test_return)] in trial order."""
  if not os.path.isdir(path): raise SystemExit(f'Output folder {path} does not exist')
  rows = []
  for name in sorted((e for e in os.listdir(path) if e.isdigit() and os.path.isdir(os.path.join(path, e))), key=int):
    with open(os.path.join(path, name, 'overrides.yaml')) as f: overrides = yaml.safe_load(f) or []
    values = dict(str(o).partition('=')[::2] for o in overrides if not str(o).startswith('algorithm='))
    rows.append((int(name), values, min_avg_test_return(os.path.join(path, name))))
  if not rows: raise SystemExit(f'{path}: no trial directories')
  return rows


def varying(rows):
  keys = []
  for _, v, _ in rows:
    for k in v:
      if k not in keys: keys.append(k)
  return [k for k in keys if len({r[1].get(k) for r in rows}) > 1]


def overlay(values):
  """Nested dict of dotted keys, values parsed as the command line parses them."""
  out = {}
  for k, v in values.items():
    node = out
    parts = k.lstrip('+').split('.')
    for p in parts[:-1]: node = node.setdefault(p, {})
    node[parts[-1]] = _parse(v)
  return out


def main(argv=None):
  ap = argparse.ArgumentParser(description='Print hyperparameter optimisation results')
  ap.add_argument('--path', type=str, required=True, help='Search output path (<ALG>_all_sweeper/<timestamp>)')
  ap.add_argument('--out', type=str, default='', help='Write the sorted table as JSON')
  ap.add_argument('--write-overlay', type=str, default='', help="Write the best trial's searched values as an optimised_hyperparameters YAML")
  args = ap.parse_args(argv)
  rows = load(args.path)
  keys = varying(rows)
  ranked = sorted(rows, key=lambda r: (np.isnan(r[2]), -r[2] if not np.isnan(r[2]) else 0.0, r[0]))  # NaN (diverged) trials last, in trial order
  table = [dict(trial=t, **{k: v.get(k) for k in keys}, min_avg_test_return=s) for t, v, s in ranked]
  cols = ['trial'] + keys + ['min_avg_test_return']
  width = {c: max(len(c), *(len(f'{r[c]:.6f}' if isinstance(r[c], float) else str(r[c])) for r in table)) for c in cols}
  print('  '.join(c.rjust(width[c]) for c in cols))
  for r in table: print('  '.join((f'{r[c]:.6f}' if isinstance(r[c], float) else str(r[c])).rjust(width[c]) for c in cols))
  if args.out:
    with open(args.out, 'w') as f: json.dump(table, f, indent=1)
  if args.write_overlay:
    record = os.path.join(args.path, 'hpo.json')
    if not os.path.isfile(record): raise SystemExit(f'--write-overlay needs {record}: it names the searched keys (the fixed overrides are not an overlay\'s)')
    with open(record) as f: searched = json.load(f)['searched']
    if np.isnan(ranked[0][2]): raise SystemExit('--write-overlay: every trial diverged on some env; there is no best trial')
    t, best, score = ranked[0]
    missing = [k for k in searched if k not in best]
    if missing: raise SystemExit(f'trial {t}: overrides.yaml lacks the searched key(s) {missing}')
    with open(args.write_overlay, 'w') as f:
      f.write(f'# Best trial ({t}, min_avg_test_return {score:.6f}) of the search under {os.path.abspath(args.path)}\n')
      yaml.safe_dump(overlay({k: best[k] for k in searched}), f, default_flow_style=None, sort_keys=False)
  return table


if __name__ == '__main__':
  main()
