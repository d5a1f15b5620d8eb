"""Prints the seed-sweep results the reference publishes (its scripts/print_plot_seed_sweep_results.py, without the figure): per
trajectory count and algorithm, the final IQM of the normalised test return over runs x envs with the half-width of its 95 %
stratified-bootstrap interval. The statistics run on the GPU (il_b200.results). `--out` writes the point and interval curves, the data of
the reference's figure, as JSON.

Each (algorithm, env, trajectories) cell is one sweep directory holding a job directory <n>/metrics.pth per job, as `train.py -m ...
seed=1,...,10` writes it; a job of replicas=R contributes R runs.

  python scripts/print_seed_sweep_results.py --algorithms GAIL --envs hopper,walker2d --trajectories 5 \\
      --path 'outputs/{algorithm}_{env}_sweeper/*' --out results.json
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ALGORITHMS = ['BC', 'AdRIL', 'DRIL', 'GAIL', 'GMMIL', 'PWIL', 'RED']
TRAJECTORIES = ['5', '10', '25']
DEFAULT_PATH = os.path.join('outputs', '{algorithm}_{env}_sweeper', 'traj_{trajectories}')
_split = lambda s: [x for x in s.split(',') if x]


def parse_args(argv=None):
  from il_b200.environments import ENVS
  p = argparse.ArgumentParser(description='Print seed sweep results')
  p.add_argument('--reps', type=int, default=50000, help='Number of bootstrap samples')
  p.add_argument('--algorithms', type=_split, default=ALGORITHMS, help='Algorithms to evaluate')
  p.add_argument('--envs', type=_split, default=ENVS, help='Envs to evaluate')
  p.add_argument('--seeds', type=int, default=10, help='Max number of seeds to evaluate')
  p.add_argument('--unnormalise', action=argparse.BooleanOptionalAction, help='Use unnormalised returns')
  p.add_argument('--trajectories', type=_split, default=None, help='Expert trajectory counts (default 5,10,25; 0 when SAC is evaluated)')
  p.add_argument('--path', default=DEFAULT_PATH, help='Sweep directory of one cell: a pattern with {algorithm}, {env}, {trajectories} and optional glob '
                 'wildcards that must match exactly one directory')
  p.add_argument('--bootstrap-seed', type=int, default=0, help='Key of the device bootstrap draws')
  p.add_argument('--out', default=None, help='JSON file for the point and interval curves')
  args = p.parse_args(argv)
  if args.reps < 1: p.error('--reps must be positive')
  if args.seeds < 1: p.error('--seeds must be positive')
  if not 0 <= args.bootstrap_seed < 2**64: p.error('--bootstrap-seed must be in [0, 2^64)')
  if args.trajectories is None: args.trajectories = ['0'] if 'SAC' in args.algorithms else TRAJECTORIES  # the reference's SAC special case
  return args


def main(argv=None):
  args = parse_args(argv)
  from il_b200 import results
  out = dict(reps=args.reps, confidence=0.95, bootstrap_seed=args.bootstrap_seed, seeds=args.seeds, envs=args.envs, unnormalise=bool(args.unnormalise), trajectories={})
  print('IQM ± 1 C.I.')
  for trajectories in args.trajectories:
    score_dict, steps, dirs = {}, {}, {}
    for algorithm in args.algorithms:
      dirs[algorithm] = [results.resolve_sweep_dir(args.path, algorithm, env, trajectories) for env in args.envs]
      steps[algorithm], score_dict[algorithm] = results.load_score_matrix(dirs[algorithm], args.seeds, bool(args.unnormalise))
    points, intervals = results.get_interval_estimates(score_dict, reps=args.reps, seed=args.bootstrap_seed)
    print(f'\nTrajectories: {trajectories}')
    cell = out['trajectories'][trajectories] = {}
    for algorithm in args.algorithms:
      ci = intervals[algorithm]
      print(f'{algorithm}: {points[algorithm][-1]:.2f} ± {(ci[1, -1] - ci[0, -1]) / 2:.2f}')
      cell[algorithm] = dict(steps=steps[algorithm], iqm=points[algorithm].tolist(), ci_low=ci[0].tolist(), ci_high=ci[1].tolist(), dirs=dirs[algorithm])
  if args.out:
    with open(args.out, 'w') as f: json.dump(out, f, indent=1)
  return out


if __name__ == '__main__':
  main()
