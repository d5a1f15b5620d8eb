"""Build-container only: times the reference's REAL train.train() (oracle/ref_train.py) against the restated oracle loop
(oracle/loop.py, the `cpu_baseline` / `--impl reference` arm) on one CPU thread — GAIL hopper, B = 256, 200 update
steps after 300 update-free steps."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from il_b200 import config  # noqa: E402
from oracle import loop, ref_train  # noqa: E402


def reference_training_time(steps, start):
  cfg = config.load_config(['algorithm=GAIL', 'env=hopper', f'steps={steps}', f'training.start={start}', 'imitation.trajectories=5', f'evaluation.interval={10**9}',
                            'logging.interval=0', 'seed=0', 'check_time_usage=true'])
  for k in ('replicas', 'device_rng', 'cuda_graphs', 'gemm_mode', 'output_dir'): cfg.pop(k, None)
  raw = loop.synthesize_raw_dataset('hopper', True, 5, 1000)
  return ref_train.run_reference_train(cfg, raw, 1000)['metrics']['training_time']  # train.py:229 (loop only)


if __name__ == '__main__':
  torch.set_num_threads(1)
  prefill, total = reference_training_time(300, 301), reference_training_time(500, 301)
  ref = 200 / (total - prefill)
  mine = loop.measure_steps_per_second('GAIL', 'hopper', steps=200, warmup=5, seed=0, batch_size=256, prefill=300, threads=1)['steps_per_s']
  print(f'reference train(): {ref:.1f} steps/s; oracle loop: {mine:.1f} steps/s; ratio {mine / ref:.2f}')
