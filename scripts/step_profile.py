"""Per-kernel durations INSIDE the running step (CUPTI activity records through torch.profiler: no serialisation, no cache flush, the
CUDA graph replays as in bench.py) — the complement of the ncu launch list, whose per-launch times are cold and serialised.
  python scripts/step_profile.py [steps] > step_kernel_times.json"""
import collections
import json
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from torch.profiler import ProfilerActivity, profile

import il_b200  # noqa: F401
from il_b200.config import load_config
from il_b200.train import Trainer


def main():
  K = int(sys.argv[1]) if len(sys.argv) > 1 else 10
  R, start = 1024, 30
  cfg = load_config(['algorithm=GAIL', 'env=hopper', 'steps=100000', f'training.start={start}', 'training.batch_size=256', 'imitation.trajectories=5', f'replicas={R}', 'gemm_mode=tf32x3',
                     'memory.size=4096', 'seed=0'])
  tr = Trainer(cfg, replicas=R, fast_init=True)
  for _ in range(start + 8): tr.train_step()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(K): tr.train_step()
  e1.record(); torch.cuda.synchronize()
  plain_ms = e0.elapsed_time(e1) / K
  with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(K): tr.train_step()
    torch.cuda.synchronize()
  agg = collections.OrderedDict()
  trace = os.path.join(os.environ.get('TMPDIR', '/tmp'), 'il_step_trace.json')
  prof.export_chrome_trace(trace)  # kernels launched by the library (and replayed from graphs) carry their names in the trace's "kernel" category
  for ev in json.load(open(trace))['traceEvents']:
    if ev.get('cat') != 'kernel': continue
    name = re.sub(r'\(.*', '', ev['name'].replace('(anonymous namespace)::', '').replace('<unnamed>::', '')).replace('void ', '')
    a = agg.setdefault(name, [0, 0.0])
    a[0] += 1
    a[1] += float(ev['dur'])
  total = sum(v[1] for v in agg.values())
  rows = sorted(agg.items(), key=lambda kv: -kv[1][1])
  out = dict(how='torch.profiler (CUPTI kernel activity) over %d graph-replayed steps of the bench.py workload (GAIL hopper, R=1024, B=256, tf32x3)' % K, steps=K,
             ms_per_step_without_profiler=plain_ms, kernel_ms_per_step=total / K / 1e3,
             kernels=[dict(kernel=n, launches_per_step=c / K, us_per_step=round(t / K, 1), share=round(t / total, 4)) for n, (c, t) in rows])
  print(json.dumps(out, indent=1))


if __name__ == '__main__':
  main()
