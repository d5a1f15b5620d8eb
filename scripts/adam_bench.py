"""AdamW (+ fused polyak) streaming kernel variants on the flat parameter buffers of the bench workload (critic: 2 nets x 1024 replicas, 9 streams with
the target update; actor: 7 streams), against a plain device copy of the same number of bytes. CUDA events, L2 flushed between launches.
  python scripts/adam_bench.py > adam_variants.jsonl"""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import il_b200
from il_b200 import _lib

flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')


def timed(fn, iters=12, warmup=3):
  for _ in range(warmup): fn()
  ms = []
  for _ in range(iters):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    ms.append(e0.elapsed_time(e1))
  ms.sort()
  return ms[len(ms) // 2]


def main():
  lib, h = _lib.lib(), _lib.handle()
  R = 1024
  sizes = dict(critic=(2 * (15 * 256 + 256 + 256 * 256 + 256 + 256 + 4), True), actor=(12 * 256 + 256 + 256 * 256 + 256 + 6 * 256 + 8, False))
  for name, (per, polyak) in sizes.items():
    n = (R * per + 3) // 4 * 4
    p, g, t = torch.randn(n, device='cuda') * 0.1, torch.randn(n, device='cuda') * 0.01, torch.randn(n, device='cuda') * 0.1
    opt = il_b200.AdamW([p.view(1, -1)], lr=3e-4, weight_decay=0.0)
    st = opt.c_struct()
    streams = 9 if polyak else 7
    nbytes = streams * n * 4
    a, b = torch.empty(nbytes // 2, dtype=torch.uint8, device='cuda'), torch.empty(nbytes // 2, dtype=torch.uint8, device='cuda')
    ms = timed(lambda: b.copy_(a))
    print(json.dumps(dict(kernel='torch copy (read + write, same total bytes)', buffer=name, bytes=nbytes, ms=ms, gbs=nbytes / ms / 1e6)), flush=True)
    del a, b
    for variant in (0, 1, 2, 3, 4, 5, 6, 7):
      _lib.set_option('adam_tma', variant)
      def run():
        if polyak: _lib.check(lib.il_adam_step_polyak(h, p.data_ptr(), g.data_ptr(), C.byref(st), n, t.data_ptr(), 0.995, _lib.stream()))
        else: _lib.check(lib.il_adam_step(h, p.data_ptr(), g.data_ptr(), C.byref(st), n, _lib.stream()))
      ms = timed(run)
      label = {0: 'adam_kernel (LSU, 128-bit)', 1: 'tma tile 2048 x 2 stages, 2 CTA/SM', 2: 'tma 4096 x 2, 1 CTA/SM', 3: 'tma 2048 x 3, 1 CTA/SM', 4: 'tma 1024 x 4, 2 CTA/SM', 5: 'tma 1024 x 3, 3 CTA/SM',
               6: 'tma 512 x 4, 4 CTA/SM', 7: 'tma 2048 x 4, 1 CTA/SM'}[variant]
      print(json.dumps(dict(kernel=label, option=f'adam_tma={variant}', buffer=name, streams=streams, bytes=nbytes, ms=ms, gbs=nbytes / ms / 1e6)), flush=True)
  _lib.set_option('adam_tma', 1)


if __name__ == '__main__':
  main()
