"""Times the dense-layer grouped GEMM (the dominant kernel) in isolation for the three operand layouts and engines, at
G = 1024 (actor) and G = 2048 (twin critic) groups of 256 x 256 x 256, and sets each time against its floor at H100 SXM
data-sheet rates: the larger of algorithmic bytes / 3.35 TB/s and MMA work / 495 TFLOP/s dense TF32 (3 MMAs per
product for tf32x3). The card name, power limit and maximum SM clock are printed with the numbers.
Usage: python scripts/gemm_probe.py [G ...] [mode ...]"""
import os
import subprocess
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import il_b200
from il_b200 import _lib

HBM_BPS, TF32_FLOPS = 3.35e12, 495e12  # H100 SXM data sheet (not measured rates)
args = sys.argv[1:]
Gs = [int(a) for a in args if a.isdigit()] or [1024, 2048]
modes = [a for a in args if not a.isdigit()] or ['fp32', 'tf32x3', 'tf32']
M = N = K = 256
lib, h = _lib.lib(), _lib.handle()
flush = torch.empty(64 * 1024 * 1024, device='cuda')  # 256 MB > L2


def card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', str(torch.cuda.current_device())],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError) as e:
    return f'nvidia-smi unavailable ({e})'


def run(G, X, W, Cm, bias, mode, layout, iters=5):
  _lib.check(lib.il_set_gemm_mode(h, _lib.GEMM_MODE[mode]))
  ak, bk = {'fwd': (1, 1), 'dx': (1, 0), 'dw': (0, 0)}[layout]
  ts = []
  for i in range(iters + 2):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    _lib.check(lib.il_debug_gemm(h, M, N, K, G, X.data_ptr(), X.stride(0), K, ak, W.data_ptr(), W.stride(0), K, bk, Cm.data_ptr(), Cm.stride(0), N, bias.data_ptr() if layout == 'fwd' else None,
                                 N, 0 if layout == 'fwd' else -1, None, 0, N, 0, None, 0, _lib.stream()))
    e1.record()
    torch.cuda.synchronize()
    if i >= 2: ts.append(e0.elapsed_time(e1))
  ms = sorted(ts)[len(ts) // 2]
  flops = 2.0 * M * N * K * G
  nbytes = 4.0 * G * (M * K + N * K + M * N + (N if layout == 'fwd' else 0))  # A + B + C (+ bias): each read or written once
  mma = {'tf32x3': 3, 'tf32': 1}.get(mode)
  floor = max(nbytes / HBM_BPS, mma * flops / TF32_FLOPS if mma else 0.0) * 1e3
  line = f'{mode:7s} {layout:4s} G={G}: {ms:.3f} ms  {nbytes / ms / 1e6:7.1f} GB/s  {flops / ms / 1e9:6.1f} TFLOP/s'
  if mma: line += f'  ({mma * flops / ms / 1e9:5.1f} TFLOP/s of tf32 MMAs)  floor {floor:.3f} ms = {floor / ms:.0%} of this time'
  print(line, flush=True)


print('card (name, power.limit, clocks.max.sm):', card(), flush=True)
for G in Gs:
  X = torch.randn(G, M, K, device='cuda')
  W = torch.randn(G, N, K, device='cuda') / 16
  Cm = torch.empty(G, M, N, device='cuda')
  bias = torch.randn(G, N, device='cuda')
  for mode in modes:
    for layout in ('fwd', 'dx', 'dw'): run(G, X, W, Cm, bias, mode, layout)
  del X, W, Cm, bias
