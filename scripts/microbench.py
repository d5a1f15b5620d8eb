"""Kernel micro-benchmarks asked for by SURVEY §8d beyond the headline loop: the GMMIL pairwise-RBF reward at B = 256 and B = 1024 (halfcheetah,
1024 replicas), the PWIL coupling step, the GAIL update and the evaluation rollout. CUDA events, L2 flushed between timed launches, JSON lines.
  python scripts/microbench.py > microbench.jsonl"""
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import il_b200
from il_b200 import _lib
from il_b200.memory import TransitionBatch

FP32_PEAK = 132 * 128 * 2 * 1.98e9 / 1e12  # TFLOP/s: 132 SMs x 128 FMA lanes x 2 flop x 1.98 GHz (non-tensor fp32, H100 SXM)
flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')


def timed(fn, iters=10, warmup=3):
  for _ in range(warmup): fn()
  ms = []
  for _ in range(iters):
    flush.zero_()  # > 50 MB L2
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    torch.cuda.synchronize()
    ms.append(e0.elapsed_time(e1))
  ms.sort()
  return ms[len(ms) // 2]


def batch(R, B, S, A):
  _, row = _lib.py_row_layout(S, A)
  rows = torch.randn(R, B, row, device='cuda')
  rows[..., S - 1] = 0
  tb = TransitionBatch(rows, S, A, True)
  tb.rows[..., tb.off['weights']] = 1.0
  return tb


class Cfg(dict):
  __getattr__ = dict.__getitem__
  def get(self, k, d=None): return dict.get(self, k, d)


def main():
  R = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
  out = []
  for B in (256, 1024):  # GMMIL halfcheetah (SURVEY §8d config 3 and its B = 1024 microbench)
    S, A = 18, 6
    d = il_b200.GMMILDiscriminator(S, A, Cfg(state_only=False), replicas=R)
    p, e = batch(R, B, S, A), batch(R, B, S, A)
    d.predict_reward_batch(p, e)  # sets the bandwidths
    rew = torch.empty(R, B, device='cuda')
    ms = timed(lambda: d.predict_reward_batch(p, e, reward_out=rew))
    mac = 2.0 * B * B * (S + A) * R  # two distance matrices (policy-expert, policy-policy)
    exps = 4.0 * B * B * R
    out.append(dict(kernel='gmmil_kernel', config=f'halfcheetah R={R} B={B}', ms=ms, algorithmic_gflop=2 * mac / 1e9, exp_evaluations=exps, tflops=2 * mac / ms / 1e9,
                    frac_of_fp32_peak=2 * mac / ms / 1e9 / FP32_PEAK, fp32_peak_tflops=FP32_PEAK, bytes=2 * R * B * (S + A) * 4 + 3 * R * B * 4,
                    bound='FMA + SFU (SURVEY §8d: not HBM, not tensor)'))
  # PWIL hopper: N_e expert atoms, one agent atom per replica per env step
  S, A, N = 12, 3, 5000
  z = torch.zeros
  mem = il_b200.ReplayMemory(N, S, A, True, transitions=dict(states=torch.randn(N, S), actions=torch.tanh(torch.randn(N, A)), rewards=z(N), next_states=z(N, S), terminals=z(N),
                                                            timeouts=z(N), weights=torch.ones(N), num_trajectories=5), shared=True)
  Rp = min(R, 256)
  pw = il_b200.PWILDiscriminator(S, A, Cfg(state_only=False, reward_scale=5, reward_bandwidth_scale=5), mem, 1000, replicas=Rp)
  st, ac, rw = torch.randn(Rp, S, device='cuda'), torch.tanh(torch.randn(Rp, A, device='cuda')), torch.empty(Rp, device='cuda')
  ms = timed(lambda: pw.compute_reward_batch(st, ac, out=rw))
  out.append(dict(kernel='pwil_reward_kernel', config=f'hopper R={Rp} N_e={N}', ms=ms, algorithmic_gflop=2.0 * N * (S + A) * Rp / 1e9, bytes=N * (S + A + 2) * 4 * 1.0 + Rp * N * 4 * 2,
                  gbs=(N * (S + A) * 4 + Rp * N * 4 * 2) / ms / 1e6, bound='latency (block arg-min rounds per consumed atom)'))
  # GAIL update (default config) — the register-tiled kernel vs the first kernel
  S, A, B = 12, 3, 256
  icfg = Cfg(state_only=False, spectral_norm=True, loss_function='BCE', grad_penalty=1.0, mixup_alpha=1, entropy_bonus=0.0, pos_class_prior=0.7, nonnegative_margin=float('inf'),
             discriminator=Cfg(hidden_size=64, depth=1, activation='relu', input_dropout=0.5, dropout=0.75, reward_shaping=False, subtract_log_policy=False, reward_function='AIRL'))
  disc = il_b200.GAILDiscriminator(S, A, icfg, 0.97, replicas=1)
  disc.mlp.flat = disc.mlp.flat.expand(R, -1).contiguous(); disc.mlp.replicas = disc.replicas = R
  disc.u, disc.v = disc.u.expand(R, -1).contiguous(), disc.v.expand(R, -1).contiguous()
  opt = il_b200.AdamW(disc.parameters(), lr=3e-5, weight_decay=10)
  pol, exp = batch(R, B, S, A), batch(R, B, S, A)
  eps = torch.rand(R, B, device='cuda')
  disc.train()
  for tiled in (0, 1):
    _lib.set_option('gail_tiled', tiled)
    ms = timed(lambda: il_b200.adversarial_imitation_update(None, disc, pol, exp, opt, icfg, eps_gp=eps))
    mac = 11.0 * ((S + A) * 64 + 64) * B * R  # SURVEY §8d: 11 W_d MAC per sample
    out.append(dict(kernel='gail_update_tiled_kernel' if tiled else 'gail_update_kernel', config=f'hopper R={R} B={B} H=64 (BCE + GP + SN)', ms=ms, algorithmic_gflop=2 * mac / 1e9,
                    tflops=2 * mac / ms / 1e9, frac_of_fp32_peak=2 * mac / ms / 1e9 / FP32_PEAK))
  _lib.set_option('gail_tiled', 1)
  for o in out: print(json.dumps(o), flush=True)


if __name__ == '__main__':
  main()
