"""torch.optim.Adam / AdamW mirrors whose state lives next to the flat replica parameter buffers
(train.py:66,84). The step itself is fused into the update kernels (csrc/mlp.cu adam_kernel: the arithmetic of
torch's `_single_tensor_adam`, hyper-parameters kept in double like the Python floats they are).

`lr` and `weight_decay` are a float (every replica) or a length-R sequence (one value per replica of the flat buffer, for
hyper-parameter sweeps); a sequence is kept as a device float64 tensor and replica r owns floats [r n / R, (r + 1) n / R)."""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Optional, Sequence, Union

import torch
from torch import Tensor

from . import _lib


Hyper = Union[float, Sequence[float], Tensor]


class Adam:
  decoupled = False

  def __init__(self, params: Iterable[Tensor], lr: Hyper = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: Hyper = 0.0):
    params = list(params)
    assert len(params) == 1 and params[0].is_cuda, 'expects the single flat parameter tensor returned by module.parameters()'
    self.param = params[0]
    self.lr_r, self.weight_decay_r = self._per_replica(lr), self._per_replica(weight_decay)
    if not self.decoupled and (self.weight_decay_r is not None or weight_decay != 0):
      raise NotImplementedError('coupled (L2) weight decay is not used by the reference (train.py:66)')
    self.lr = 0.0 if self.lr_r is not None else float(lr)
    self.weight_decay = 0.0 if self.weight_decay_r is not None else float(weight_decay)
    self.betas, self.eps = betas, eps
    n = {t.numel() for t in (self.lr_r, self.weight_decay_r) if t is not None}
    assert len(n) <= 1, 'per-replica lr and weight_decay must have the same length'
    R = n.pop() if n else 0
    assert not R or self.param.numel() % R == 0, f'{R} replicas do not divide the {self.param.numel()}-float buffer'
    self.replica_floats = self.param.numel() // R if R else 0
    self.exp_avg, self.exp_avg_sq = torch.zeros_like(self.param), torch.zeros_like(self.param)
    self.step_count = torch.zeros(1, dtype=torch.int64, device=self.param.device)

  def _per_replica(self, x: Hyper) -> Optional[Tensor]:
    if isinstance(x, (int, float)): return None
    return torch.as_tensor(x, dtype=torch.float64).to(self.param.device).reshape(-1).contiguous()

  def c_struct(self) -> _lib.Adam:
    a = _lib.Adam()
    a.m, a.v, a.step = self.exp_avg.data_ptr(), self.exp_avg_sq.data_ptr(), self.step_count.data_ptr()
    a.lr, a.beta1, a.beta2, a.eps, a.weight_decay = self.lr, self.betas[0], self.betas[1], self.eps, self.weight_decay
    a.lr_r, a.weight_decay_r, a.replica_floats = _lib.ptr(self.lr_r), _lib.ptr(self.weight_decay_r), self.replica_floats
    return a

  def zero_grad(self, set_to_none: bool = True):
    pass  # gradients never persist between fused updates (training.py:29,40,47 zero them every call)

  def step_with(self, grads: Tensor):
    """One optimiser step from an explicit flat gradient (tests / custom losses)."""
    a = self.c_struct()
    _lib.check(_lib.lib().il_adam_step(_lib.handle(), self.param.data_ptr(), grads.contiguous().data_ptr(), C.byref(a), self.param.numel(), _lib.stream()))

  def state_dict(self):
    return dict(exp_avg=self.exp_avg.clone(), exp_avg_sq=self.exp_avg_sq.clone(), step=int(self.step_count.item()))


class AdamW(Adam):
  decoupled = True

  def __init__(self, params, lr: Hyper = 1e-3, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: Hyper = 1e-2):
    super().__init__(params, lr, betas, eps, weight_decay)
