"""Replica-batched flat-parameter MLPs: the device-side storage behind SoftActor / TwinCritic / discriminators.

Layout (include/il_b200.h `il_mlp`): parameters of G nets in one [G, stride] fp32 buffer; per net, per layer the
weight [out, in] (row-major) then the bias, each starting on a 4-float boundary — the order of
`nn.Module.parameters()` for the reference's `_create_fcnn` (models.py:48-69), so optimiser state lines up.
"""
from __future__ import annotations

import contextlib
import ctypes as C
from typing import Dict, List, Optional, Sequence

import torch
from torch import Tensor, nn

from . import _lib


class ReplicaRNG:
  """Per-replica CPU RNG streams so that replica r initialises exactly like a reference run with seed + r
  (train.py:51-52 seeds the global torch RNG once; constructors then draw from it in order)."""

  def __init__(self, seed: int, replicas: int):
    self.states = []
    for r in range(replicas):
      g = torch.Generator()
      g.manual_seed(seed + r)
      self.states.append(g.get_state())

  @classmethod
  def repeated(cls, state: Tensor, replicas: int) -> 'ReplicaRNG':
    """Every replica starts from the same CPU RNG state: replica r draws what a single run constructed from `state` draws (Trainer(fast_init=True)
    with per-replica discriminator widths)."""
    rng = cls(0, 0)
    rng.states = [state.clone() for _ in range(replicas)]
    return rng

  @contextlib.contextmanager
  def replica(self, r: int):
    saved = torch.get_rng_state()
    torch.set_rng_state(self.states[r])
    try:
      yield
    finally:
      self.states[r] = torch.get_rng_state()
      torch.set_rng_state(saved)


@contextlib.contextmanager
def _null_ctx():
  yield


def init_fcnn_params(sizes: Sequence[int], activation: str, final_gain: float = 1.0) -> List[Tensor]:
  """CPU initialisation with the reference's RNG consumption (models.py:52-66): nn.Linear's own reset draws,
  then orthogonal_ (gain from the activation; `final_gain` for the head) and zero bias."""
  out = []
  for l in range(len(sizes) - 1):
    layer = nn.Linear(sizes[l], sizes[l + 1])
    gain = nn.init.calculate_gain(activation) if l < len(sizes) - 2 else final_gain
    nn.init.orthogonal_(layer.weight, gain=gain)
    nn.init.constant_(layer.bias, 0)
    out += [layer.weight.detach(), layer.bias.detach()]
  return out


class ReplicaMLP:
  """G = replicas * nets_per_replica independent MLPs in one flat device buffer."""

  def __init__(self, dims: Sequence[int], activation: str, replicas: int, nets_per_replica: int = 1, device: Optional[torch.device] = None):
    assert activation in _lib.ACT, activation
    assert 2 <= len(dims) <= _lib.MAX_LAYERS + 1
    self.dims, self.activation, self.replicas, self.nets = list(dims), activation, replicas, nets_per_replica
    self.w_off, self.b_off, self.stride = _lib.py_mlp_offsets(self.dims)
    self.device = torch.device('cuda') if device is None else torch.device(device)
    self.flat = torch.zeros(replicas, nets_per_replica * self.stride, device=self.device, dtype=torch.float32)

  @property
  def n_layers(self) -> int: return len(self.dims) - 1

  @property
  def groups(self) -> int: return self.replicas * self.nets

  def c_struct(self, flat: Optional[Tensor] = None) -> _lib.Mlp:
    m = _lib.Mlp()
    m.params = (self.flat if flat is None else flat).data_ptr()
    m.stride, m.n_layers, m.activation = self.stride, self.n_layers, _lib.ACT[self.activation]
    for i, d in enumerate(self.dims): m.dims[i] = d
    return m

  def layer_views(self, flat: Optional[Tensor] = None) -> List[List[Tensor]]:
    """views[net][2*l] = W_l [R, out, in], views[net][2*l+1] = b_l [R, out] (views into the flat buffer)."""
    flat = self.flat if flat is None else flat
    out = []
    for n in range(self.nets):
      vs, base = [], n * self.stride
      for l in range(self.n_layers):
        o, i = self.dims[l + 1], self.dims[l]
        vs.append(flat[:, base + self.w_off[l]: base + self.w_off[l] + o * i].view(self.replicas, o, i))
        vs.append(flat[:, base + self.b_off[l]: base + self.b_off[l] + o])
      out.append(vs)
    return out

  def load_params(self, r: int, net: int, params: Sequence[Tensor]):
    views = self.layer_views()[net]
    for v, p in zip(views, params): v[r].copy_(p.to(self.device, torch.float32))

  def export_params(self, r: int, net: int) -> List[Tensor]:
    return [v[r].detach().cpu().clone() for v in self.layer_views()[net]]
