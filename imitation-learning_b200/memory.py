"""ReplayMemory (reference memory.py:12-68) on the device, replica-batched.

Storage is one packed row per transition (include/il_b200.h `il_replay`): [state | action | reward | next_state |
terminal | timeout | weight | step | pad] — 128 B for hopper — so a sampled transition is one coalesced 128-byte
read. The reference's 8 field tensors are exposed as strided views of that buffer.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Union

import numpy as np
import torch
from torch import Tensor

from . import _lib

FIELDS = ('step', 'states', 'actions', 'rewards', 'next_states', 'terminals', 'timeouts', 'weights')  # memory.py:17


def _field_view(rows: Tensor, off: Dict[str, int], S: int, A: int, key: str) -> Tensor:
  o = off[key]
  if key in ('states', 'next_states'): return rows[..., o:o + S]
  if key == 'actions': return rows[..., o:o + A]
  return rows[..., o]


class TransitionBatch:
  """A sampled batch: dict-like view over packed rows [R, B, row] (what memory.py:58-63 returns as a dict of
  tensors). Reads give views (R == 1: without the replica axis, i.e. the reference's shapes); writes copy into
  the packed rows, so in-place relabelling (train.py:183,192-198) works as in the reference."""

  def __init__(self, rows: Tensor, S: int, A: int, absorbing: bool):
    assert rows.dim() == 3 and rows.is_contiguous()
    self.rows, self.S, self.A, self.absorbing = rows, S, A, absorbing
    self.off, self.row = _lib.py_row_layout(S, A)
    assert rows.size(2) == self.row

  @property
  def R(self) -> int: return self.rows.size(0)

  @property
  def B(self) -> int: return self.rows.size(1)

  def _squeeze(self, t: Tensor) -> Tensor:
    return t[0] if self.R == 1 else t

  def keys(self):
    return list(FIELDS) + ['absorbing']

  def __contains__(self, key): return key in self.keys()

  def __getitem__(self, key: str) -> Tensor:
    if key == 'absorbing':  # memory.py:62
      return self._squeeze(self.rows[..., self.off['states'] + self.S - 1] if self.absorbing else torch.zeros_like(self.rows[..., 0]))
    return self._squeeze(_field_view(self.rows, self.off, self.S, self.A, key))

  def __setitem__(self, key: str, value: Tensor):
    if key == 'absorbing':
      assert self.absorbing
      self.rows[..., self.off['states'] + self.S - 1].copy_(value.reshape(self.R, self.B))
      return
    view = _field_view(self.rows, self.off, self.S, self.A, key)
    view.copy_(torch.as_tensor(value, device=self.rows.device, dtype=torch.float32).reshape(view.shape))

  def items(self):
    return [(k, self[k]) for k in self.keys()]

  def c_struct(self) -> _lib.Batch:
    b = _lib.Batch()
    b.rows, b.replica_stride, b.B, b.S, b.A, b.row = self.rows.data_ptr(), self.rows.stride(0), self.B, self.S, self.A, self.row
    return b

  @staticmethod
  def from_dict(d: Dict[str, Tensor], absorbing: Optional[bool] = None, device=None) -> 'TransitionBatch':
    """Packs a reference-style dict of tensors ([B, .] or [R, B, .]) into device rows."""
    states = torch.as_tensor(d['states'])
    if states.dim() == 2: d = {k: torch.as_tensor(v).unsqueeze(0) for k, v in d.items()}
    states = torch.as_tensor(d['states'])
    R, B, S = states.shape
    A = torch.as_tensor(d['actions']).size(2)
    device = torch.device('cuda') if device is None else device
    _, row = _lib.py_row_layout(S, A)
    if absorbing is None: absorbing = 'absorbing' in d and bool(torch.equal(torch.as_tensor(d['absorbing']).float().cpu(), states[..., -1].float().cpu()))
    tb = TransitionBatch(torch.zeros(R, B, row, device=device), S, A, absorbing)
    for k in FIELDS:
      if k in d: tb[k] = torch.as_tensor(d[k]).to(device, torch.float32)
      elif k == 'weights': tb[k] = torch.ones(R, B, device=device)
    return tb


class ReplayMemory:
  """Drop-in for the reference class (same constructor / methods / attributes) with a leading replica axis.
  `replicas=1` reproduces the reference's shapes and its numpy index stream (memory.py:51-56)."""

  def __init__(self, size: int, state_size: int, action_size: int, absorbing: bool, transitions: Optional[Dict[str, Union[Tensor, int]]] = None, replicas: int = 1,
               shared: bool = False, device=None):
    self.size, self.state_size, self.action_size, self.absorbing, self.replicas, self.shared = size, state_size, action_size, absorbing, replicas, shared
    self.device = torch.device('cuda') if device is None else torch.device(device)
    self.off, self.row = _lib.py_row_layout(state_size, action_size)
    n_store = 1 if shared else replicas
    self.rows = torch.zeros(n_store, size, self.row, device=self.device, dtype=torch.float32)
    self._idx = torch.zeros(n_store, dtype=torch.int32, device=self.device)
    self._full = torch.zeros(n_store, dtype=torch.int32, device=self.device)
    self._num_trajectories = torch.zeros(n_store, dtype=torch.int32, device=self.device)
    self._rng_counter = torch.zeros(1, dtype=torch.int64, device=self.device)
    self.seed = 0
    if transitions is not None:  # memory.py:18-23
      n = min(transitions['states'].size(0), size)
      self.rows[:, :n, self.off['step']] = torch.arange(1, n + 1, dtype=torch.float32, device=self.device)
      for k in FIELDS[1:]:
        _field_view(self.rows, self.off, state_size, action_size, k)[:, :n] = torch.as_tensor(transitions[k])[:n].to(self.device, torch.float32)
      self._num_trajectories.fill_(int(transitions['num_trajectories']))
      self._idx.fill_(n % size)
      self._full.fill_(int(n % size == 0 and n > 0))

  @property
  def seed(self) -> Union[int, List[int]]:
    """Key of the device index draws: one key, or R per-replica keys (seed sweeps), with which replica r draws the indices a single-replica
    memory seeded seed[r] draws (il_replay_sample_indices_r)."""
    return self._seed

  @seed.setter
  def seed(self, seed: Union[int, Sequence[int]]):
    if not isinstance(seed, int): assert len(seed) == self.replicas, f'{len(seed)} seeds for {self.replicas} replicas'
    self._seed, self._seed_r = (seed, None) if isinstance(seed, int) else (list(seed), _lib.seed_array(seed, self.device))

  # ---- reference attributes (host reads synchronise; used by the drop-in path only) ----
  @property
  def idx(self): return int(self._idx[0]) if self._idx.numel() == 1 else self._idx

  @property
  def full(self): return bool(self._full[0]) if self._full.numel() == 1 else self._full

  @property
  def num_trajectories(self): return int(self._num_trajectories[0]) if self._num_trajectories.numel() == 1 else self._num_trajectories

  def _view(self, key: str) -> Tensor:
    v = _field_view(self.rows, self.off, self.state_size, self.action_size, key)
    return v[0] if v.size(0) == 1 else v

  step = property(lambda self: self._view('step'))
  states = property(lambda self: self._view('states'))
  actions = property(lambda self: self._view('actions'))
  rewards = property(lambda self: self._view('rewards'))
  next_states = property(lambda self: self._view('next_states'))
  terminals = property(lambda self: self._view('terminals'))
  timeouts = property(lambda self: self._view('timeouts'))
  weights = property(lambda self: self._view('weights'))

  def __getitem__(self, idx: Union[int, str]):  # memory.py:26-35
    if isinstance(idx, str):
      if idx in ('states', 'actions', 'terminals'): return self._view(idx)
      return None
    return {k: self._view(k)[..., idx, :] if k in ('states', 'actions', 'next_states') else self._view(k)[..., idx] for k in FIELDS}

  def __len__(self) -> int:
    return self.size  # memory.py:37-38

  def c_struct(self) -> _lib.Replay:
    m = _lib.Replay()
    m.rows, m.replica_stride = self.rows.data_ptr(), (0 if self.shared else self.rows.stride(0))
    m.idx, m.full, m.num_trajectories = self._idx.data_ptr(), self._full.data_ptr(), self._num_trajectories.data_ptr()
    m.size, m.S, m.A, m.row, m.absorbing, m.shared = self.size, self.state_size, self.action_size, self.row, int(self.absorbing), int(self.shared)
    return m

  def _dev(self, x, shape) -> Tensor:
    return torch.as_tensor(x, dtype=torch.float32).to(self.device).reshape(shape).contiguous()

  def append(self, step, state, action, reward, next_state, terminal, timeout, active: Optional[Tensor] = None, wrap: bool = False):
    """memory.py:40-44 for every replica. Scalars / [1, .] tensors (R == 1) or [R, .] tensors."""
    assert not self.shared, 'shared (expert) memories are read-only'
    R, S, A = self.replicas, self.state_size, self.action_size
    lib, m = _lib.lib(), self.c_struct()
    args = [self._dev(step, (-1, )).expand(R).contiguous() if torch.as_tensor(step).numel() == 1 else self._dev(step, (R, )), self._dev(state, (R, S)), self._dev(action, (R, A)),
            self._dev(reward, (-1, )).expand(R).contiguous() if torch.as_tensor(reward).numel() == 1 else self._dev(reward, (R, )), self._dev(next_state, (R, S)),
            self._dev(terminal, (-1, )).expand(R).contiguous() if torch.as_tensor(terminal).numel() == 1 else self._dev(terminal, (R, )),
            self._dev(timeout, (-1, )).expand(R).contiguous() if torch.as_tensor(timeout).numel() == 1 else self._dev(timeout, (R, ))]
    _lib.check(lib.il_replay_append(_lib.handle(), C.byref(m), R, *[a.data_ptr() for a in args], _lib.ptr(active), int(wrap), _lib.stream()))

  def wrap_for_absorbing_states(self, mask: Optional[Tensor] = None):
    """memory.py:65-68."""
    m = self.c_struct()
    _lib.check(_lib.lib().il_replay_wrap_absorbing(_lib.handle(), C.byref(m), self.replicas, _lib.ptr(mask), _lib.stream()))

  def transfer_transitions(self, memory: 'ReplayMemory'):
    """memory.py:46-48: append every transition of `memory` to every replica's ring (weights reset to 1 by append) — one
    device pass (il_replay_transfer) instead of len(memory) appends."""
    assert memory.rows.size(0) == 1, 'transfer_transitions expects a single-store source memory (e.g. the shared expert buffer)'
    assert not self.shared, 'shared (expert) memories are read-only'
    d, s = self.c_struct(), memory.c_struct()
    _lib.check(_lib.lib().il_replay_transfer(_lib.handle(), C.byref(d), self.replicas, C.byref(s), _lib.stream()))

  # ---- sampling ----
  def draw_indices_host(self, n: int) -> np.ndarray:
    """memory.py:51-59 with the reference's global numpy stream: one np.random.randint per index, re-draw when
    the newest row is hit. Vectorised draws consume the stream exactly like n scalar calls (SURVEY §7)."""
    out = np.empty((self._idx.numel(), n), dtype=np.int32)
    idxs, fulls = self._idx.cpu().numpy(), self._full.cpu().numpy()
    for r in range(out.shape[0]):
      hi = self.size if fulls[r] else int(idxs[r]) - 1
      newest = (int(idxs[r]) - 1) % self.size
      got = np.empty(0, dtype=np.int64)
      while got.size < n:
        d = np.random.randint(0, hi, size=n - got.size)
        got = np.concatenate([got, d[d != newest]])
      out[r] = got
    return out

  def gather(self, idx: Tensor, out: Optional[TransitionBatch] = None) -> TransitionBatch:
    """memory.py:60-62 for given indices [R, n] (int32, device)."""
    R, n = self.replicas, idx.size(-1)
    idx = idx.reshape(-1, n)
    if idx.size(0) != R: idx = idx.expand(R, n)
    idx = idx.to(self.device, torch.int32).contiguous()
    if out is None: out = TransitionBatch(torch.empty(R, n, self.row, device=self.device), self.state_size, self.action_size, self.absorbing)
    m, b = self.c_struct(), out.c_struct()
    _lib.check(_lib.lib().il_replay_gather(_lib.handle(), C.byref(m), R, idx.data_ptr(), C.byref(b), _lib.stream()))
    return out

  def sample_indices_device(self, n: int, out: Optional[Tensor] = None, stream_id: int = 0, uniform: Optional[Tensor] = None) -> Tensor:
    """`_sample_idx` x n on the device (same distribution as memory.py:51-56). `uniform` ([R, n] U[0,1) floats, e.g.
    drawn by numpy on the host like the reference) replaces the device Philox draws."""
    R = self.replicas
    if out is None: out = torch.empty(R, n, dtype=torch.int32, device=self.device)
    m, lib = self.c_struct(), _lib.lib()
    if self._seed_r is None:
      _lib.check(lib.il_replay_sample_indices(_lib.handle(), C.byref(m), R, n, out.data_ptr(), _lib.ptr(uniform), self.seed, stream_id, self._rng_counter.data_ptr(), _lib.stream()))
    else:
      _lib.check(lib.il_replay_sample_indices_r(_lib.handle(), C.byref(m), R, n, out.data_ptr(), _lib.ptr(uniform), self._seed_r.data_ptr(), stream_id, self._rng_counter.data_ptr(),
                                                _lib.stream()))
    if uniform is None: _lib.check(lib.il_counter_add(_lib.handle(), self._rng_counter.data_ptr(), R * n if self._seed_r is None else n, _lib.stream()))
    return out

  def sample(self, n: int, device_rng: bool = False) -> TransitionBatch:
    """memory.py:58-63. Default: the reference's numpy stream drawn on the host (drop-in semantics)."""
    if device_rng: return self.gather(self.sample_indices_device(n))
    return self.gather(torch.from_numpy(self.draw_indices_host(n)))
