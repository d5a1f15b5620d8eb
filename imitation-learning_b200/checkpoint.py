"""Checkpoints of training runs, multirun sweeps and hyper-parameter searches, and their resumption bit for bit.

Layout: `<dir>/step<t>/` holds `meta.json` and one `rank<k>.pt` per rank (the rank's shard of the replica axis, Trainer.checkpoint_state), and
`<dir>/LATEST` names the newest complete step directory. A save writes and fsyncs a whole step directory, then points LATEST at it with
os.replace of a small file, and only then deletes the older step directory: a kill at any moment leaves LATEST naming a complete checkpoint,
and a step directory that LATEST does not name is never read.

`<dir>` is `<run dir>/checkpoint` for a single run, `<sweep dir>/checkpoint/group<k>` for group k of a multirun and
`<search dir>/checkpoint/round<r>/<env>/group<k>` for a program of a hyper-parameter search.
"""
from __future__ import annotations

import hashlib
import json
import os
import shutil
from typing import Any, Dict, List, Optional, Sequence, Tuple

import torch

FORMAT_VERSION = 1
LATEST = 'LATEST'
META = 'meta.json'
SCORES = 'scores.json'


class CheckpointError(ValueError):
  """A checkpoint that cannot be written or resumed; the message is one line giving the reason."""


def interval_of(cfg) -> int:
  """`checkpoint.interval` (steps between checkpoints; 0 or absent: off). Anything but an integer >= 0 is refused."""
  node = cfg.get('checkpoint') if hasattr(cfg, 'get') else None
  if node is None: return 0
  if not isinstance(node, dict): raise CheckpointError(f'checkpoint={node!r}: set checkpoint.interval=N (an integer >= 0)')
  v = node.get('interval', 0)
  if v is None: return 0
  if not isinstance(v, int) or isinstance(v, bool) or v < 0: raise CheckpointError(f'checkpoint.interval={v!r} must be an integer >= 0')
  return v


def il_version() -> int:
  from . import _lib
  return int(_lib.lib().il_version())


# ---- files ---------------------------------------------------------------------------------------------------------------------
def _fsync_dir(path: str):
  fd = os.open(path, os.O_RDONLY)
  try:
    os.fsync(fd)
  finally:
    os.close(fd)


def _write_atomic(path: str, data: bytes):
  """data to path through a fsynced temporary file and os.replace."""
  tmp = path + '.tmp'
  with open(tmp, 'wb') as f:
    f.write(data)
    f.flush()
    os.fsync(f.fileno())
  os.replace(tmp, path)


def _sha256(path: str) -> str:
  h = hashlib.sha256()
  with open(path, 'rb') as f:
    for chunk in iter(lambda: f.read(1 << 24), b''): h.update(chunk)
  return h.hexdigest()


def latest(ckpt_dir: Optional[str]) -> Optional[str]:
  """The step directory LATEST names, or None when there is no complete checkpoint under ckpt_dir."""
  if not ckpt_dir: return None
  try:
    with open(os.path.join(ckpt_dir, LATEST)) as f: name = f.read().strip()
  except FileNotFoundError:
    return None
  path = os.path.join(ckpt_dir, name)
  return path if name and os.path.isfile(os.path.join(path, META)) else None


def read_meta(ckpt_dir: str) -> Dict[str, Any]:
  path = latest(ckpt_dir)
  if path is None: raise CheckpointError(f'no checkpoint under {ckpt_dir}')
  with open(os.path.join(path, META)) as f: return json.load(f)


def save(ckpt_dir: str, step: int, state: Dict[str, Any], meta: Dict[str, Any], rank: int = 0, world: int = 1, version: Optional[int] = None,
         barrier=None) -> str:
  """Writes `state` (this rank's shard) as checkpoint `step` under ckpt_dir and makes it the latest; returns its directory. `meta` (the
  resolved config, override list, replicas, ...) goes into meta.json with the format version, step, world size, il_version() and each rank
  file's byte size and sha256. `barrier` synchronises the ranks (distributed.barrier); rank 0 writes meta.json and LATEST after it."""
  barrier = barrier or (lambda: None)
  name = f'step{step}'
  path = os.path.join(ckpt_dir, name)
  if rank == 0:
    os.makedirs(ckpt_dir, exist_ok=True)
    if os.path.isdir(path): shutil.rmtree(path)  # a half-written directory of an earlier, killed attempt: LATEST never named it
    os.makedirs(path)
  barrier()
  f = os.path.join(path, f'rank{rank}.pt')
  with open(f + '.tmp', 'wb') as fh:
    torch.save(state, fh)
    fh.flush()
    os.fsync(fh.fileno())
  os.replace(f + '.tmp', f)
  barrier()
  if rank == 0:
    files = {}
    for k in range(world):
      p = os.path.join(path, f'rank{k}.pt')
      files[f'rank{k}.pt'] = dict(bytes=os.path.getsize(p), sha256=_sha256(p))
    m = dict(meta, format=FORMAT_VERSION, step=int(step), world_size=int(world), il_version=il_version() if version is None else int(version), files=files)
    _write_atomic(os.path.join(path, META), json.dumps(m, indent=1, sort_keys=True).encode())
    _fsync_dir(path)
    _write_atomic(os.path.join(ckpt_dir, LATEST), name.encode())
    _fsync_dir(ckpt_dir)
    for old in os.listdir(ckpt_dir):  # the previous checkpoint, and any directory a killed save left behind
      p = os.path.join(ckpt_dir, old)
      if old != name and old.startswith('step') and os.path.isdir(p): shutil.rmtree(p, ignore_errors=True)
  barrier()
  return path


def check(meta: Dict[str, Any], world: int, version: Optional[int] = None):
  """Refuses a checkpoint of another format, world size or library version."""
  if meta.get('format') != FORMAT_VERSION: raise CheckpointError(f'checkpoint format {meta.get("format")} is not this build\'s format {FORMAT_VERSION}')
  if meta.get('world_size') != world: raise CheckpointError(f'checkpoint was written by {meta.get("world_size")} rank(s); this launch has {world}')
  v = il_version() if version is None else version
  if meta.get('il_version') != v: raise CheckpointError(f'checkpoint was written by il_version {meta.get("il_version")}; this build is {v}')


def load(ckpt_dir: str, rank: int = 0, world: int = 1, version: Optional[int] = None) -> Tuple[Dict[str, Any], Dict[str, Any]]:
  """(meta, this rank's state) of the latest checkpoint under ckpt_dir, after checking its format, world size, library version and the size
  and sha256 of this rank's file."""
  path = latest(ckpt_dir)
  if path is None: raise CheckpointError(f'no checkpoint under {ckpt_dir}')
  with open(os.path.join(path, META)) as f: meta = json.load(f)
  check(meta, world, version)
  name = f'rank{rank}.pt'
  f, want = os.path.join(path, name), meta['files'].get(name)
  if want is None or not os.path.isfile(f): raise CheckpointError(f'{f} is missing')
  if os.path.getsize(f) != want['bytes'] or _sha256(f) != want['sha256']: raise CheckpointError(f'{f} does not match the size and sha256 in its meta.json')
  return meta, torch.load(f, map_location='cpu', weights_only=False)


def expert_digest(rows: torch.Tensor) -> str:
  """sha256 of the expert memory's rows: a resumed run refuses an expert memory other than the one its checkpoint was trained on."""
  return hashlib.sha256(rows.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


# ---- resumption plans ------------------------------------------------------------------------------------------------------------
def resume_run_meta(run_dir: str, others: Sequence[str], world: int = 1, version: Optional[int] = None) -> Dict[str, Any]:
  """meta.json of the run `train.py resume=<run_dir>` continues, after the checks that need no GPU: no other override, the directory and a
  checkpoint exist, and the world size and library version match."""
  if others: raise CheckpointError(f'resume= takes no other override (the configuration comes from the checkpoint); got {" ".join(others)}')
  if not os.path.isdir(run_dir): raise CheckpointError(f'no run directory {run_dir}')
  meta = read_meta(os.path.join(run_dir, 'checkpoint'))
  check(meta, world, version)
  return meta


def read_scores(root: str) -> Dict[str, Any]:
  try:
    with open(os.path.join(root, SCORES)) as f: return json.load(f)
  except FileNotFoundError:
    return {}


def write_scores(root: str, scores: Dict[str, Any]):
  os.makedirs(root, exist_ok=True)
  _write_atomic(os.path.join(root, SCORES), json.dumps(scores, indent=1, sort_keys=True).encode())


def group_plan(job_dirs: Sequence[str], scored: bool, ckpt_dir: Optional[str]) -> str:
  """How a resumed multirun handles one group: 'skip' when every job has its metrics.pth and the group's scores were recorded, 'continue'
  when the group has a checkpoint, else 'run'."""
  if scored and all(os.path.isfile(os.path.join(d, 'metrics.pth')) for d in job_dirs): return 'skip'
  return 'continue' if latest(ckpt_dir) is not None else 'run'


def sweep_plan(base: str, groups: Sequence[Sequence[int]]) -> List[str]:
  """group_plan of every group of the multirun in `base` (groups: the job numbers of each group, in order)."""
  root, scores = os.path.join(base, 'checkpoint'), read_scores(os.path.join(base, 'checkpoint'))
  return [group_plan([os.path.join(base, str(j)) for j in g], all(str(j) in scores for j in g), os.path.join(root, f'group{k}')) for k, g in enumerate(groups)]


def remove(ckpt_dir: Optional[str]):
  """Deletes a finished program's checkpoint directory."""
  if ckpt_dir and os.path.isdir(ckpt_dir): shutil.rmtree(ckpt_dir, ignore_errors=True)
