"""HBM-resident replay with the reference's `dqn_zoo/replay.py` surface.

Same class names, constructor arguments, return types/dtypes and exceptions as the
reference (cited per method), so agents and tests written for `dqn_zoo.replay`
run unchanged, with two stated differences: a (snappy) encoder/decoder pair is applied as a
host round trip at insert time instead of at rest, and the accumulators return lists, not
generators.  What else differs is where things live:

  * transition storage (`OrderedDict` in the reference, `replay.py:140,688`) is a
    transition-major uint8 array in device memory: row = id % capacity holds
    s_tm1 | s_t back to back (DESIGN.md §3); or, with `frame_dedup=True`, a frame pool
    that keeps each distinct H*W plane of the stored frame stacks once (`_FramePoolStore`);
  * the float64 sum tree (`replay.py:246-426`) is a device array traversed by a
    warp-cooperative CUDA kernel (csrc/dz_replay.cu);
  * O(1) integer bookkeeping per add (free-slot stack, swap-remove lists,
    id<->index maps; `replay.py:52-74,475-534`) stays on the host exactly as in the
    reference, and is mirrored to the device as (position, value) patches so that
    sampling needs no host lookups;
  * the host `np.random.RandomState` is consumed in the reference's order
    (`replay.py:551-567`), its draws are shipped to the device, and index selection,
    probabilities, importance weights and the gather run in CUDA.

No CPU fallback: every numeric result returned by `sample()` is computed on the GPU.
"""

from __future__ import annotations

import collections
import copy
import ctypes as C
import os
from typing import Any, Callable, Iterable, List, Mapping, NamedTuple, Optional, Sequence, Tuple

import numpy as np
import torch

from dqn_zoo_b200 import _lib

_FLAG_NAMES = {1: 'value must be finite and positive', 2: 'index out of range', 4: 'Require 0 <= target < total sum.',
               8: 'sum-tree root is zero in the fused path', 16: 'Weights are not finite'}


class Transition(NamedTuple):
  """`replay.py:36-41`."""
  s_tm1: Any
  a_tm1: Any
  r_t: Any
  discount_t: Any
  s_t: Any


def _device():
  if not torch.cuda.is_available():
    raise RuntimeError('dqn_zoo_b200.replay needs a CUDA device (there is no CPU fallback)')
  return torch.device('cuda', torch.cuda.current_device())


def _stream():
  return torch.cuda.current_stream().cuda_stream


def _ptr(t):
  return 0 if t is None else t.data_ptr()


def _power(base, exponent):
  """`replay.py:203-208` for the HOST-side add path (float64 scalar per add, as the
  reference evaluates it at `replay.py:507`).  The float32 `update_priorities` path is
  evaluated on the device instead (csrc/dz_replay.cu:exponentiate_f32)."""
  b = np.asarray(base, dtype=np.float64)
  return np.where(b == 0.0, 0.0, b ** exponent)


def importance_sampling_weights(probabilities, uniform_probability, exponent, normalize):
  """`replay.py:211-243`, evaluated on the device (float64)."""
  if not 0.0 <= exponent <= 1.0:
    raise ValueError('Require 0 <= exponent <= 1.')
  if not 0.0 <= uniform_probability <= 1.0:
    raise ValueError('Expected 0 <= uniform_probability <= 1.')
  p = torch.as_tensor(np.asarray(probabilities, dtype=np.float64), device=_device())
  w = (uniform_probability / p) ** exponent
  if normalize:
    w = w / w.max()
  w = w.cpu().numpy()
  if not np.isfinite(w).all():
    raise ValueError('Weights are not finite: %s.' % w)
  return w


# ------------------------------------------------------------------------------------------------
# R1: SumTree
# ------------------------------------------------------------------------------------------------


class SumTree:
  """Device-resident float64 sum tree with the interface of `replay.py:246-426`."""

  def __init__(self):
    self._size = 0
    self._first_leaf = 0
    self._nodes = torch.zeros(0, dtype=torch.float64, device=_device())
    self._flags = torch.zeros(1, dtype=torch.int32, device=_device())

  # -- helpers ---------------------------------------------------------------------------------
  def _rebuild(self, n_valid):
    if self._first_leaf:
      _lib.call('dz_sumtree_rebuild', _ptr(self._nodes), self._first_leaf, n_valid, _stream())

  def _raise_flags(self):
    f = int(self._flags.item())
    if f:
      self._flags.zero_()
      if f & _lib.DZ_FLAG_BAD_INDEX:
        raise IndexError('index out of range, expect 0 <= index < %s' % self._size)
      raise ValueError(_FLAG_NAMES.get(f & -f, 'device flag %d' % f))

  def _initialize(self, size, values):
    """`replay.py:361-392`."""
    assert size >= 0
    assert values is None or len(values) == size
    fl = self._first_leaf
    if size < self._size:
      self._size = size
      if values is not None:
        self._nodes[fl:fl + size] = values
      self._rebuild(size)
    elif size <= fl:
      self._size = size
      if values is not None:
        self._nodes[fl:fl + size] = values
        self._rebuild(size)
    else:
      cap = 1
      while cap < size:
        cap *= 2
      new = torch.empty(2 * cap, dtype=torch.float64, device=self._nodes.device)
      if values is None:
        keep = self._size
        new[cap:cap + keep] = self._nodes[fl:fl + keep]
      else:
        keep = size
        new[cap:cap + keep] = values
      self._nodes, self._first_leaf, self._size = new, cap, size
      self._rebuild(keep)

  @staticmethod
  def _validated(values, msg):
    v = np.asarray(values, dtype=np.float64)
    if not np.isfinite(v).all() or (v < 0.0).any():
      raise ValueError(msg)
    return v

  # -- reference surface -------------------------------------------------------------------------
  def resize(self, size: int) -> None:
    """`replay.py:267-269`."""
    self._initialize(size, None)

  def get(self, indices) -> np.ndarray:
    """`replay.py:271-276`."""
    idx = np.asarray(indices, dtype=np.int64)
    if idx.size and not ((0 <= idx) & (idx < self._size)).all():
      raise IndexError('index out of range, expect 0 <= index < %s' % self._size)
    if idx.size == 0:
      return np.zeros(idx.shape, dtype=np.float64)
    d_idx = torch.as_tensor(idx.reshape(-1), device=self._nodes.device)
    out = torch.empty(idx.size, dtype=torch.float64, device=self._nodes.device)
    _lib.call('dz_sumtree_get', _ptr(self._nodes), self._first_leaf, self._size, _ptr(d_idx), idx.size, _ptr(out),
              _ptr(self._flags), _stream())
    return out.cpu().numpy().reshape(idx.shape)

  def set(self, indices, values) -> None:
    """`replay.py:278-290`."""
    v = self._validated(values, 'value must be finite and positive.').reshape(-1)
    idx = np.asarray(indices, dtype=np.int64).reshape(-1)
    if idx.size == 0:
      return
    if not ((0 <= idx) & (idx < self._size)).all():
      raise IndexError('index out of range')
    self.set_device(torch.as_tensor(idx, device=self._nodes.device), torch.as_tensor(v, device=self._nodes.device))

  def set_device(self, d_idx: torch.Tensor, d_values: torch.Tensor) -> None:
    """`set` with device-resident int64 indices / float64 values (no host round trip)."""
    _lib.call('dz_sumtree_set', _ptr(self._nodes), self._first_leaf, self._size, _ptr(d_idx), _ptr(d_values),
              d_idx.numel(), _ptr(self._flags), _stream())

  def set_all(self, values) -> None:
    """`replay.py:292-297`."""
    v = self._validated(values, 'Values must be finite positive numbers.')
    self._initialize(len(v), torch.as_tensor(v, device=self._nodes.device))

  def query(self, targets) -> List[int]:
    """`replay.py:299-313`: ValueError unless 0 <= target < root for every target."""
    t = np.asarray(targets, dtype=np.float64).reshape(-1)
    root = self.root()
    if t.size and not ((0.0 <= t) & (t < root)).all():
      raise ValueError('Require 0 <= target < total sum.')
    if t.size == 0:
      return []
    d_t = torch.as_tensor(t, device=self._nodes.device)
    out = torch.empty(t.size, dtype=torch.int64, device=self._nodes.device)
    _lib.call('dz_sumtree_query', _ptr(self._nodes), self._first_leaf, _ptr(d_t), t.size, _ptr(out), _ptr(self._flags),
              _stream())
    return out.cpu().tolist()

  def root(self) -> float:
    """`replay.py:315-317`."""
    return float(self._nodes[1].item()) if self._size > 0 else np.nan

  @property
  def values(self) -> np.ndarray:
    """`replay.py:319-322` (a host COPY here; the reference returns a view)."""
    return self._nodes[self._first_leaf:self._first_leaf + self._size].cpu().numpy()

  @property
  def size(self) -> int:
    return self._size

  @property
  def capacity(self) -> int:
    return self._first_leaf

  @property
  def device_nodes(self) -> torch.Tensor:
    return self._nodes

  def get_state(self) -> Mapping[str, Any]:
    """`replay.py:334-340`: same keys; `storage` is a host float64 array."""
    return {'size': self._size, 'storage': self._nodes.cpu().numpy(), 'first_leaf': self._first_leaf}

  def set_state(self, state: Mapping[str, Any]) -> None:
    """`replay.py:342-346`."""
    self._size = int(state['size'])
    self._first_leaf = int(state['first_leaf'])
    self._nodes = torch.as_tensor(np.array(state['storage'], dtype=np.float64), device=self._nodes.device)

  def check_valid(self) -> Tuple[bool, str]:
    """`replay.py:348-359` (consistency is verified on a host copy)."""
    nodes = self._nodes.cpu().numpy()
    fl = self._first_leaf
    if len(nodes) != 2 * fl:
      return False, 'first_leaf should be half the size of storage.'
    if not 0 <= self._size <= fl:
      return False, 'Require 0 <= self.size <= self.capacity.'
    if fl > 1:
      sums = nodes[2:2 * fl:2] + nodes[3:2 * fl:2]
      bad = np.nonzero(nodes[1:fl] != sums)[0]
      if bad.size:
        return False, 'Non-leaf node %d should be sum of child nodes.' % (bad[0] + 1)
    return True, ''


# ------------------------------------------------------------------------------------------------
# Device mirrors of the dense host lists
# ------------------------------------------------------------------------------------------------


class _DeviceList:
  """int64 device array that mirrors a host list through (position, value) patches."""

  def __init__(self, n=0):
    self.t = torch.zeros(max(n, 1), dtype=torch.int64, device=_device())

  def ensure(self, n):
    if n > self.t.numel():
      new = torch.zeros(max(n, 2 * self.t.numel()), dtype=torch.int64, device=self.t.device)
      new[:self.t.numel()] = self.t
      self.t = new

  def upload(self, values):
    v = np.asarray(values, dtype=np.int64)
    self.ensure(len(v))
    if len(v):
      self.t[:len(v)] = torch.as_tensor(v, device=self.t.device)


def _apply_index_record(view, patches, tree_index=-1, leaf_value=0.0, evict_index=-1, size_after=0, slot=0,
                        action=0, reward=0.0, discount=0.0, h_s_tm1=None, h_s_t=None, d_priority=None, alpha=1.0,
                        release_row=False):
  """One dz_replay_add call: <=4 list patches + optional evict/set on the tree (+ optional row write)."""
  rec = _lib.AddRecord()
  rec.release_row = 1 if release_row else 0
  rec.slot, rec.action, rec.reward, rec.discount = slot, action, reward, discount
  rec.n_patches = len(patches)
  for k, (target, pos, val) in enumerate(patches):
    rec.patch_target[k], rec.patch_pos[k], rec.patch_val[k] = target, pos, val
  rec.tree_index, rec.leaf_value, rec.evict_index, rec.size_after = tree_index, leaf_value, evict_index, size_after
  rec.d_priority = None if d_priority is None else d_priority.data_ptr()
  rec.alpha = alpha
  def addr(x):
    if x is None:
      return None
    return x.data_ptr() if isinstance(x, torch.Tensor) else x.ctypes.data
  _lib.call('dz_replay_add', C.byref(view), C.byref(rec), addr(h_s_tm1), addr(h_s_t), _stream())


class _MirroredIndex:
  """The device mirrors of a distribution's host lists, kept equal to them through (target, position, value) patches.
  A distribution says how many pending patches are cheaper to `_upload` as whole lists (`_BULK`), which host lists and
  device mirrors a checkpoint holds (`_HOST_LISTS`, `_device_mirrors`, `_manifest`), and how a replay's add, reset and
  synthetic fill change its lists (`_insert`, `_reset`, `_fill`)."""

  _scratch = None

  def flush(self):
    """Pushes pending patches to the device mirrors."""
    patches = self.take_patches()
    if not patches:
      return
    if len(patches) > self._BULK:
      self._upload()
      return
    v = self.device_view()
    # dz_replay_add also writes the row scalars; give it a scratch row.
    if self._scratch is None:
      self._scratch = torch.zeros(8, dtype=torch.float64, device=_device())
    v.d_action, v.d_reward, v.d_discount, v.d_obs = (_ptr(self._scratch),) * 4
    for k in range(0, len(patches), 4):
      _apply_index_record(v, patches[k:k + 4])


# ------------------------------------------------------------------------------------------------
# R6: UniformDistribution
# ------------------------------------------------------------------------------------------------


class UniformDistribution(_MirroredIndex):
  """`replay.py:44-117`.  Host swap-remove list + device mirror for in-kernel lookups."""

  _BULK = 16
  _HOST_LISTS = {'ids': list, 'id_to_index': dict}

  def __init__(self, random_state: np.random.RandomState):
    self._random_state = random_state
    self._ids: List[int] = []
    self._id_to_index = {}
    self._mirror = _DeviceList()
    self._pending = []  # (target=2, position, value) patches not yet on the device

  def add(self, ids: Sequence[int]) -> None:
    """`replay.py:52-61`."""
    for i in ids:
      if i in self._id_to_index:
        raise IndexError('Cannot add ID %d, it already exists.' % i)
    for i in ids:
      self._id_to_index[i] = len(self._ids)
      self._pending.append((2, len(self._ids), i))
      self._ids.append(i)

  def remove(self, ids: Sequence[int]) -> None:
    """`replay.py:63-74`."""
    for i in ids:
      if i not in self._id_to_index:
        raise IndexError('Cannot remove ID %d, it does not exist.' % i)
    for i in ids:
      hole = self._id_to_index.pop(i)
      tail = self._ids.pop()
      if tail != i:
        self._ids[hole] = tail
        self._id_to_index[tail] = hole
        self._pending.append((2, hole, tail))

  def take_patches(self):
    p, self._pending = self._pending, []
    self._mirror.ensure(len(self._ids))
    return p

  def _upload(self):
    self._mirror.upload(self._ids)

  def _insert(self, item_id, evicted_id=None):
    """One replay add: removes `evicted_id` (if any), adds `item_id`.  No tree: (evict_index, tree_index) = (-1, -1)."""
    if evicted_id is not None:
      self.remove([evicted_id])
    self.add([item_id])
    return -1, -1

  def _reset(self, capacity):
    self._ids, self._id_to_index, self._pending = [], {}, []

  def _fill(self, capacity, priority):
    self._ids = list(range(capacity))
    self._id_to_index = {i: i for i in range(capacity)}
    self._pending = []
    self._mirror.upload(self._ids)

  def _device_mirrors(self):
    return {'ids_mirror': self._mirror.t}

  def _manifest(self):
    return {}

  def device_view(self):
    v = _lib.ReplayView()
    v.capacity = 1
    v.d_ids = _ptr(self._mirror.t)
    return v

  def sample(self, size: int) -> np.ndarray:
    """`replay.py:76-82`: host randint draw, device lookup (uniform_sample_kernel)."""
    picks = self._random_state.randint(self.size, size=size).astype(np.int64)
    self.flush()
    dev = self._mirror.t.device
    d_pos = torch.as_tensor(picks, device=dev)
    out_i = torch.empty(2 * size, dtype=torch.int64, device=dev)
    sin = _lib.SampleInputs(_ptr(d_pos), None, None, None)
    sout = _lib.SampleOutputs(out_i.data_ptr(), None, out_i.data_ptr() + 8 * size, None, None)
    v = self.device_view()
    _lib.call('dz_replay_sample', C.byref(v), 0, C.byref(sin), C.byref(sout), size, _stream())
    return out_i[:size].cpu().numpy()

  def ids(self) -> Iterable[int]:
    return self._id_to_index.keys()

  @property
  def size(self) -> int:
    return len(self._ids)

  @property
  def device_ids(self):
    return self._mirror.t

  def get_state(self) -> Mapping[str, Any]:
    """`replay.py:93-98`."""
    return {'ids': self._ids, 'id_to_index': self._id_to_index}

  def set_state(self, state: Mapping[str, Any]) -> None:
    """`replay.py:100-103`."""
    self._ids = state['ids']
    self._id_to_index = state['id_to_index']
    self._pending = []
    self._mirror.upload(self._ids)

  def check_valid(self) -> Tuple[bool, str]:
    """`replay.py:105-117` plus: the device mirror equals the host list."""
    if len(self._ids) != len(self._id_to_index):
      return False, 'ids and id_to_index should be the same size.'
    if len(set(self._ids)) != len(self._ids):
      return False, 'IDs should be unique.'
    for pos, i in enumerate(self._ids):
      if self._id_to_index.get(i) != pos:
        return False, 'ID %d should map to itself.' % i
    self.flush()
    if self._ids and self._mirror.t[:len(self._ids)].cpu().tolist() != list(self._ids):
      return False, 'device mirror of ids is stale.'
    return True, ''


# ------------------------------------------------------------------------------------------------
# R2: PrioritizedDistribution
# ------------------------------------------------------------------------------------------------


class PrioritizedDistribution(_MirroredIndex):
  """`replay.py:429-651`: host id/index bookkeeping, device sum tree and sampling."""

  _BULK = 32
  _HOST_LISTS = {'id_to_index': dict, 'index_to_id': dict, 'inactive_indices': list, 'active_indices': list,
                 'active_indices_location': dict}

  def __init__(self, priority_exponent: float, uniform_sample_probability: float,
               random_state: np.random.RandomState, min_capacity: int = 0, max_capacity: Optional[int] = None):
    if priority_exponent < 0.0:
      raise ValueError('Require priority_exponent >= 0.')
    if not 0.0 <= uniform_sample_probability <= 1.0:
      raise ValueError('Require 0 <= uniform_sample_probability <= 1.')
    if max_capacity is not None and max_capacity < min_capacity:
      raise ValueError('Require max_capacity >= min_capacity.')
    if min_capacity < 0:
      raise ValueError('Require min_capacity >= 0.')
    self._priority_exponent = priority_exponent
    self._uniform_sample_probability = uniform_sample_probability
    self._max_capacity = max_capacity
    self._random_state = random_state
    self._sum_tree = SumTree()
    self._sum_tree.resize(min_capacity)
    self._id_to_index = {}
    self._index_to_id = {}
    self._inactive_indices = list(range(min_capacity))
    self._active_indices: List[int] = []
    self._active_indices_location = {}
    self._live_dev = _DeviceList(min_capacity)     # mirror of _active_indices
    self._id_at_dev = _DeviceList(min_capacity)    # mirror of _index_to_id (dense by tree index)
    self._pending = []                             # (target, position, value): 0 = live, 1 = id_at
    self._stage = None

  # -- capacity ----------------------------------------------------------------------------------
  def ensure_capacity(self, capacity: int) -> None:
    """`replay.py:463-473`."""
    if self._max_capacity is not None and capacity > self._max_capacity:
      raise ValueError('capacity %d cannot exceed max_capacity %d' % (capacity, self._max_capacity))
    if capacity <= self._sum_tree.size:
      return
    self._inactive_indices.extend(range(self._sum_tree.size, capacity))
    self._sum_tree.resize(capacity)
    self._live_dev.ensure(capacity)
    self._id_at_dev.ensure(capacity)

  # -- host bookkeeping (no device work) -----------------------------------------------------------
  def _host_add(self, ids):
    for i in ids:
      if i in self._id_to_index:
        raise IndexError('ID %d already exists.' % i)
    new_size = self.size + len(ids)
    if self._max_capacity is not None and new_size > self._max_capacity:
      raise ValueError('Cannot add IDs as max capacity would be exceeded.')
    if new_size > self.capacity:
      grown = max(new_size, 2 * self.capacity)
      if self._max_capacity is not None:
        grown = min(self._max_capacity, grown)
      self.ensure_capacity(grown)
    got = []
    for i in ids:
      idx = self._inactive_indices.pop()          # allocation pops from the END (`replay.py:499`)
      pos = len(self._active_indices)
      self._active_indices_location[idx] = pos
      self._active_indices.append(idx)
      self._id_to_index[i] = idx
      self._index_to_id[idx] = i
      self._pending.append((0, pos, idx))
      self._pending.append((1, idx, i))
      got.append(idx)
    return got

  def _host_remove(self, ids):
    gone = [self._id_to_index[i] for i in ids]
    for i, idx in zip(ids, gone):
      del self._id_to_index[i]
      del self._index_to_id[idx]
      hole = self._active_indices_location.pop(idx)
      tail = self._active_indices.pop()
      if tail != idx:                             # swap-remove (`replay.py:519-531`)
        self._active_indices[hole] = tail
        self._active_indices_location[tail] = hole
        self._pending.append((0, hole, tail))
    self._inactive_indices.extend(gone)
    return gone

  def take_patches(self):
    p, self._pending = self._pending, []
    return p

  def _upload(self):
    self._live_dev.upload(self._active_indices)
    dense = np.zeros(max(self._sum_tree.size, 1), dtype=np.int64)
    if self._index_to_id:
      k = np.fromiter(self._index_to_id.keys(), dtype=np.int64, count=len(self._index_to_id))
      dense[k] = np.fromiter(self._index_to_id.values(), dtype=np.int64, count=len(self._index_to_id))
    self._id_at_dev.upload(dense)

  def _insert(self, item_id, evicted_id=None):
    """One replay add: removes `evicted_id` (if any), adds `item_id`; returns their (evict_index, tree_index), -1 for
    no eviction."""
    evict_index = -1
    if evicted_id is not None:
      (evict_index,) = self._host_remove([evicted_id])
    (tree_index,) = self._host_add([item_id])
    return evict_index, tree_index

  def _reset(self, capacity):
    self._id_to_index, self._index_to_id, self._pending = {}, {}, []
    self._inactive_indices = list(range(capacity))
    self._active_indices, self._active_indices_location = [], {}
    self._sum_tree._nodes.zero_()
    self._sum_tree._size = capacity

  def _fill(self, capacity, priority):
    idx = np.arange(capacity - 1, -1, -1, dtype=np.int64)          # id i -> index C-1-i
    self._id_to_index = dict(zip(range(capacity), idx.tolist()))
    self._index_to_id = dict(zip(idx.tolist(), range(capacity)))
    self._inactive_indices = []
    self._active_indices = idx.tolist()
    self._active_indices_location = dict(zip(idx.tolist(), range(capacity)))
    self._pending = []
    self._live_dev.upload(idx)
    self._id_at_dev.upload(idx)                                     # id_at[index] = C-1-index
    leaf = float(_power([priority], self._priority_exponent)[0])
    self._sum_tree.set_all(np.full(capacity, leaf, dtype=np.float64))

  def _device_mirrors(self):
    return {'sum_tree': self._sum_tree._nodes, 'live_mirror': self._live_dev.t, 'id_at_mirror': self._id_at_dev.t}

  def _manifest(self):
    return {'tree_size': self._sum_tree.size, 'tree_first_leaf': self._sum_tree.capacity}

  def device_view(self):
    v = _lib.ReplayView()
    v.capacity = 1
    v.d_tree = _ptr(self._sum_tree.device_nodes)
    v.first_leaf = self._sum_tree.capacity
    v.d_live = _ptr(self._live_dev.t)
    v.d_id_at = _ptr(self._id_at_dev.t)
    v.d_flags = _ptr(self._sum_tree._flags)
    return v

  # -- reference surface ---------------------------------------------------------------------------
  def add_priorities(self, ids: Sequence[int], priorities: Sequence[float]) -> None:
    """`replay.py:475-507`."""
    got = self._host_add(ids)
    self.flush()
    self._sum_tree.set(got, _power(priorities, self._priority_exponent))

  def remove_priorities(self, ids: Sequence[int]) -> None:
    """`replay.py:509-534`."""
    gone = self._host_remove(ids)
    self.flush()
    self._sum_tree.set(gone, np.zeros((len(gone),), dtype=np.float64))

  def update_priorities(self, ids: Sequence[int], priorities: Sequence[float]) -> None:
    """`replay.py:536-545`.  float32 priorities (what comes back from the learner) are
    exponentiated on the device in float32 as the reference's numpy does; other dtypes take the
    reference's float64 host `_power` and only the tree update runs on the device."""
    where = []
    for i in ids:
      if i not in self._id_to_index:
        raise IndexError('ID %d does not exist.' % i)
      where.append(self._id_to_index[i])
    pri = np.asarray(priorities)
    if pri.dtype == np.float32:
      if not np.isfinite(pri).all() or (pri < 0.0).any():
        raise ValueError('value must be finite and positive.')
      dev = self._live_dev.t.device
      self.update_priorities_device(torch.as_tensor(np.asarray(where, dtype=np.int64), device=dev),
                                    torch.as_tensor(pri.reshape(-1), device=dev))
    else:
      self._sum_tree.set(where, _power(pri, self._priority_exponent))

  def update_priorities_device(self, d_indices: torch.Tensor, d_priorities: torch.Tensor) -> None:
    """Priority write-back with device-resident tree indices (int64) and float32 priorities."""
    v = self.device_view()
    _lib.call('dz_replay_update_priorities', C.byref(v), _ptr(d_indices), _ptr(d_priorities), d_indices.numel(),
              float(self._priority_exponent), self._sum_tree.size, _stream())

  def _draw(self, size):
    """The three host draws of `replay.py:551-567`, in order; needs root (one 8-byte D2H)."""
    pos = self._random_state.randint(self.size, size=size).astype(np.int64)
    root = self._sum_tree.root()
    u_tree = self._random_state.uniform(size=size) if root != 0.0 else np.zeros(size)
    u_mix = self._random_state.uniform(size=size)
    return pos, u_tree, u_mix

  def sample_device(self, size, beta=1.0, normalize=False, capacity_for_slots=1):
    """Runs the sampling kernel; returns device tensors (ids, indices, slots, probs, weights)."""
    if self.size == 0:
      raise RuntimeError('No IDs to sample.')
    self.flush()
    pos, u_tree, u_mix = self._draw(size)
    dev = self._live_dev.t.device
    out_i = torch.empty(3 * size, dtype=torch.int64, device=dev)
    out_f = torch.empty(2 * size, dtype=torch.float64, device=dev)
    v = self.device_view()
    v.capacity = capacity_for_slots
    chunk = 1024  # the kernel normalises over one block; larger requests run in chunks, normalised below
    big = size > chunk
    for lo in range(0, size, chunk):
      n = min(chunk, size - lo)
      host = np.concatenate([u_tree[lo:lo + n], u_mix[lo:lo + n],
                             [float(self.size), float(beta), float(self._uniform_sample_probability),
                              1.0 if (normalize and not big) else 0.0]])
      d_f = torch.as_tensor(host, device=dev)
      d_pos = torch.as_tensor(pos[lo:lo + n], device=dev)
      sin = _lib.SampleInputs(_ptr(d_pos), d_f.data_ptr(), d_f.data_ptr() + 8 * n, d_f.data_ptr() + 16 * n)
      ip, fp = out_i.data_ptr() + 8 * lo, out_f.data_ptr() + 8 * lo
      sout = _lib.SampleOutputs(ip, ip + 8 * size, ip + 16 * size, fp, fp + 8 * size)
      _lib.call('dz_replay_sample', C.byref(v), 1, C.byref(sin), C.byref(sout), n, _stream())
    if big and normalize:
      out_f[size:] /= out_f[size:].max()
    return out_i[:size], out_i[size:2 * size], out_i[2 * size:], out_f[:size], out_f[size:]

  def sample(self, size: int) -> Tuple[np.ndarray, np.ndarray]:
    """`replay.py:547-583`."""
    ids, _, _, probs, _ = self.sample_device(size)
    self._sum_tree._raise_flags()
    return ids.cpu().numpy(), probs.cpu().numpy()

  def get_exponentiated_priorities(self, ids: Sequence[int]) -> Sequence[float]:
    """`replay.py:585-590`."""
    return self._sum_tree.get(np.fromiter((self._id_to_index[i] for i in ids), dtype=np.int64, count=len(ids)))

  def ids(self) -> Iterable[int]:
    return self._id_to_index.keys()

  @property
  def capacity(self) -> int:
    return self._sum_tree.size

  @property
  def size(self) -> int:
    return len(self._id_to_index)

  def get_state(self) -> Mapping[str, Any]:
    """`replay.py:606-615` (same keys)."""
    return {
        'sum_tree': self._sum_tree.get_state(),
        'id_to_index': self._id_to_index,
        'index_to_id': self._index_to_id,
        'inactive_indices': self._inactive_indices,
        'active_indices': self._active_indices,
        'active_indices_location': self._active_indices_location,
    }

  def set_state(self, state: Mapping[str, Any]) -> None:
    """`replay.py:617-624`."""
    self._sum_tree.set_state(state['sum_tree'])
    self._id_to_index = state['id_to_index']
    self._index_to_id = state['index_to_id']
    self._inactive_indices = state['inactive_indices']
    self._active_indices = state['active_indices']
    self._active_indices_location = state['active_indices_location']
    self._live_dev.ensure(self._sum_tree.size)
    self._id_at_dev.ensure(self._sum_tree.size)
    self._pending = [(0, 0, 0)] * 64  # forces a full re-upload of both mirrors
    self.flush()

  def check_valid(self) -> Tuple[bool, str]:
    """`replay.py:626-651`, plus the device mirrors agree with the host lists."""
    if len(self._id_to_index) != len(self._index_to_id):
      return False, 'ID to index maps are not the same size.'
    for i, idx in self._id_to_index.items():
      if self._index_to_id.get(idx) != i:
        return False, 'ID %d should map to itself.' % i
    if len(set(self._inactive_indices)) != len(self._inactive_indices):
      return False, 'Inactive indices should be unique.'
    if len(set(self._active_indices)) != len(self._active_indices):
      return False, 'Active indices should be unique.'
    if set(self._active_indices) != set(self._index_to_id.keys()):
      return False, 'Active indices should match index to ID mapping keys.'
    if sorted(self._inactive_indices + self._active_indices) != list(range(self._sum_tree.size)):
      return False, 'Inactive and active indices should partition all indices.'
    for pos, idx in enumerate(self._active_indices):
      if self._active_indices_location.get(idx) != pos:
        return False, 'Active index location %d not correct for index %d.' % (pos, idx)
    self.flush()
    n = len(self._active_indices)
    if n and self._live_dev.t[:n].cpu().tolist() != list(self._active_indices):
      return False, 'device mirror of active indices is stale.'
    if n:
      id_at = self._id_at_dev.t.cpu().numpy()
      for idx, i in self._index_to_id.items():
        if id_at[idx] != i:
          return False, 'device mirror of index_to_id is stale at %d.' % idx
    return self._sum_tree.check_valid()


# ------------------------------------------------------------------------------------------------
# Transition storage in HBM
# ------------------------------------------------------------------------------------------------


class _TransitionStore:
  """Row = id % capacity; each row holds s_tm1 | s_t (uint8, stride padded to 16 B)."""

  def __init__(self, capacity):
    self.capacity = capacity
    self.obs = None
    self.obs_shape = None
    self.obs_dtype = None
    dev = _device()
    n = max(capacity, 1)
    self.action = torch.zeros(n, dtype=torch.int32, device=dev)
    self.reward = torch.zeros(n, dtype=torch.float64, device=dev)
    self.discount = torch.zeros(n, dtype=torch.float64, device=dev)
    self.flags = torch.zeros(1, dtype=torch.int32, device=dev)
    self.obs_bytes = 0
    self.obs_stride = 0
    self._batch = None

  def add_batch_buffers(self, view):
    """(records, workspace, adds per call) of dz_replay_add_batch, allocated on first use: the workspace is sized by
    dz_replay_add_batch_workspace for min(capacity, ADD_BATCH_MAX) adds, lowered to what one call takes."""
    if self._batch is None:
      most, nbytes = C.c_int32(max(1, min(self.capacity, ADD_BATCH_MAX))), C.c_int64()
      _lib.call('dz_replay_add_batch_workspace', C.byref(view), C.byref(most), C.byref(nbytes))
      ws = torch.empty(nbytes.value, dtype=torch.uint8, device=self.action.device)
      self._batch = (_AddBatchRecords(most.value, self.action.device), ws, most.value)
    return self._batch

  def allocate(self, obs_shape, obs_dtype=np.uint8):
    if self.obs is not None:
      return
    self.obs_shape, self.obs_dtype = tuple(obs_shape), np.dtype(obs_dtype)
    self.obs_bytes = int(np.prod(obs_shape)) * self.obs_dtype.itemsize
    self.obs_stride = (self.obs_bytes + 15) // 16 * 16
    self.obs = torch.empty((max(self.capacity, 1), 2, self.obs_stride), dtype=torch.uint8, device=self.action.device)

  def fill_view(self, v):
    v.d_obs, v.d_action, v.d_reward, v.d_discount = _ptr(self.obs), _ptr(self.action), _ptr(self.reward), _ptr(self.discount)
    v.capacity, v.obs_bytes, v.obs_stride = self.capacity, self.obs_bytes, self.obs_stride
    v.d_flags = _ptr(self.flags)
    return v

  def gather(self, d_slots, size):
    """`np.stack` of `get(ids)` (`replay.py:718-722`) on the device; returns device tensors."""
    dev = self.action.device
    s_tm1 = torch.empty((size, self.obs_bytes), dtype=torch.uint8, device=dev)
    s_t = torch.empty((size, self.obs_bytes), dtype=torch.uint8, device=dev)
    a = torch.empty(size, dtype=torch.int64, device=dev)
    r = torch.empty(size, dtype=torch.float64, device=dev)
    d = torch.empty(size, dtype=torch.float64, device=dev)
    v = self.fill_view(_lib.ReplayView())
    _lib.call('dz_replay_gather', C.byref(v), _ptr(d_slots), size, _ptr(s_tm1), _ptr(s_t), _ptr(a), _ptr(r), _ptr(d),
              _stream())
    return s_tm1, a, r, d, s_t

  def get_rows(self, structure, slots, chunk=4096):
    """`[storage[i] for i in ids]` (`replay.py:153-156`): rows are gathered on the device and copied to the host in
    chunks, so the staging memory is bounded (2 * chunk * obs_bytes) whatever the number of rows — `get_state()` of a
    full 1M-capacity replay goes through here."""
    out = []
    dev = self.action.device
    for lo in range(0, len(slots), chunk):
      part = np.ascontiguousarray(slots[lo:lo + chunk])
      tr = self.to_host_transition(structure, self.gather(torch.as_tensor(part, device=dev), len(part)))
      out.extend(type(structure)(*[f[k] for f in tr]) for k in range(len(part)))
    return out

  def storage_bytes(self):
    """Device bytes this store holds (observations and per-row scalars)."""
    ts = [t for t in (self.obs, self.action, self.reward, self.discount, self.flags) if t is not None]
    return sum(t.numel() * t.element_size() for t in ts)

  def to_host_transition(self, structure, tensors):
    s_tm1, a, r, d, s_t = [t.cpu().numpy() for t in tensors]
    shape = (len(a),) + self.obs_shape
    return type(structure)(s_tm1.view(self.obs_dtype).reshape(shape), a, r, d, s_t.view(self.obs_dtype).reshape(shape))


# Default pool size is 2 * capacity + FRAME_POOL_SLACK planes.  For stacks built as `processors.atari()` builds them
# (trailing-zero padded, one new frame per step), the live planes of one actor stream are at most
# transitions + episodes + (stack - 1), and an episode holds at least one transition: 2 * capacity covers the
# transitions and episodes of every stream together, and the slack covers plane 0 plus the (stack - 1) planes of the
# oldest, partly evicted episode of up to 21 interleaved 4-deep streams (and the at most one new frame an add brings in
# before the evicted row releases its planes).
FRAME_POOL_SLACK = 64
_POOL_FULL = ('frame pool is full: an add found no free plane and stored zeros instead (frame_capacity=%d is too '
              'small for these observations; construct the replay with a larger frame_capacity)')


class _FramePoolStore(_TransitionStore):
  """Frame-deduplicated layout (DESIGN.md §3): an observation [H, W, C] uint8 is C planes of H*W bytes; every
  distinct plane is stored once in a device pool of `frame_capacity` planes and row = id % capacity keeps the 2*C
  plane ids of s_tm1 | s_t.  Content-addressed inserts and the reconstruction of HWC stacks run in CUDA
  (csrc/dz_frames.cu); `gather`, `get_rows` and `to_host_transition` return exactly the transition-major bytes."""

  def __init__(self, capacity, frame_capacity=None):
    super().__init__(capacity)
    if frame_capacity is not None and not 1 <= int(frame_capacity) < 2 ** 31:
      raise ValueError('frame_capacity must be in [1, 2**31)')
    self._requested = None if frame_capacity is None else int(frame_capacity)
    self.frames = None
    self.frame_capacity = 0

  def allocate(self, obs_shape, obs_dtype=np.uint8):
    if self.frames is not None:
      return
    shape, dtype = tuple(obs_shape), np.dtype(obs_dtype)
    if len(shape) != 3 or dtype != np.uint8:
      raise ValueError('frame_dedup stores 3-D uint8 observations [H, W, C]; got shape %s dtype %s' % (shape, dtype))
    h, w, c = shape
    if not 1 <= c <= 32:
      raise ValueError('frame_dedup supports 1..32 channels, got %d' % c)
    self.obs_shape, self.obs_dtype = shape, dtype
    self.obs_bytes = h * w * c
    self.obs_stride = (self.obs_bytes + 15) // 16 * 16
    self.channels = c
    self.frame_bytes = h * w
    self.frame_stride = (self.frame_bytes + 15) // 16 * 16
    fc = self._requested if self._requested is not None else 2 * self.capacity + FRAME_POOL_SLACK
    self.frame_capacity = fc
    self.table_size = 1 << max(1, (2 * fc - 1).bit_length())
    dev = self.action.device
    n = max(self.capacity, 1)
    self.frames = torch.empty((fc, self.frame_stride), dtype=torch.uint8, device=dev)
    self.planes = torch.zeros((n, 2 * c), dtype=torch.int32, device=dev)
    self.refcount = torch.zeros(fc, dtype=torch.int32, device=dev)
    self.hashes = torch.zeros(fc, dtype=torch.int64, device=dev)
    self.table = torch.empty(self.table_size, dtype=torch.int32, device=dev)
    self.free = torch.empty(fc, dtype=torch.int32, device=dev)
    self.counters = torch.zeros(1, dtype=torch.int64, device=dev)
    self.staging = torch.zeros(2 * self.obs_stride + 2 * c * self.frame_stride, dtype=torch.uint8, device=dev)
    self.reset()

  def fill_view(self, v):
    v.d_action, v.d_reward, v.d_discount = _ptr(self.action), _ptr(self.reward), _ptr(self.discount)
    v.capacity, v.obs_bytes, v.obs_stride = self.capacity, self.obs_bytes, self.obs_stride
    v.d_flags = _ptr(self.flags)
    if self.frames is not None:
      v.d_frames, v.frame_bytes, v.frame_stride = _ptr(self.frames), self.frame_bytes, self.frame_stride
      v.obs_channels, v.frame_capacity = self.channels, self.frame_capacity
      v.d_planes, v.d_refcount, v.d_hashes = _ptr(self.planes), _ptr(self.refcount), _ptr(self.hashes)
      v.d_table, v.table_size, v.d_free = _ptr(self.table), self.table_size, _ptr(self.free)
      v.d_pool_counters, v.d_add_staging = _ptr(self.counters), _ptr(self.staging)
    return v

  def reset(self):
    """Empties the pool: no row references a plane, the next fresh planes are 1, 2, 3, ..."""
    if self.frames is not None:
      _lib.call('dz_replay_frame_pool_reset', C.byref(self.fill_view(_lib.ReplayView())), _stream())

  def frames_in_use(self):
    """Live planes, plane 0 included (synchronises)."""
    if self.frames is None:
      return 0
    out = C.c_int64()
    _lib.call('dz_replay_frames_in_use', C.byref(self.fill_view(_lib.ReplayView())), C.byref(out), _stream())
    return out.value

  def storage_bytes(self):
    n = super().storage_bytes()
    if self.frames is not None:
      n += sum(t.numel() * t.element_size() for t in (self.frames, self.planes, self.refcount, self.hashes, self.table,
                                                      self.free, self.counters, self.staging))
    return n

  def check_pool(self, slots):
    """Each refcount equals its references from the live rows `slots` (+1 for plane 0), and the free stack and the
    live planes partition the pool."""
    if self.frames is None:
      return True, ''
    fc = self.frame_capacity
    planes = self.planes[torch.as_tensor(np.asarray(slots, dtype=np.int64), device=self.planes.device)].cpu().numpy()
    want = np.bincount(planes.reshape(-1), minlength=fc)
    want[0] += 1
    ref = self.refcount.cpu().numpy()
    bad = np.nonzero(ref != want)[0]
    if bad.size:
      return False, 'refcount of plane %d is %d, rows reference it %d times.' % (bad[0], ref[bad[0]], want[bad[0]])
    top = int(self.counters.item())
    free = self.free[:top].cpu().numpy()
    live = np.nonzero(ref)[0]
    if len(free) + len(live) != fc or len(np.union1d(free, live)) != fc:
      return False, 'free stack and live planes do not partition the frame pool.'
    return True, ''


def _make_store(capacity, frame_dedup, frame_capacity):
  if frame_dedup:
    return _FramePoolStore(capacity, frame_capacity)
  if frame_capacity is not None:
    raise ValueError('frame_capacity needs frame_dedup=True')
  return _TransitionStore(capacity)


def _host_obs(x, store):
  """Flat uint8 view of an observation to be written into a replay row.  Host arrays are copied H2D by
  dz_replay_add; CUDA tensors (e.g. the frame stack of `processors.atari(device_observations=True)`) are copied
  device-to-device on the same stream — the device-resident insert path, no host round trip."""
  if isinstance(x, torch.Tensor) and x.is_cuda:
    t = x.contiguous()
    dtype = np.dtype(str(t.dtype).replace('torch.', ''))
    store.allocate(tuple(t.shape), dtype)
    if tuple(t.shape) != store.obs_shape or dtype != store.obs_dtype:
      raise ValueError('observation shape/dtype changed: %s %s' % (tuple(t.shape), dtype))
    return t.view(torch.uint8).reshape(-1)
  arr = np.ascontiguousarray(x)
  store.allocate(arr.shape, arr.dtype)
  if arr.shape != store.obs_shape or arr.dtype != store.obs_dtype:
    raise ValueError('observation shape/dtype changed: %s %s' % (arr.shape, arr.dtype))
  return arr.view(np.uint8).reshape(-1)


ADD_BATCH_MAX = 256   # adds per dz_replay_add_batch call (the workspace holds two host-source copies per add)


class _AddBatchRecords:
  """The [K] record arrays of dz_add_batch as one pinned host block (numpy views, filled per call) and its device twin,
  shipped with one copy per call.  The host block is rewritten only after the previous copy out of it has completed."""

  _FIELDS = (('tree_index', np.int64, 1), ('evict_index', np.int64, 1), ('patch_pos', np.int64, 4),
             ('patch_val', np.int64, 4), ('reward', np.float64, 1), ('discount', np.float64, 1), ('leaf', np.float64, 1),
             ('action', np.int32, 1), ('release', np.int32, 1), ('patch_target', np.int32, 4))

  def __init__(self, max_count, device):
    offsets, off = {}, 0
    for name, dtype, per in self._FIELDS:
      offsets[name] = off
      off += per * max_count * np.dtype(dtype).itemsize
    self.host = torch.empty(off, dtype=torch.uint8).pin_memory()
    self.dev = torch.empty(off, dtype=torch.uint8, device=device)
    raw = self.host.numpy()
    self.h = {name: raw[offsets[name]:offsets[name] + per * max_count * np.dtype(dt).itemsize].view(dt)
              for name, dt, per in self._FIELDS}
    self.d = {name: self.dev.data_ptr() + offsets[name] for name in offsets}
    self._copied = torch.cuda.Event()
    self._pending = False

  def writable(self):
    if self._pending:
      self._copied.synchronize()
      self._pending = False
    return self.h

  def ship(self):
    self.dev.copy_(self.host, non_blocking=True)
    self._copied.record()
    self._pending = True


def _batch_obs(x, store, count):
  """`_host_obs` for a [K, *obs_shape] batch: (array or CUDA tensor kept alive for the call, address, bytes per item)."""
  if isinstance(x, torch.Tensor) and x.is_cuda:
    t = x.contiguous()
    dtype = np.dtype(str(t.dtype).replace('torch.', ''))
    shape, addr = tuple(t.shape), t.data_ptr()
  else:
    t = np.ascontiguousarray(x)
    dtype, shape, addr = t.dtype, t.shape, t.ctypes.data
  if len(shape) < 1 or shape[0] != count:
    raise ValueError('observations must have a leading axis of length %d, got shape %s' % (count, shape))
  store.allocate(shape[1:], dtype)
  if shape[1:] != store.obs_shape or dtype != store.obs_dtype:
    raise ValueError('observation shape/dtype changed: %s %s' % (shape[1:], dtype))
  return t, addr


def _batch_vector(x, count, dtype, name):
  if isinstance(x, torch.Tensor):
    x = x.detach().cpu().numpy()
  v = np.asarray(x)
  if v.shape != (count,):
    raise ValueError('%s must have shape (%d,), got %s' % (name, count, v.shape))
  return v.astype(dtype)


def _batch_items(items, codec, store):
  """Validates a batch `items` (Transition with a leading K axis) before anything changes: returns K, the observation
  sources (s_tm1, s_t) and the scalars as host arrays (action int32, reward / discount float64)."""
  count = len(items[1])
  if codec is not None:
    coded = [codec(type(items)(*[f[k] for f in items])) for k in range(count)]
    items = type(items)(*[np.stack([np.asarray(c[i]) for c in coded]) if count else np.asarray(items[i])
                          for i in range(5)])
  s_tm1 = _batch_obs(items[0], store, count)
  s_t = _batch_obs(items[4], store, count)
  # int(a) into an int32 record, float(r) into a double, as `add` does
  a = _batch_vector(items[1], count, np.int64, 'a_tm1').astype(np.int32)
  r = _batch_vector(items[2], count, np.float64, 'r_t')
  d = _batch_vector(items[3], count, np.float64, 'discount_t')
  return count, s_tm1, s_t, a, r, d


def _add_batch(rep, items, leaves=None, d_priority=None, alpha=1.0):
  """Shared body of `add_batch` on a validated batch (`_batch_items`): chunks of at most min(capacity, adds per call)
  transitions, so no call evicts a row it wrote itself, each add's host bookkeeping done by `rep._book()` as `add`
  does it."""
  count, (o_tm1, p_tm1), (o_t, p_t), a, r, d = items
  if count == 0:
    return
  store = rep._store
  v = rep.device_view()
  recs, ws, most = store.add_batch_buffers(v)
  chunk = min(rep._capacity, most)
  obs_bytes = store.obs_bytes
  for lo in range(0, count, chunk):
    k = min(chunk, count - lo)
    h = recs.writable()
    first_slot = rep._t % rep._capacity
    patches = []
    for j in range(k):
      release, evict, tree, p = rep._book()
      h['release'][j], h['evict_index'][j], h['tree_index'][j] = release, evict, tree
      patches.extend(p)
    n = len(patches)
    if n:
      pt = np.asarray(patches, dtype=np.int64)
      h['patch_target'][:n], h['patch_pos'][:n], h['patch_val'][:n] = pt[:, 0], pt[:, 1], pt[:, 2]
    h['action'][:k], h['reward'][:k], h['discount'][:k] = a[lo:lo + k], r[lo:lo + k], d[lo:lo + k]
    if leaves is not None:
      h['leaf'][:k] = leaves[lo:lo + k]
    recs.ship()
    b = _lib.AddBatch()
    b.count, b.first_slot = k, first_slot
    b.d_action, b.d_reward, b.d_discount = recs.d['action'], recs.d['reward'], recs.d['discount']
    b.d_release_row = recs.d['release']
    if leaves is not None:
      b.d_tree_index, b.d_evict_index, b.d_leaf_value = recs.d['tree_index'], recs.d['evict_index'], recs.d['leaf']
    b.d_priority = None if d_priority is None else d_priority.data_ptr()
    b.alpha = alpha
    b.n_patches = n
    b.d_patch_pos, b.d_patch_val, b.d_patch_target = recs.d['patch_pos'], recs.d['patch_val'], recs.d['patch_target']
    b.s_tm1, b.s_t, b.src_pitch = p_tm1 + lo * obs_bytes, p_t + lo * obs_bytes, obs_bytes
    _lib.call('dz_replay_add_batch', C.byref(v), C.byref(b), ws.data_ptr(), ws.numel(), _stream())


def _check_codec(encoder, decoder):
  """The reference stores `encoder(item)` and returns `decoder(stored)` (`replay.py:148,155`; every run_atari.py passes
  the snappy pair of `replay.py:895-904` so that 1M x 56 KB fits in host RAM).  HBM holds raw observations, so a codec
  pair is accepted and applied as the round trip `decoder(encoder(item))` on the host at insert time — the identity
  for a lossless codec such as snappy — and both must be given together."""
  if (encoder is None) != (decoder is None):
    raise ValueError('encoder and decoder must be given together')
  if encoder is None:
    return None
  return lambda item: decoder(encoder(item))


# ------------------------------------------------------------------------------------------------
# The body of both replays
# ------------------------------------------------------------------------------------------------


class _Replay:
  """What `TransitionReplay` and `PrioritizedTransitionReplay` share: the codec, the transition store, the ids stored
  oldest first, the add bookkeeping, state, checkpoints and checks.  A subclass builds its index distribution and
  defines the device view, the sticky flags, the id check of `get` (`_stored`), how a priority becomes a leaf in `add`
  and `add_batch`, and sampling."""

  def __init__(self, codec, capacity, structure, random_state, distribution, frame_dedup, frame_capacity):
    self._codec = codec
    self._capacity = capacity
    self._structure = structure
    self._random_state = random_state
    self._distribution = distribution
    self._store = _make_store(capacity, frame_dedup, frame_capacity)
    self._live_ids = collections.deque()   # ids currently stored, oldest first (keys of the OrderedDict)
    self._t = 0

  def _observations(self, item):
    """The codec round trip of one added item and its flat observations: (item, s_tm1, s_t)."""
    if self._codec is not None:
      item = self._codec(item)
    return item, _host_obs(item[0], self._store), _host_obs(item[4], self._store)

  def _book(self):
    """The host bookkeeping of one add, in `add` and `add_batch` alike: evicts the oldest id when the replay is full
    and registers id `_t`.  Returns (release_row, evict_index, tree_index, patches) of the add's device record."""
    evicted = self._live_ids.popleft() if self.size == self._capacity else None
    evict_index, tree_index = self._distribution._insert(self._t, evicted)
    self._live_ids.append(self._t)
    self._t += 1
    return evicted is not None, evict_index, tree_index, self._distribution.take_patches()

  def _add(self, item, s_tm1, s_t, **leaf):
    """`add` after `_observations`: the bookkeeping, then one dz_replay_add call carrying the row, the list patches
    and, for a prioritized add, the sum-tree fields `leaf`."""
    slot = self._t % self._capacity
    release, evict, tree, patches = self._book()
    assert len(patches) <= 4
    _apply_index_record(self.device_view(), patches, tree_index=tree, evict_index=evict, slot=slot,
                        action=int(item[1]), reward=float(item[2]), discount=float(item[3]), h_s_tm1=s_tm1, h_s_t=s_t,
                        release_row=release, **leaf)

  def get(self, ids: Sequence[int]):
    """`replay.py:153-156`."""
    ids = [int(i) for i in ids]
    for i in ids:
      if not self._stored(i):
        raise KeyError(i)
    self._raise_if_pool_full()
    return self._store.get_rows(self._structure, np.asarray(ids, dtype=np.int64) % self._capacity)

  @property
  def size(self) -> int:
    return len(self._live_ids)

  @property
  def capacity(self) -> int:
    return self._capacity

  @property
  def frames_in_use(self) -> int:
    """Live planes of the frame pool, plane 0 included (a synchronising read; for sizing `frame_capacity`)."""
    if not isinstance(self._store, _FramePoolStore):
      raise ValueError('frames_in_use needs a replay constructed with frame_dedup=True')
    return self._store.frames_in_use()

  @property
  def storage_bytes(self) -> int:
    """Device bytes of the transition storage (observations or frame pool, plus per-row scalars)."""
    return self._store.storage_bytes()

  def get_state(self) -> Mapping[str, Any]:
    """`replay.py:179-187` / `:747-754`: same keys; `storage` is a list of (id, Transition) with host arrays."""
    ids = list(self._live_ids)
    return {'storage': list(zip(ids, self.get(ids))) if ids else [], 't': self._t,
            'distribution': self._distribution.get_state()}

  def set_state(self, state: Mapping[str, Any]) -> None:
    """`replay.py:189-193` / `:756-760`."""
    _restore_rows(self, state['storage'])
    self._t = state['t']
    self._distribution.set_state(state['distribution'])

  def save_checkpoint(self, directory: str) -> None:
    """Writes the replay into `directory` (DESIGN.md §9): device arrays streamed through a fixed staging ring with a
    digest per chunk, the host bookkeeping as int64 arrays, a JSON manifest.  Host memory stays bounded by the ring
    plus the O(capacity) integer bookkeeping.  The RandomState is not saved (as for `get_state`).  The raw sum-tree
    nodes of a prioritized replay are written bit for bit."""
    from dqn_zoo_b200 import checkpoint as ck
    _replay_files(self, False).write(directory, ck.Transfer(self._store.action.device))

  def load_checkpoint(self, directory: str) -> None:
    """Restores `save_checkpoint` of a replay of the same class, layout, capacity, observation shape and
    frame_capacity: afterwards every device array and host list equals the saved replay's, the frame pool's plane
    ids and free stack included, so later adds and samples are those the saved replay would make.  A mismatch of
    those raises ValueError before anything changes; a digest, size or pool-consistency failure raises RuntimeError
    naming the file (and chunk) and leaves the replay empty."""
    from dqn_zoo_b200 import checkpoint as ck
    m = ck.read_manifest(directory, REPLAY_FORMAT)
    ck.validate(m, _checkpoint_header(self), directory)
    st = self._store
    saved_shape = None if m.get('obs_shape') is None else (tuple(m['obs_shape']), np.dtype(m['obs_dtype']))
    if saved_shape is not None and st.obs_shape is not None and saved_shape != (st.obs_shape, st.obs_dtype):
      raise ValueError('%s: checkpoint has observations %s %s, this replay stores %s %s'
                       % (directory, saved_shape[0], saved_shape[1], st.obs_shape, st.obs_dtype))
    try:
      _restore_checkpoint(self, directory, m, saved_shape, ck)
    except BaseException as e:
      _reset_empty(self)
      if isinstance(e, RuntimeError):
        raise
      raise RuntimeError('%s: checkpoint data is inconsistent (%s: %s); the replay was reset to empty'
                         % (directory, type(e).__name__, e)) from e

  def snapshot_checkpoint(self):
    """A `checkpoint.Snapshot` of the replay at the current point of the CUDA stream (DESIGN.md §9): device copies of
    the per-row scalars, the sum tree or id mirror, the plane table, the free stack and the live planes' ids and
    hashes, the observation bytes of the live rows packed and digested in one pass, and copies of the host
    bookkeeping.  Its `write(directory)` gives the files `save_checkpoint(directory)` would give now, byte for byte,
    while the replay goes on changing."""
    from dqn_zoo_b200 import checkpoint as ck
    held = []
    files = _replay_files(self, True, held)
    return ck.Snapshot(files.write, held, self._store.action.device)

  def snapshot_checkpoint_bytes(self) -> int:
    """An upper bound of the device memory `snapshot_checkpoint()` takes now (a synchronising read)."""
    return _snapshot_bytes(self)

  def check_valid(self) -> Tuple[bool, str]:
    """`replay.py:195-200` / `:762-768`, plus for a frame pool: the pool-full flag, refcounts and the free-stack
    partition."""
    if self._t < self.size:
      return False, 't should be >= storage size.'
    if set(self._live_ids) != set(self._distribution.ids()):
      return False, 'IDs in storage and distribution do not match.'
    if isinstance(self._store, _FramePoolStore):
      self._raise_if_pool_full()
      ok, msg = self._store.check_pool(np.asarray(list(self._live_ids), dtype=np.int64) % self._capacity)
      if not ok:
        return ok, msg
    return self._distribution.check_valid()

  def _raise_if_pool_full(self):
    """DZ_FLAG_FRAME_POOL_FULL is sticky: the stored bytes are wrong from that add on, so every sync point raises."""
    if isinstance(self._store, _FramePoolStore) and int(self._flags().item()) & _lib.DZ_FLAG_FRAME_POOL_FULL:
      raise RuntimeError(_POOL_FULL % self._store.frame_capacity)

  # -- what a learner step reads of the replay -----------------------------------------------------------------------
  def _flush(self):
    """Brings the device mirrors up to date with the host lists (before a learner step is captured)."""
    self._distribution.flush()

  def _alpha(self) -> float:
    """The priority exponent of the learner's priority write-back (1 for a replay without priorities)."""
    return 1.0

  def _sample_constants(self) -> Tuple[float, float, float, float]:
    """The last four words of the learner's staging record: size, importance-sampling exponent, uniform sample
    probability and normalize weights (1 or 0)."""
    return float(self.size), 1.0, 0.0, 0.0

  def _rng_state(self):
    """The state of the RandomState the samples are drawn from (which `get_state` leaves to the run)."""
    return self._random_state.get_state()

  def _set_rng_state(self, state) -> None:
    self._random_state.set_state(state)


# ------------------------------------------------------------------------------------------------
# R6: TransitionReplay
# ------------------------------------------------------------------------------------------------


class TransitionReplay(_Replay):
  """Uniform replay with oldest-out eviction (`replay.py:120-200`), storage in HBM.

  `frame_dedup=True` stores each distinct H*W plane of the (3-D uint8) observations once (`_FramePoolStore`,
  DESIGN.md §3): a reference-sized replay of 84x84x4 frame stacks then takes about a quarter of the HBM.  Everything
  read back (samples, `get`, `get_state`, learner batches) is byte-identical to the default transition-major layout.
  `frame_capacity` sizes the pool in planes (default 2 * capacity + FRAME_POOL_SLACK, enough for frame stacks built as
  `processors.atari()` builds them); running out is a data error, raised as RuntimeError at the next sync point.  The
  layout is the caller's choice because the replay cannot tell at construction whether its observations are frame
  stacks, and the pool has to be sized up front."""

  prioritized = False   # whether an agent adds with priorities and learns by them from this replay

  def __init__(self, capacity: int, structure, random_state: np.random.RandomState, encoder=None, decoder=None,
               frame_dedup: bool = False, frame_capacity: Optional[int] = None):
    super().__init__(_check_codec(encoder, decoder), capacity, structure, random_state,
                     UniformDistribution(random_state=random_state), frame_dedup, frame_capacity)
    self._distribution._mirror.ensure(capacity)   # fixed address: captured CUDA graphs keep pointing at it

  def device_view(self):
    v = self._store.fill_view(_lib.ReplayView())
    v.d_ids = _ptr(self._distribution.device_ids)
    return v

  def _flags(self):
    """The sticky device flags the kernels of this replay's view set."""
    return self._store.flags

  def _stored(self, i):
    return bool(self._live_ids) and self._live_ids[0] <= i <= self._live_ids[-1]

  def add(self, item) -> None:
    """`replay.py:142-151`."""
    self._add(*self._observations(item))

  def add_batch(self, items) -> None:
    """K transitions at once: `items` is a Transition whose fields have a leading K axis (observations [K, *obs_shape]
    as a numpy array or a CUDA tensor; a_tm1, r_t, discount_t of length K).  The replay afterwards equals the replay
    after `for k in range(K): add(item_k)`.  Unlike that loop, the whole batch is validated first: a shape or dtype
    mismatch raises what `add` raises and leaves the replay unchanged."""
    _add_batch(self, _batch_items(items, self._codec, self._store))

  def sample_device(self, size: int):
    """Host randint draw (`replay.py:78`), device id lookup + gather; returns device tensors."""
    picks = self._random_state.randint(self.size, size=size).astype(np.int64)
    dev = self._store.action.device
    d_pos = torch.as_tensor(picks, device=dev)
    out_i = torch.empty(2 * size, dtype=torch.int64, device=dev)
    sin = _lib.SampleInputs(_ptr(d_pos), None, None, None)
    sout = _lib.SampleOutputs(out_i.data_ptr(), None, out_i.data_ptr() + 8 * size, None, None)
    v = self.device_view()
    _lib.call('dz_replay_sample', C.byref(v), 0, C.byref(sin), C.byref(sout), size, _stream())
    return out_i[:size], out_i[size:], self._store.gather(out_i[size:], size)

  def sample(self, size: int):
    """`replay.py:158-165`."""
    _, _, tensors = self.sample_device(size)
    self._raise_if_pool_full()
    return self._store.to_host_transition(self._structure, tensors)

  def ids(self) -> Iterable[int]:
    return list(self._live_ids)


# ------------------------------------------------------------------------------------------------
# Checkpoint directories (DESIGN.md §9)
# ------------------------------------------------------------------------------------------------

REPLAY_FORMAT = 'dqn_zoo_b200.replay'
REPLAY_FORMAT_VERSION = 1


def _pool_capacity(store):
  """frame_capacity the store has or will allocate (None: transition-major)."""
  if not isinstance(store, _FramePoolStore):
    return None
  if store.frames is not None:
    return store.frame_capacity
  return store._requested if store._requested is not None else 2 * store.capacity + FRAME_POOL_SLACK


def _checkpoint_header(rep):
  return {'version': REPLAY_FORMAT_VERSION, 'kind': type(rep).__name__,
          'layout': 'frames' if isinstance(rep._store, _FramePoolStore) else 'rows', 'capacity': rep._capacity,
          'frame_capacity': _pool_capacity(rep._store)}


def _bytes_of(t):
  return t.reshape(-1).view(torch.uint8)


def _dict_array(d):
  return np.fromiter((x for kv in d.items() for x in kv), dtype=np.int64, count=2 * len(d)).reshape(-1, 2)


def _array_dict(a):
  return dict(zip(a[:, 0].tolist(), a[:, 1].tolist()))


def _slot_runs(slots):
  """(first slot, count, position) of each run of consecutive slots."""
  if not len(slots):
    return []
  cut = np.nonzero(np.diff(slots) != 1)[0] + 1
  starts = np.concatenate([[0], cut])
  ends = np.concatenate([cut, [len(slots)]])
  return [(int(slots[s]), int(e - s), int(s)) for s, e in zip(starts, ends)]


def _row_copier(rep, live, to_replay):
  """`Transfer` callback moving packed rows (live ids in order, 2 * obs_bytes each) from the staging buffer to the
  transition-major rows: with FIFO eviction the live slots are at most two runs, each one pitched copy."""
  st = rep._store
  row = 2 * st.obs_bytes
  v = st.fill_view(_lib.ReplayView())

  def copy(off, n, staging):
    r0 = off // row
    for first, count, pos in _slot_runs(live[r0:r0 + n // row] % rep._capacity):
      _lib.call('dz_ckpt_rows', C.byref(v), first, count, staging.data_ptr() + pos * row, int(to_replay), _stream())
    return staging
  return copy


def _replay_files(rep, snapshot, held=None):
  """The files and manifest of the replay's checkpoint directory (`checkpoint.Files`), ordered on the current stream
  after the work already enqueued there.  snapshot=False: the live arrays, read by the write that follows (the blocking
  save: host memory bounded by the staging ring).  snapshot=True: device copies (appended to `held`) and copies of the
  host containers, with the bulk records packed and digested per chunk by one `dz_ckpt_snapshot` pass, so the replay
  may change before the files are written."""
  from dqn_zoo_b200 import checkpoint as ck
  st, dist = rep._store, rep._distribution
  rep._raise_if_pool_full()
  dist.flush()                                    # device mirrors up to date with the host lists

  def dev(t):
    b = _bytes_of(t)
    if snapshot:
      b = b.clone()
      held.append(b)
    return b
  keep = copy.copy if snapshot else (lambda x: x)
  files = ck.Files()
  live = np.fromiter(rep._live_ids, dtype=np.int64, count=len(rep._live_ids))
  files.host['live_ids'] = lambda: live
  for name, kind in dist._HOST_LISTS.items():
    x = keep(getattr(dist, '_' + name))
    files.host[name] = (lambda x=x: _dict_array(x)) if kind is dict else (lambda x=x: np.asarray(x, dtype=np.int64))
  for name, t in dist._device_mirrors().items():
    files.dev[name] = dev(t)
  extra = dist._manifest()
  allocated = st.obs_shape is not None
  if allocated:
    for name in ('action', 'reward', 'discount'):
      files.dev[name] = dev(getattr(st, name))
    device = st.action.device
    v = st.fill_view(_lib.ReplayView())
    if isinstance(st, _FramePoolStore):
      fc = st.frame_capacity
      records = torch.empty(fc, dtype=torch.int32, device=device)    # the live plane ids
      hashes = torch.empty(fc, dtype=torch.int64, device=device)
      count = torch.zeros(1, dtype=torch.int64, device=device)
      _lib.call('dz_ckpt_pool_live', C.byref(v), _ptr(records), _ptr(hashes), _ptr(count), _stream())
      n, top = int(count.item()), int(st.counters.item())
      files.dev['planes'] = dev(st.planes)
      files.dev['free'] = dev(st.free[:top])
      files.dev['pool_ids'] = dev(records[:n])
      files.dev['pool_hashes'] = dev(hashes[:n])
      name, record = 'frames', st.frame_bytes
      extra.update(pool_top=top, pool_planes=n)
    else:
      n = len(live)
      records = torch.as_tensor((live % rep._capacity).astype(np.int32), device=device)   # the live rows' slots
      name, record = 'rows', 2 * st.obs_bytes
    chunk = max(1, ck.CHUNK_BYTES // record) * record
    if snapshot:
      packed = torch.empty(max(n * record, 1), dtype=torch.uint8, device=device)
      digests = torch.empty(max(-(-n * record // chunk), 1), dtype=torch.int64, device=device)
      _lib.call('dz_ckpt_snapshot', C.byref(v), _ptr(records), n, _ptr(packed), chunk, _ptr(digests), _stream())
      held.extend([packed, digests])
      files.bulk = (name, n * record, packed, chunk, digests)
    else:
      def pack(off, nb, staging, digest):
        _lib.call('dz_ckpt_snapshot', C.byref(v), _ptr(records) + 4 * (off // record), nb // record, staging.data_ptr(),
                  chunk, digest, _stream())
        return staging
      files.bulk = (name, n * record, pack, chunk, None)
  files.manifest = dict(_checkpoint_header(rep), format=REPLAY_FORMAT, t=rep._t,
                        obs_shape=list(st.obs_shape) if allocated else None,
                        obs_dtype=st.obs_dtype.str if allocated else None, **extra)
  return files


def _snapshot_bytes(rep):
  """An upper bound of the device bytes `_replay_files(rep, True)` allocates, transient buffers included (the frame
  pool's live count is a synchronising read)."""
  st = rep._store
  n = sum(t.numel() * t.element_size() for t in rep._distribution._device_mirrors().values())
  if st.obs_shape is None:
    return n
  n += sum(getattr(st, k).numel() * getattr(st, k).element_size() for k in ('action', 'reward', 'discount'))
  if isinstance(st, _FramePoolStore):
    live = st.frame_capacity - int(st.counters.item()) - 1
    n += st.planes.numel() * 4 + 4 * st.frame_capacity + 24 * st.frame_capacity + live * st.frame_bytes
    record = st.frame_bytes
  else:
    live = len(rep._live_ids)
    n += live * (4 + 2 * st.obs_bytes)
    record = 2 * st.obs_bytes
  from dqn_zoo_b200 import checkpoint as ck
  return n + 8 * (live * record // max(1, ck.CHUNK_BYTES // record * record) + 1) + 4096


def _reset_empty(rep):
  """A replay that failed to load: empty, with the host lists, mirrors' meaning, sum tree and pool of a new one."""
  rep._live_ids = collections.deque()
  rep._t = 0
  rep._distribution._reset(rep._capacity)
  if isinstance(rep._store, _FramePoolStore):
    rep._store.reset()
  rep._flags().zero_()


def _restore_checkpoint(rep, directory, m, saved_shape, ck):
  st, dist = rep._store, rep._distribution
  files = m['files']
  path = lambda name: os.path.join(directory, name + '.bin')
  host = {name: ck.Transfer.load_host(path(name), e) for name, e in files.items() if 'dtype' in e}
  live = host['live_ids']
  rep._flags().zero_()
  xfer = ck.Transfer(st.action.device)

  def dev(name, consume):
    xfer.load_device(path(name), files[name], consume)

  for key, value in dist._manifest().items():
    if m.get(key) != value:
      raise RuntimeError('%s: the manifest has %s = %r, this replay has %r' % (directory, key, m.get(key), value))
  for name, t in dist._device_mirrors().items():
    dev(name, _bytes_of(t))
  if saved_shape is not None:
    st.allocate(*saved_shape)
    for name in ('action', 'reward', 'discount'):
      dev(name, _bytes_of(getattr(st, name)))
    if isinstance(st, _FramePoolStore):
      _restore_pool(rep, directory, m, live, dev)
    else:
      dev('rows', _row_copier(rep, live, True))
  # host bookkeeping last: the same containers, filled in the saved insertion order
  rep._live_ids = collections.deque(live.tolist())
  rep._t = int(m['t'])
  for name, kind in dist._HOST_LISTS.items():
    setattr(dist, '_' + name, _array_dict(host[name]) if kind is dict else host[name].tolist())
  dist._pending = []


def _restore_pool(rep, directory, m, live, dev):
  """Plane table, plane bytes and free stack from the files; refcounts, hashes and the lookup table rebuilt on the
  device and checked against the saved live list and hashes."""
  st = rep._store
  fc, n, top = st.frame_capacity, int(m['pool_planes']), int(m['pool_top'])
  if not (0 <= n < fc and 0 <= top < fc and n + 1 + top == fc):
    raise RuntimeError('%s: %d live planes and a free stack of %d do not partition a pool of %d planes'
                       % (directory, n, top, fc))
  device = st.frames.device
  st.reset()
  dev('planes', _bytes_of(st.planes))
  ids = torch.empty(max(n, 1), dtype=torch.int32, device=device)
  hashes = torch.empty(max(n, 1), dtype=torch.int64, device=device)
  dev('pool_ids', _bytes_of(ids)[:4 * n])
  dev('pool_hashes', _bytes_of(hashes)[:8 * n])
  bad = torch.zeros(4, dtype=torch.int32, device=device)
  v = st.fill_view(_lib.ReplayView())
  fb = st.frame_bytes

  def scatter(off, nb, staging):
    _lib.call('dz_ckpt_pool_scatter', C.byref(v), _ptr(ids) + 4 * (off // fb), nb // fb, staging.data_ptr(), _ptr(bad),
              _stream())
  dev('frames', scatter)
  dev('free', _bytes_of(st.free)[:4 * top])
  st.counters.fill_(top)
  slots = torch.as_tensor(live % rep._capacity, device=device)
  _lib.call('dz_ckpt_pool_rebuild', C.byref(v), _ptr(slots), len(live), _ptr(ids), _ptr(hashes), n, top, _ptr(bad),
            _stream())
  got = bad.cpu().numpy()
  flags, referenced = int(got[0]), int(got.view(np.uint64)[1])
  if flags or referenced != n + 1:
    what = [text for bit, text in ((_lib.DZ_CKPT_BAD_PLANE_ID, 'a plane id out of range or an unsorted live list'),
                                   (_lib.DZ_CKPT_UNREFERENCED_PLANE, 'a listed plane no live row references'),
                                   (_lib.DZ_CKPT_HASH_MISMATCH, 'a plane whose bytes do not match its saved hash'),
                                   (_lib.DZ_CKPT_BAD_FREE_STACK, 'a free-stack entry naming a referenced plane'))
            if flags & bit]
    if referenced != n + 1:
      what.append('%d referenced planes for %d listed (+ plane 0)' % (referenced, n))
    raise RuntimeError('%s: frame pool is inconsistent: %s' % (directory, '; '.join(what)))


def _restore_rows(rep, storage):
  """Rewrites device rows from a `storage` list of (id, item) (set_state).  A frame pool is emptied first and the rows
  are re-added in id order, so the plane table is the one those adds leave (and either layout loads the other's
  state)."""
  if isinstance(rep._store, _FramePoolStore):
    storage = sorted(storage, key=lambda x: int(x[0]))
    rep._store.reset()
    rep._flags().bitwise_and_(~_lib.DZ_FLAG_FRAME_POOL_FULL)   # the emptied pool holds no wrong bytes
  rep._live_ids = collections.deque(int(i) for i, _ in storage)
  v = None
  for i, item in storage:
    s_tm1 = _host_obs(item[0], rep._store)
    s_t = _host_obs(item[4], rep._store)
    if v is None:
      v = rep.device_view()
    _apply_index_record(v, [], slot=int(i) % rep._capacity, action=int(item[1]), reward=float(item[2]),
                        discount=float(item[3]), h_s_tm1=s_tm1, h_s_t=s_t)


# ------------------------------------------------------------------------------------------------
# R5: PrioritizedTransitionReplay
# ------------------------------------------------------------------------------------------------


class PrioritizedTransitionReplay(_Replay):
  """Proportional prioritized replay (`replay.py:654-768`), storage + sum tree in HBM."""

  prioritized = True    # as TransitionReplay.prioritized

  def __init__(self, capacity: int, structure, priority_exponent: float,
               importance_sampling_exponent: Callable[[int], float], uniform_sample_probability: float,
               normalize_weights: bool, random_state: np.random.RandomState, encoder=None, decoder=None,
               frame_dedup: bool = False, frame_capacity: Optional[int] = None):
    """`frame_dedup` / `frame_capacity`: the storage layout, as for `TransitionReplay`."""
    super().__init__(_check_codec(encoder, decoder), capacity, structure, random_state, PrioritizedDistribution(
        min_capacity=capacity, max_capacity=capacity, priority_exponent=priority_exponent,
        uniform_sample_probability=uniform_sample_probability, random_state=random_state), frame_dedup, frame_capacity)
    self._importance_sampling_exponent = importance_sampling_exponent
    self._normalize_weights = normalize_weights

  def device_view(self):
    v = self._distribution.device_view()
    self._store.fill_view(v)
    v.d_flags = _ptr(self._distribution._sum_tree._flags)
    return v

  def _flags(self):
    return self._distribution._sum_tree._flags

  def _stored(self, i):
    return i in self._distribution._id_to_index

  def add(self, item, priority: float) -> None:
    """`replay.py:690-699`: one device call carries the row, the list patches, the evicted
    leaf's zeroing and the new leaf (= priority**alpha evaluated in float64 on the host, as
    `replay.py:507` does)."""
    item, s_tm1, s_t = self._observations(item)
    alpha = self._distribution._priority_exponent
    d_priority = None
    if isinstance(priority, torch.Tensor):
      # priority kept on the device by the agent (max_seen_priority); exact for alpha in {0.5, 1}
      if alpha in (0.5, 1.0):
        d_priority, priority = priority, 1.0
      else:
        priority = float(priority.item())
    leaf = np.asarray(_power([priority], alpha))
    if not np.isfinite(leaf).all() or (leaf < 0.0).any():
      raise ValueError('value must be finite and positive.')
    self._add(item, s_tm1, s_t, leaf_value=float(leaf[0]), size_after=self._distribution._sum_tree.size,
              d_priority=d_priority, alpha=float(alpha))

  def add_batch(self, items, priorities) -> None:
    """K transitions at once (`items` as for `TransitionReplay.add_batch`).  `priorities`: a float, a length-K sequence
    or array, or a device float32 scalar tensor (the agent's max_seen_priority, taken on the device for alpha in
    {0.5, 1} as `add` does).  The replay afterwards equals the replay after `for k: add(item_k, priority_k)`.  Unlike
    that loop, the whole batch is validated first: a bad priority or a shape or dtype mismatch raises what `add` raises
    and leaves the replay unchanged."""
    batch = _batch_items(items, self._codec, self._store)
    count = batch[0]
    alpha = self._distribution._priority_exponent
    d_priority = None
    if isinstance(priorities, torch.Tensor) and priorities.numel() == 1 and priorities.is_cuda \
        and priorities.dtype == torch.float32 and alpha in (0.5, 1.0):
      d_priority, pri = priorities, np.ones(count)
    else:
      if isinstance(priorities, torch.Tensor):
        priorities = priorities.detach().cpu().numpy()
      pri = np.asarray(priorities, dtype=np.float64)
      if pri.ndim == 0:
        pri = np.full(count, float(pri))
      elif pri.shape != (count,):
        raise ValueError('priorities must be a scalar or have shape (%d,), got %s' % (count, pri.shape))
    leaves = np.asarray(_power(pri, alpha), dtype=np.float64)
    if not np.isfinite(leaves).all() or (leaves < 0.0).any():
      raise ValueError('value must be finite and positive.')
    _add_batch(self, batch, leaves=leaves, d_priority=d_priority, alpha=float(alpha))

  def sample_device(self, size: int):
    """Sampling + gather, everything left on the device: (ids, indices, slots, probs, weights, batch)."""
    beta = self.importance_sampling_exponent
    if not 0.0 <= beta <= 1.0:
      raise ValueError('Require 0 <= exponent <= 1.')
    ids, indices, slots, probs, weights = self._distribution.sample_device(
        size, beta=beta, normalize=self._normalize_weights, capacity_for_slots=self._capacity)
    return ids, indices, slots, probs, weights, self._store.gather(slots, size)

  def sample(self, size: int):
    """`replay.py:701-723`: (Transition of stacked arrays, ids int64, weights float64)."""
    ids, _, _, _, weights, tensors = self.sample_device(size)
    tr = self._store.to_host_transition(self._structure, tensors)
    w = weights.cpu().numpy()
    self._raise_if_pool_full()
    self._distribution._sum_tree._raise_flags()
    if not np.isfinite(w).all():
      raise ValueError('Weights are not finite: %s.' % w)
    return tr, ids.cpu().numpy(), w

  def update_priorities(self, ids: Sequence[int], priorities: Sequence[float]) -> None:
    """`replay.py:725-730`."""
    self._distribution.update_priorities(ids, np.asarray(priorities))

  @property
  def importance_sampling_exponent(self):
    """`replay.py:742-745`."""
    return self._importance_sampling_exponent(self._t)

  def _alpha(self):
    return self._distribution._priority_exponent

  def _sample_constants(self):
    return (float(self.size), float(self.importance_sampling_exponent),
            float(self._distribution._uniform_sample_probability), 1.0 if self._normalize_weights else 0.0)


def bulk_fill_synthetic(rep, obs_shape, seed, num_actions, discount=0.99, priority=1.0):
  """Benchmark/test helper: brings `rep` (uniform or prioritized, empty) to the exact state it
  has after `capacity` sequential `add()`s of synthetic transitions (ids 0..C-1, priority
  `priority` each) without C host->device copies: contents are generated on the device
  (dz_replay_fill_synthetic, byte-identical to oracle/replay_oracle.py:synthetic_rows) and the
  host bookkeeping is written in closed form (allocation order of replay.py:457,499: id i gets
  tree index C-1-i)."""
  assert rep._t == 0 and rep.size == 0
  if isinstance(rep._store, _FramePoolStore):
    raise ValueError('bulk_fill_synthetic writes iid rows that share no frames; fill a frame_dedup replay with '
                     'bulk_fill_synthetic_stacked')
  cap = rep._capacity
  rep._store.allocate(obs_shape, np.uint8)
  v = rep._store.fill_view(_lib.ReplayView())
  _lib.call('dz_replay_fill_synthetic', C.byref(v), 0, cap, int(seed), int(num_actions), float(discount), _stream())
  _fill_bookkeeping(rep, priority)


def bulk_fill_synthetic_stacked(rep, obs_shape, seed, num_actions, episode_len=1000, discount=0.99, priority=1.0):
  """`bulk_fill_synthetic` with frame stacks instead of iid rows, for either layout: transition i is step
  i % episode_len of episode i // episode_len, its observations trailing-zero-padded stacks of splitmix frames
  (dz_replay_fill_synthetic_stacked, byte-identical to oracle/frame_pool_oracle.py:synthetic_stacked_rows).  A
  frame_dedup replay is left with the plane table, refcounts and free stack that `capacity` sequential adds leave."""
  assert rep._t == 0 and rep.size == 0
  if len(obs_shape) != 3:
    raise ValueError('stacked fill needs [H, W, C] observations')
  cap = rep._capacity
  rep._store.allocate(obs_shape, np.uint8)
  v = rep.device_view()
  v.obs_channels = int(obs_shape[2])
  _lib.call('dz_replay_fill_synthetic_stacked', C.byref(v), cap, int(seed), int(episode_len), int(num_actions),
            float(discount), _stream())
  _fill_bookkeeping(rep, priority)


def _fill_bookkeeping(rep, priority):
  """Host state (and device mirrors) of `capacity` sequential adds of ids 0..C-1 with priority `priority`."""
  cap = rep._capacity
  rep._live_ids = collections.deque(range(cap))
  rep._t = cap
  rep._distribution._fill(cap, priority)


# ------------------------------------------------------------------------------------------------
# R7: accumulators (host, insert time)
# ------------------------------------------------------------------------------------------------


def _fold_n_steps(window):
  """`replay.py:808-824`: discounted return and discount product in python floats (f64)."""
  ret, disc = 0.0, 1.0
  for tr in window:
    ret += disc * tr.r_t
    disc *= tr.discount_t
  return Transition(s_tm1=window[0].s_tm1, a_tm1=window[0].a_tm1, r_t=ret, discount_t=disc, s_t=window[-1].s_t)


class NStepTransitionAccumulator:
  """`replay.py:827-892`."""

  def __init__(self, n):
    self._transitions = collections.deque(maxlen=n)
    self.reset()

  def step(self, timestep_t, a_t) -> Iterable[Transition]:
    if timestep_t.first():
      self.reset()
    if self._timestep_tm1 is None:
      if not timestep_t.first():
        raise ValueError('Expected FIRST timestep, got %s.' % str(timestep_t))
      self._timestep_tm1, self._a_tm1 = timestep_t, a_t
      return []
    self._transitions.append(Transition(s_tm1=self._timestep_tm1.observation, a_tm1=self._a_tm1,
                                        r_t=timestep_t.reward, discount_t=timestep_t.discount,
                                        s_t=timestep_t.observation))
    self._timestep_tm1, self._a_tm1 = timestep_t, a_t
    out = []
    if timestep_t.last():
      while self._transitions:
        out.append(_fold_n_steps(list(self._transitions)))
        self._transitions.popleft()
    elif len(self._transitions) == self._transitions.maxlen:
      out.append(_fold_n_steps(list(self._transitions)))
    return out

  def reset(self) -> None:
    self._transitions.clear()
    self._timestep_tm1 = None
    self._a_tm1 = None


class VectorNStepAccumulator:
  """`num_streams` independent `NStepTransitionAccumulator`s as array code: the insert-side counterpart of
  `processors.VectorScalars`, fed the struct-of-arrays timesteps of `VectorizedAtariPreprocessor.step_arrays` and
  emitting one Transition with a leading K axis for `add_batch`.

  The emitting streams' observations are copied into a device ring [E][n + 1][*obs_shape] (the caller's stacks are
  overwritten in place on later ticks); the returned s_tm1 / s_t are gathered from it into fresh [K] tensors.  Returns
  and discounts are folded in float64 as `_fold_n_steps` does, one numpy multiply and one add per step, which round as
  the Python floats do."""

  FIRST, MID, LAST = 0, 1, 2

  def __init__(self, num_streams: int, n: int, device='cuda'):
    if num_streams < 1 or n < 1:
      raise ValueError('num_streams and n must be positive')
    self._E, self._n = int(num_streams), int(n)
    self._device = torch.device(device)
    self._ring = None
    self._len = np.zeros(self._E, np.int64)      # transitions in each stream's window
    self._pos = np.zeros(self._E, np.int64)      # ring slot of each stream's latest observation
    self._has_tm1 = np.zeros(self._E, bool)
    self._a_tm1 = np.zeros(self._E, np.int64)
    self._r = np.zeros((self._E, self._n))       # window of each stream, oldest transition first
    self._d = np.zeros((self._E, self._n))
    self._a = np.zeros((self._E, self._n), np.int64)

  def reset(self, stream: Optional[int] = None) -> None:
    sel = slice(None) if stream is None else stream
    self._len[sel] = 0
    self._has_tm1[sel] = False

  _STATE_ARRAYS = ('_len', '_pos', '_has_tm1', '_a_tm1', '_r', '_d', '_a')

  def get_state(self) -> Mapping[str, Any]:
    """The pending windows of every stream, with the observation ring copied to the host."""
    state = {k.lstrip('_'): getattr(self, k).copy() for k in self._STATE_ARRAYS}
    state['ring'] = None if self._ring is None else self._ring.cpu().numpy()
    return state

  def set_state(self, state: Mapping[str, Any]) -> None:
    """Restores `get_state()` of an accumulator with the same stream count and n."""
    if np.shape(state['r']) != (self._E, self._n):
      raise ValueError('state is for [streams, n] = %s, this accumulator is %s' % (np.shape(state['r']), (self._E, self._n)))
    for k in self._STATE_ARRAYS:
      setattr(self, k, np.array(state[k.lstrip('_')], copy=True))
    self._ring = None if state['ring'] is None else torch.as_tensor(state['ring']).to(self._device)

  def step(self, emit, step_type, reward, discount, observations, actions) -> Optional[Transition]:
    """emit: bool [E], the streams with a new timestep; step_type / reward / discount: [E] (NaN = None); observations:
    [E, *obs_shape] (e.g. `VectorizedAtariPreprocessor.stacks`); actions: [E], the a_t chosen on this timestep.
    Returns the transitions completed this tick in stream-major order, or None."""
    e = np.nonzero(np.asarray(emit, bool))[0]
    if e.size == 0:
      return None
    st = np.asarray(step_type)[e].astype(np.int64)
    first = st == self.FIRST
    bad = ~first & ~self._has_tm1[e]
    if bad.any():
      k = int(np.argmax(bad))
      raise ValueError('Expected FIRST timestep, got step_type %d on stream %d.' % (st[k], e[k]))
    if isinstance(actions, torch.Tensor):
      actions = actions.detach().cpu().numpy()
    act = np.asarray(actions)[e].astype(np.int64)
    rw = np.asarray(reward, np.float64)[e]
    dc = np.asarray(discount, np.float64)[e]
    n, ring_n = self._n, self._n + 1
    if isinstance(observations, torch.Tensor):
      obs = observations.index_select(0, torch.as_tensor(e, device=observations.device)).to(self._device)
    else:
      obs = torch.as_tensor(np.asarray(observations)[e], device=self._device)
    if self._ring is None:
      self._ring = torch.zeros((self._E * ring_n,) + tuple(obs.shape[1:]), dtype=obs.dtype, device=self._device)
    pos = np.where(first, 0, (self._pos[e] + 1) % ring_n)
    self._ring[torch.as_tensor(e * ring_n + pos, device=self._device)] = obs
    # FIRST resets the stream; every other timestep appends (s_tm1, a_tm1, r_t, discount_t, s_t) to its window
    self._len[e[first]] = 0
    app = e[~first]
    L = self._len[app]
    full = app[L == n]
    if full.size:
      for w in (self._r, self._d, self._a):
        w[full, :-1] = w[full, 1:]
    L = np.minimum(L, n - 1)
    self._r[app, L], self._d[app, L], self._a[app, L] = rw[~first], dc[~first], self._a_tm1[app]
    self._len[app] = L + 1
    self._pos[e], self._a_tm1[e], self._has_tm1[e] = pos, act, True
    # LAST: the n, n-1, ..., 1-step windows ending at s_T; otherwise the full window
    last = st == self.LAST
    L = self._len[e]
    count = np.where(last, L, (L == n).astype(np.int64))
    total = int(count.sum())
    self._len[e[last]] = 0
    if total == 0:
      return None
    rows = np.repeat(e, count)
    start = np.arange(total) - np.repeat(np.cumsum(count) - count, count)
    end = np.repeat(L, count)
    ret, disc = np.zeros(total), np.ones(total)
    with np.errstate(all='ignore'):
      for j in range(n):
        m = (start <= j) & (j < end)
        ret = np.where(m, ret + disc * self._r[rows, j], ret)
        disc = np.where(m, disc * self._d[rows, j], disc)
    latest = self._pos[rows]
    tm1 = (latest - (end - start)) % ring_n
    s_tm1 = self._ring[torch.as_tensor(rows * ring_n + tm1, device=self._device)]
    s_t = self._ring[torch.as_tensor(rows * ring_n + latest, device=self._device)]
    return Transition(s_tm1=s_tm1, a_tm1=self._a[rows, start], r_t=ret, discount_t=disc, s_t=s_t)


class TransitionAccumulator(NStepTransitionAccumulator):
  """`replay.py:771-805` (the n = 1 case; equivalence pinned by `replay_test.py:264-280`)."""

  def __init__(self):
    super().__init__(1)
