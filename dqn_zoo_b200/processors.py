"""Device-backed Atari preprocessing: the `processors.atari()` surface of the reference (dqn_zoo/processors.py:399-505).

Same call protocol — a processor is a callable with `reset()`, fed one raw timestep per frame, returning `None`
on the frames where the previous action is repeated and a processed timestep otherwise — but the pixel work
(max-pool of the last two raw frames, rgb2y, PIL bilinear resize, frame stack; processors.py:367-388, 482-501)
runs in one CUDA kernel (csrc/dz_preprocess.cu) for any number of environment streams at once, and the frame
stacks live in device memory so that acting (`Learner.q_values`) and replay inserts can consume them without a
host round trip.  The scalar half (life-loss discount, action-repeat cadence, reward sum/clip, discount product,
step-type reduction; processors.py:121-215, 254-365) is a per-stream host state machine.

There is no CPU fallback: without the CUDA library the import of `dqn_zoo_b200._lib` fails.
"""

import ctypes as C
import math
from typing import Any, List, Mapping, Optional, Sequence, Tuple

import numpy as np
import torch

from dqn_zoo_b200 import _lib
from dqn_zoo_b200 import parts

StepType = parts.StepType

# processors.py:370 — the third weight is computed, not the literal 0.114
LUMA = (0.299, 0.587, 1 - (0.299 + 0.587))
_PRECISION_BITS = 32 - 8 - 2


def bilinear_axis(in_size: int, out_size: int) -> Tuple[np.ndarray, np.ndarray, int]:
  """Window + fixed-point coefficient tables of Pillow's bilinear resampling along one axis.

  (Pillow libImaging/Resample.c precompute_coeffs / normalize_coeffs_8bpc; Pillow is what processors.py:381-386
  calls.)  Returns bounds int32 [out, 2] = (first, count), kk int32 [out, ksize], ksize."""
  scale = in_size / out_size
  filterscale = scale if scale > 1.0 else 1.0
  support = filterscale                      # bilinear filter support is 1.0
  ksize = int(math.ceil(support)) * 2 + 1
  bounds = np.zeros((out_size, 2), np.int32)
  kk = np.zeros((out_size, ksize), np.int32)
  inv = 1.0 / filterscale
  one = float(1 << _PRECISION_BITS)
  for xx in range(out_size):
    center = (xx + 0.5) * scale
    first = max(int(center - support + 0.5), 0)
    last = min(int(center + support + 0.5), in_size)
    weights = []
    total = 0.0
    for x in range(first, last):
      t = abs((x - center + 0.5) * inv)
      w = 1.0 - t if t < 1.0 else 0.0
      weights.append(w)
      total += w
    bounds[xx, 0], bounds[xx, 1] = first, last - first
    for i, w in enumerate(weights):
      if total != 0.0:
        w = w / total
      kk[xx, i] = int(w * one - 0.5) if w < 0 else int(w * one + 0.5)
  return bounds, kk, ksize


class _Axis:
  """Device copy of one axis' tables + the C struct pointing at them."""

  def __init__(self, in_size, out_size, device):
    bounds, kk, ksize = bilinear_axis(in_size, out_size)
    self.bounds_host = bounds
    self.d_bounds = torch.from_numpy(bounds).to(device)
    self.d_kk = torch.from_numpy(kk).to(device)
    self.c = _lib.ResampleAxis(self.d_bounds.data_ptr(), self.d_kk.data_ptr(), ksize, in_size, out_size)


class _Stream:
  """Scalar state of one environment stream (everything processors.atari() keeps besides pixels)."""

  def __init__(self, repeats):
    self.repeats = repeats
    self.reset()

  def reset(self):
    self.lives = None
    self.index = (-1) % self.repeats          # FixedPaddedBuffer(length, initial_index=-1), processors.py:142-145
    self.slots = [None] * self.repeats        # (step_type, reward, discount) or None
    self.has_frame = [False] * self.repeats
    self.since_first = None
    self.should_reset = False
    self.count = 0                            # frames in the stack deque


class BatchedAtariPreprocessor:
  """`processors.atari()` for `num_streams` independent environment streams sharing one kernel launch per tick."""

  def __init__(self, num_streams: int = 1, additional_discount: float = 0.99, max_abs_reward: Optional[float] = 1.0,
               resize_shape: Optional[Tuple[int, int]] = (84, 84), num_action_repeats: int = 4, num_pooled_frames: int = 2,
               zero_discount_on_life_loss: bool = True, num_stacked_frames: int = 4, grayscaling: bool = True,
               device: Any = 'cuda', device_observations: bool = False):
    if not grayscaling or resize_shape is None or num_pooled_frames != 2:
      raise ValueError('the device preprocessing implements the standard DQN pipeline only: grayscaling=True, '
                       'a resize_shape, num_pooled_frames=2')
    if num_action_repeats < 2:
      raise ValueError('num_action_repeats must be >= num_pooled_frames')
    self._n = num_streams
    self._gamma = additional_discount
    self._clip = max_abs_reward
    self._out = tuple(resize_shape)
    self._repeats = num_action_repeats
    self._life_loss = zero_discount_on_life_loss
    self._stack = num_stacked_frames
    self._device = torch.device(device)
    self._device_obs = device_observations
    self._streams = [_Stream(num_action_repeats) for _ in range(num_streams)]
    self._in_shape = None
    self._luma = (C.c_double * 3)(*LUMA)
    self._band_rows = int(_lib.lib.dz_atari_preprocess_band_rows())

  # -- device state, created when the first frame tells us the raw geometry ------------------------------------
  def _allocate(self, shape):
    h, w, c = shape
    if c != 3:
      raise ValueError('expected RGB frames [H, W, 3], got %s' % (shape,))
    self._in_shape = (h, w, 3)
    oh, ow = self._out
    self._axis_h = _Axis(w, ow, self._device)
    self._axis_v = _Axis(h, oh, self._device)
    bv = self._axis_v.bounds_host
    self._max_band_rows = max(
        int(bv[min(y0 + self._band_rows, oh) - 1].sum() - bv[y0, 0]) for y0 in range(0, oh, self._band_rows))
    # only the last two slots of the action-repeat buffer are ever pooled (processors.py:485)
    self._raw = torch.zeros((self._n, 2, h, w, 3), dtype=torch.uint8, device=self._device)
    # one pinned staging area + one H2D copy per tick and pooled slot instead of one copy per stream
    self._stage = [torch.zeros((self._n, h, w, 3), dtype=torch.uint8).pin_memory() for _ in range(2)]
    self._stage_np = [t.numpy() for t in self._stage]
    self._stage_dev = torch.zeros((self._n, h, w, 3), dtype=torch.uint8, device=self._device) if self._n > 1 else None
    self._stage_done = [torch.cuda.Event() for _ in range(2)]
    self._stage_pending = [False, False]
    self._stacks = torch.zeros((self._n, oh, ow, self._stack), dtype=torch.uint8, device=self._device)
    self._meta_host = torch.zeros((4, self._n), dtype=torch.int64).pin_memory()
    self._meta = torch.zeros((4, self._n), dtype=torch.int64, device=self._device)
    self._counts = torch.zeros(self._n, dtype=torch.int32, device=self._device)
    self._meta_done = torch.cuda.Event()
    self._meta_pending = False

  def reset(self, stream: Optional[int] = None) -> None:
    for i in (range(self._n) if stream is None else [stream]):
      self._streams[i].reset()
      if self._in_shape is not None:
        self._stacks[i].zero_()

  @property
  def stacks(self) -> torch.Tensor:
    """uint8 [num_streams, out_h, out_w, num_stacked_frames] on the device (valid after the first emission)."""
    return self._stacks

  # -- one tick: one raw timestep per stream (None = stream idle this tick) ---------------------------------------
  def step(self, timesteps: Sequence[Any]) -> List[Any]:
    if len(timesteps) != self._n:
      raise ValueError('expected %d timesteps' % self._n)
    emit = []
    scalars = [None] * self._n
    uploads = ([], [])                          # per pooled slot: streams whose new frame goes there this tick
    for e, ts in enumerate(timesteps):
      if ts is None:
        continue
      st = self._streams[e]
      rgb, lives = ts.observation
      if self._in_shape is None:
        self._allocate(np.shape(rgb))
      step_type, reward, discount = ts.step_type, ts.reward, ts.discount
      if self._life_loss:                       # ZeroDiscountOnLifeLoss, processors.py:254-260
        lost = step_type == StepType.MID and lives < st.lives
        st.lives = lives
        if lost:
          discount = 0.0
      if st.index >= self._repeats:             # FixedPaddedBuffer, processors.py:146-154
        st.index = 0
        st.slots = [None] * self._repeats
        st.has_frame = [False] * self._repeats
      st.slots[st.index] = (step_type, reward, discount)
      pooled_slot = st.index - (self._repeats - 2)
      if pooled_slot >= 0:
        frame = np.ascontiguousarray(rgb, dtype=np.uint8)
        if frame.shape != self._in_shape:
          raise ValueError('frame shape changed: %s vs %s' % (frame.shape, self._in_shape))
        if self._stage_pending[pooled_slot] and not uploads[pooled_slot]:
          self._stage_done[pooled_slot].synchronize()        # the previous copy out of this staging area has finished
          self._stage_pending[pooled_slot] = False
        np.copyto(self._stage_np[pooled_slot][len(uploads[pooled_slot])], frame)
        uploads[pooled_slot].append(e)
        st.has_frame[st.index] = True
      st.index += 1
      if self._should_emit(st):
        scalars[e] = self._reduce_scalars(st)
        emit.append(e)
    for slot in (0, 1):
      if uploads[slot]:
        self._upload(slot, uploads[slot])
    if emit:
      self._launch(emit)
    outs = [None] * self._n
    for e in emit:
      step_type, reward, discount = scalars[e]
      # a snapshot, not a view: accumulators and the replay keep references across later emissions
      obs = self._stacks[e].clone() if self._device_obs else self._stacks[e].cpu().numpy()
      outs[e] = parts.TimeStep(step_type=step_type, reward=reward, discount=discount, observation=obs)
    return outs

  def _upload(self, slot, streams):
    """Staged frames [0, k) of `slot` -> raw[streams, slot]: one async H2D, then (if needed) one device scatter."""
    k = len(streams)
    src = self._stage[slot][:k]
    if k == self._n and streams == list(range(k)):
      self._raw[:, slot].copy_(src, non_blocking=True)
    elif k == 1:
      self._raw[streams[0], slot].copy_(src[0], non_blocking=True)
    else:
      dev = self._stage_dev[:k]
      dev.copy_(src, non_blocking=True)
      index = torch.as_tensor(streams, dtype=torch.int64).to(self._device)
      self._raw[:, slot].index_copy_(0, index, dev)
    self._stage_done[slot].record()
    self._stage_pending[slot] = True

  def _should_emit(self, st) -> bool:           # TimestepBufferCondition, processors.py:165-215
    if st.should_reset:
      raise RuntimeError('Should have reset.')
    main = StepType.MID
    for v in st.slots:
      if v is None:
        continue
      if v[0] in (StepType.FIRST, StepType.LAST):
        if main in (StepType.FIRST, StepType.LAST):
          raise RuntimeError('Expected at most one FIRST or LAST.')
        main = v[0]
    if st.since_first is None and main != StepType.FIRST:
      raise RuntimeError('After reset first timestep should be FIRST.')
    if main == StepType.FIRST:
      st.since_first = 0
      return True
    if main == StepType.LAST:
      st.since_first = None
      st.should_reset = True
      return True
    st.since_first += 1
    return st.since_first % self._repeats == 0

  def _reduce_scalars(self, st):
    """none_to_zero_pad + reduce_step_type + aggregate_rewards/discounts (processors.py:54-66, 267-365, 464-481)."""
    # padding slots: np.zeros_like(None) in the reference is an object-dtype zero, not None — so only a real FIRST
    # timestep (reward/discount None) makes the aggregate None
    slots = [(0, 0.0, 0.0) if v is None else v for v in st.slots]
    out_type = StepType.MID
    for v in slots:
      if v[0] == 0:
        out_type = StepType.FIRST
        break
      if v[0] == StepType.LAST:
        out_type = StepType.LAST
        break
      if v[0] != StepType.MID:
        raise ValueError('Expected MID if not FIRST or LAST.')
    rewards = [v[1] for v in slots]
    if any(r is None for r in rewards):
      reward = None
    else:
      reward = sum(rewards)
      if self._clip:
        reward = max(min(reward, self._clip), -self._clip)
    discounts = [v[2] for v in slots]
    if any(d is None for d in discounts):
      discount = None
    else:
      discount = 1
      for d in discounts:
        discount *= d
      discount = self._gamma * discount
    return out_type, reward, discount

  def _launch(self, emit):
    n = len(emit)
    if self._meta_pending:                      # the previous tick's async H2D copy still owns the pinned buffer
      self._meta_done.synchronize()
    meta = self._meta_host
    for i, e in enumerate(emit):
      st = self._streams[e]
      a_ok = st.has_frame[self._repeats - 2] and st.slots[self._repeats - 2] is not None
      b_ok = st.has_frame[self._repeats - 1] and st.slots[self._repeats - 1] is not None
      meta[0, i] = self._raw[e, 0].data_ptr() if a_ok else 0
      meta[1, i] = self._raw[e, 1].data_ptr() if b_ok else 0
      meta[2, i] = self._stacks[e].data_ptr()
      meta[3, i] = st.count
      st.count = min(st.count + 1, self._stack)
    self._meta.copy_(meta, non_blocking=True)
    self._meta_done.record()
    self._meta_pending = True
    self._counts[:n].copy_(self._meta[3, :n])
    _lib.call('dz_atari_preprocess', self._meta[0].data_ptr(), self._meta[1].data_ptr(), n, C.byref(self._axis_h.c),
              C.byref(self._axis_v.c), self._meta[2].data_ptr(), self._counts.data_ptr(), self._stack,
              C.cast(self._luma, C.c_void_p), self._max_band_rows, torch.cuda.current_stream().cuda_stream)


class VectorScalars:
  """The scalar half of `processors.atari()` for n streams as numpy array code (no per-stream Python objects): exactly the
  state machine of `BatchedAtariPreprocessor.step()` — ZeroDiscountOnLifeLoss (processors.py:254-260), FixedPaddedBuffer
  (:121-163), TimestepBufferCondition (:165-215), none_to_zero_pad + reduce_step_type + reward/discount aggregation
  (:54-66, 267-365, 464-481) — with `None` rewards / discounts carried as masks.  Pure host code: tested on CPU against the
  per-stream implementation and the oracle (tests/test_oracle_processors.py)."""

  FIRST, MID, LAST = int(StepType.FIRST), int(StepType.MID), int(StepType.LAST)

  def __init__(self, n, repeats, gamma, clip, life_loss, stack):
    self.n, self.R, self.gamma, self.clip, self.life_loss, self.stack = n, repeats, gamma, clip, life_loss, stack
    self.reset()

  def reset(self, streams=None):
    n, R = self.n, self.R
    if streams is None:
      self.lives = np.zeros(n, np.int64); self.has_lives = np.zeros(n, bool)
      self.index = np.full(n, (-1) % R, np.int64)
      self.valid = np.zeros((n, R), bool); self.type = np.zeros((n, R), np.int64)
      self.reward = np.zeros((n, R)); self.reward_none = np.zeros((n, R), bool)
      self.disc = np.zeros((n, R)); self.disc_none = np.zeros((n, R), bool)
      self.has_frame = np.zeros((n, R), bool)
      self.since = np.zeros(n, np.int64); self.since_none = np.ones(n, bool)
      self.should_reset = np.zeros(n, bool)
      self.count = np.zeros(n, np.int64)
      return
    e = np.asarray(streams)
    self.has_lives[e] = False; self.index[e] = (-1) % R
    self.valid[e] = False; self.has_frame[e] = False
    self.since_none[e] = True; self.should_reset[e] = False; self.count[e] = 0

  def tick(self, step_type, reward, discount, lives, active=None):
    """One raw timestep per active stream.  reward / discount: float64 arrays, NaN = None.  Returns a dict:
    emit (bool [n]), pooled_slot (int [n]; >= 0: this tick's frame goes to that pooled slot), and for emitting streams
    step_type, reward, discount (NaN = None), a_ok / b_ok (pooled frames present), count (stack fill before the push)."""
    n, R = self.n, self.R
    act = np.ones(n, bool) if active is None else np.asarray(active, bool)
    st = np.asarray(step_type, np.int64)
    rw = np.asarray(reward, np.float64).copy(); rn = np.isnan(rw)
    dc = np.asarray(discount, np.float64).copy(); dn = np.isnan(dc)
    lv = np.asarray(lives, np.int64)
    if self.life_loss:
      lost = act & (st == self.MID) & self.has_lives & (lv < self.lives)
      self.lives = np.where(act, lv, self.lives); self.has_lives |= act
      dc[lost] = 0.0; dn[lost] = False
    wrap = act & (self.index >= R)
    self.index[wrap] = 0; self.valid[wrap] = False; self.has_frame[wrap] = False
    rows = np.nonzero(act)[0]; col = self.index[rows]
    self.valid[rows, col] = True; self.type[rows, col] = st[rows]
    self.reward[rows, col] = np.where(rn[rows], 0.0, rw[rows]); self.reward_none[rows, col] = rn[rows]
    self.disc[rows, col] = np.where(dn[rows], 0.0, dc[rows]); self.disc_none[rows, col] = dn[rows]
    pooled = np.where(act, self.index - (R - 2), -1)
    up = rows[pooled[rows] >= 0]
    self.has_frame[up, self.index[up]] = True
    self.index[rows] += 1
    # ---- TimestepBufferCondition
    if np.any(act & self.should_reset):
      raise RuntimeError('Should have reset.')
    boundary = self.valid & ((self.type == self.FIRST) | (self.type == self.LAST))
    nb = boundary.sum(axis=1)
    if np.any(act & (nb > 1)):
      raise RuntimeError('Expected at most one FIRST or LAST.')
    main = np.where(nb == 1, (self.type * boundary).sum(axis=1), self.MID)   # FIRST = 0: a lone FIRST sums to 0
    is_first = act & (nb == 1) & (boundary & (self.type == self.FIRST)).any(axis=1)
    is_last = act & (nb == 1) & ~is_first
    del main
    if np.any(act & self.since_none & ~is_first):
      raise RuntimeError('After reset first timestep should be FIRST.')
    mid = act & ~is_first & ~is_last
    self.since[is_first] = 0; self.since_none[is_first] = False
    self.since_none[is_last] = True; self.should_reset[is_last] = True
    self.since[mid] += 1
    emit = is_first | is_last | (mid & (self.since % R == 0))
    # ---- reduce (none_to_zero_pad: padding slots count as type 0 = FIRST, reward 0.0, discount 0.0)
    t = np.where(self.valid, self.type, 0)
    if np.any(emit[:, None] & ~np.isin(t, (self.FIRST, self.MID, self.LAST))):
      raise ValueError('Expected MID if not FIRST or LAST.')
    edge = (t == 0) | (t == self.LAST)
    first_edge = np.argmax(edge, axis=1)
    out_type = np.where(edge.any(axis=1), t[np.arange(n), first_edge], self.MID)
    r_none = (self.valid & self.reward_none).any(axis=1)
    r = np.zeros(n)
    for j in range(R):
      r = r + np.where(self.valid[:, j], self.reward[:, j], 0.0)       # python's sum(): left to right from 0
    if self.clip:
      r = np.maximum(np.minimum(r, self.clip), -self.clip)
    d_none = (self.valid & self.disc_none).any(axis=1)
    d = np.ones(n)
    for j in range(R):
      d = d * np.where(self.valid[:, j], self.disc[:, j], 0.0)
    d = self.gamma * d
    a_ok = self.has_frame[:, R - 2] & self.valid[:, R - 2]
    b_ok = self.has_frame[:, R - 1] & self.valid[:, R - 1]
    count = self.count.copy()
    self.count = np.where(emit, np.minimum(self.count + 1, self.stack), self.count)
    return {'emit': emit, 'pooled_slot': pooled, 'step_type': out_type, 'reward': np.where(r_none, np.nan, r),
            'discount': np.where(d_none, np.nan, d), 'a_ok': a_ok, 'b_ok': b_ok, 'count': count}


class VectorizedAtariPreprocessor(BatchedAtariPreprocessor):
  """`processors.atari()` for many environment streams whose raw frames are ALREADY on the device (a GPU emulator, or one
  staged H2D copy of all streams' frames per tick): `step_arrays()` takes struct-of-arrays timesteps, runs the scalar state
  machine as numpy array code (`VectorScalars`; no per-stream Python objects) and the pixel kernel once per tick.  Emits
  arrays, not TimeStep objects; the frame stacks stay in `self.stacks` for `Learner.act_batch` / the replay insert."""

  def __init__(self, num_streams: int = 1, **kwargs):
    super().__init__(num_streams=num_streams, **kwargs)
    self._vs = VectorScalars(num_streams, self._repeats, self._gamma, self._clip, self._life_loss, self._stack)
    self._all = torch.arange(num_streams)

  def reset(self, stream: Optional[int] = None) -> None:
    self._vs.reset(None if stream is None else [stream])
    if self._in_shape is not None:
      (self._stacks if stream is None else self._stacks[stream]).zero_()

  def get_state(self) -> Mapping[str, Any]:
    """The scalar state machine's arrays and, once frames have arrived, the device frame stacks and the two pooled raw
    frames of every stream, copied to the host."""
    state = {'scalars': {k: v.copy() for k, v in vars(self._vs).items() if isinstance(v, np.ndarray)},
             'in_shape': self._in_shape}
    if self._in_shape is not None:
      state['stacks'] = self._stacks.cpu().numpy()
      state['raw'] = self._raw.cpu().numpy()
    return state

  def set_state(self, state: Mapping[str, Any]) -> None:
    """Restores `get_state()` of a preprocessor with the same options and stream count."""
    scalars = state['scalars']
    if scalars['index'].shape != (self._n,):
      raise ValueError('state is for %d streams, this preprocessor has %d' % (scalars['index'].shape[0], self._n))
    for k, v in scalars.items():
      setattr(self._vs, k, np.array(v, copy=True))
    if state['in_shape'] is None:
      return
    shape = tuple(state['in_shape'])
    if self._in_shape is None:
      self._allocate(shape)
    elif self._in_shape != shape:
      raise ValueError('frame shape of the state %s != %s' % (shape, self._in_shape))
    self._stacks.copy_(torch.as_tensor(state['stacks']))
    self._raw.copy_(torch.as_tensor(state['raw']))

  def step_arrays(self, frames, step_type, reward, discount, lives, active=None):
    """frames: uint8 [n, H, W, 3] (device tensor, or a host array -> one H2D copy); step_type int [n]; reward / discount
    float [n] with NaN for None (FIRST timesteps); lives int [n].  Returns VectorScalars.tick()'s dict (host arrays)."""
    if self._in_shape is None:
      self._allocate(tuple(frames.shape[1:]))
    frames = torch.as_tensor(frames, device=self._device)
    out = self._vs.tick(step_type, reward, discount, lives, active)
    for slot in (0, 1):
      e = np.nonzero(out['pooled_slot'] == slot)[0]
      if e.size == self._n:
        self._raw[:, slot].copy_(frames, non_blocking=True)
      elif e.size:
        idx = torch.as_tensor(e, device=self._device)
        self._raw[:, slot].index_copy_(0, idx, frames.index_select(0, idx))
    emit = np.nonzero(out['emit'])[0]
    if emit.size:
      k = emit.size
      if self._meta_pending:
        self._meta_done.synchronize()
      raw0, stride_e = self._raw.data_ptr(), self._raw.stride(0)
      slot_bytes = self._raw.stride(1)
      meta = self._meta_host.numpy()
      meta[0, :k] = np.where(out['a_ok'][emit], raw0 + emit * stride_e, 0)
      meta[1, :k] = np.where(out['b_ok'][emit], raw0 + emit * stride_e + slot_bytes, 0)
      meta[2, :k] = self._stacks.data_ptr() + emit * self._stacks.stride(0)
      meta[3, :k] = out['count'][emit]
      self._meta.copy_(self._meta_host, non_blocking=True)
      self._meta_done.record()
      self._meta_pending = True
      self._counts[:k].copy_(self._meta[3, :k])
      _lib.call('dz_atari_preprocess', self._meta[0].data_ptr(), self._meta[1].data_ptr(), int(k), C.byref(self._axis_h.c),
                C.byref(self._axis_v.c), self._meta[2].data_ptr(), self._counts.data_ptr(), self._stack,
                C.cast(self._luma, C.c_void_p), self._max_band_rows, torch.cuda.current_stream().cuda_stream)
    return out


class _SingleStream:
  """The reference's per-environment processor object: `__call__(timestep)` and `reset()`."""

  def __init__(self, **kwargs):
    self._batched = BatchedAtariPreprocessor(num_streams=1, **kwargs)

  def reset(self) -> None:
    self._batched.reset()

  def __call__(self, timestep):
    return self._batched.step([timestep])[0]

  @property
  def stack(self) -> torch.Tensor:
    return self._batched.stacks[0]


def atari(additional_discount: float = 0.99, max_abs_reward: Optional[float] = 1.0,
          resize_shape: Optional[Tuple[int, int]] = (84, 84), num_action_repeats: int = 4, num_pooled_frames: int = 2,
          zero_discount_on_life_loss: bool = True, num_stacked_frames: int = 4, grayscaling: bool = True,
          device: Any = 'cuda', device_observations: bool = False):
  """Standard DQN preprocessing on Atari (processors.py:399-505), pixel path on the GPU.

  Timesteps carry `observation = (rgb uint8 [H, W, 3], lives)` exactly as the reference's environment emits them
  (the processor selects the RGB entry itself, processors.py:391-393)."""
  return _SingleStream(additional_discount=additional_discount, max_abs_reward=max_abs_reward, resize_shape=resize_shape,
                       num_action_repeats=num_action_repeats, num_pooled_frames=num_pooled_frames,
                       zero_discount_on_life_loss=zero_discount_on_life_loss, num_stacked_frames=num_stacked_frames,
                       grayscaling=grayscaling, device=device, device_observations=device_observations)
