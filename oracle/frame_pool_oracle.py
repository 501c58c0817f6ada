"""CPU model of the frame-deduplicated replay layout (`TransitionReplay(..., frame_dedup=True)`, csrc/dz_frames.cu).

TEST INFRASTRUCTURE ONLY.  The reference stores whole transitions and has no frame pool, so this is not a port: it
restates the pool rules with a dict from plane bytes to plane id, so that tests can predict the exact device plane
table, refcounts and `frames_in_use`:

  * an observation [H, W, C] uint8 is C planes of H*W bytes; a transition has 2*C plane ids (s_tm1 channels 0..C-1,
    then s_t channels 0..C-1), resolved in that order, each seeing the planes resolved before it;
  * a plane resolves to the live plane with identical bytes, else to a fresh plane popped from a LIFO free stack that
    initially hands out 1, 2, 3, ...; with the stack empty the plane maps to plane 0 and `full` is set;
  * plane 0 is the all-zero plane: always live, never freed, refcount = 1 + its references;
  * the new row's planes are referenced before the evicted row's references are released; a plane whose refcount
    drops to 0 is pushed back onto the free stack.

Also `synthetic_stacked_rows`, the bytes of `dz_replay_fill_synthetic_stacked`.
"""

from __future__ import annotations

import numpy as np

from oracle import replay_oracle


class FramePool:
  """Plane table of `capacity` rows over a pool of `frame_capacity` planes."""

  def __init__(self, capacity, obs_shape, frame_capacity):
    h, w, c = obs_shape
    self.capacity, self.obs_shape, self.channels, self.frame_capacity = capacity, tuple(obs_shape), c, frame_capacity
    self.frame_bytes = h * w
    self.reset()

  def reset(self):
    self.free = list(range(self.frame_capacity - 1, 0, -1))   # free.pop() hands out 1 first
    self.refcount = np.zeros(self.frame_capacity, dtype=np.int64)
    self.refcount[0] = 1
    zero = bytes(self.frame_bytes)
    self.by_bytes = {zero: 0}
    self.bytes_of = {0: zero}
    self.planes = np.zeros((self.capacity, 2 * self.channels), dtype=np.int64)
    self.full = False

  def _resolve(self, key):
    pid = self.by_bytes.get(key)
    if pid is None:
      if not self.free:
        self.full = True
        pid = 0
      else:
        pid = self.free.pop()
        self.by_bytes[key] = pid
        self.bytes_of[pid] = key
    self.refcount[pid] += 1
    return pid

  def add(self, slot, s_tm1, s_t, release_row):
    """One add into row `slot`; `release_row`: the row holds a live transition (it is being evicted)."""
    ids = []
    for obs in (s_tm1, s_t):
      obs = np.asarray(obs, dtype=np.uint8).reshape(self.obs_shape)
      for c in range(self.channels):
        ids.append(self._resolve(np.ascontiguousarray(obs[:, :, c]).tobytes()))
    old = self.planes[slot].copy()
    self.planes[slot] = ids
    if release_row:
      for pid in old:
        self.refcount[pid] -= 1
        if self.refcount[pid] == 0:
          del self.by_bytes[self.bytes_of.pop(pid)]
          self.free.append(pid)

  def reconstruct(self, slot):
    """(s_tm1, s_t) of row `slot` as [H, W, C] uint8 arrays."""
    h, w, c = self.obs_shape
    out = []
    for o in range(2):
      planes = [np.frombuffer(self.bytes_of[pid], dtype=np.uint8).reshape(h, w)
                for pid in self.planes[slot, o * c:(o + 1) * c]]
      out.append(np.stack(planes, axis=-1))
    return out[0], out[1]

  @property
  def frames_in_use(self):
    return self.frame_capacity - len(self.free)

  def live_planes(self):
    return sorted(self.bytes_of)


class DedupReplayModel:
  """The plane bookkeeping of a replay with oldest-out eviction: add k goes to row k % capacity and, once the ring is
  full, evicts the row's previous transition (both replay classes store transitions this way)."""

  def __init__(self, capacity, obs_shape, frame_capacity):
    self.pool = FramePool(capacity, obs_shape, frame_capacity)
    self.t = 0

  def add(self, s_tm1, s_t):
    cap = self.pool.capacity
    self.pool.add(self.t % cap, s_tm1, s_t, release_row=self.t >= cap)
    self.t += 1

  def live_slots(self):
    cap = self.pool.capacity
    return np.arange(max(0, self.t - cap), self.t, dtype=np.int64) % cap


def stacked_frame(seed, episode, frame, episode_len, frame_bytes):
  """Bytes of frame `frame` of synthetic episode `episode`: 8-byte word w is
  mix64(seed*0x9E3779B97F4A7C15 + 0x632BE59BD9B4E019 + (episode*(episode_len+1) + frame)*(frame_bytes/8) + w)."""
  words = frame_bytes // 8
  with np.errstate(over='ignore'):
    base = np.uint64(seed) * np.uint64(0x9E3779B97F4A7C15) + np.uint64(0x632BE59BD9B4E019)
    ctr = base + np.uint64(episode * (episode_len + 1) + frame) * np.uint64(words) + np.arange(words, dtype=np.uint64)
  return replay_oracle._mix64(ctr).view(np.uint8)


def stack_at(seed, episode, step, episode_len, obs_shape):
  """The [H, W, C] stack after frames 0..step of an episode, trailing-zero padded while step + 1 < C
  (A000, AB00, ABC0, ABCD, BCDE, ...; processors.py)."""
  h, w, c = obs_shape
  out = np.zeros((h, w, c), dtype=np.uint8)
  for ch in range(c):
    f = (ch if ch <= step else -1) if step + 1 < c else step - (c - 1) + ch
    if f >= 0:
      out[:, :, ch] = stacked_frame(seed, episode, f, episode_len, h * w).reshape(h, w)
  return out


def synthetic_stacked_rows(seed, rows, obs_shape, episode_len, num_actions, discount=0.99):
  """Contents of rows `rows` after `dz_replay_fill_synthetic_stacked`: transition i is step t = i % episode_len of
  episode e = i // episode_len, s_tm1 = stack after frames 0..t, s_t = stack after frames 0..t+1; the scalars are
  those of `replay_oracle.synthetic_rows`.  Returns (obs uint8 [n, 2, H*W*C], a, r, d)."""
  rows = np.asarray(rows, dtype=np.int64)
  obs = np.zeros((len(rows), 2, int(np.prod(obs_shape))), dtype=np.uint8)
  for k, i in enumerate(rows):
    e, t = divmod(int(i), episode_len)
    obs[k, 0] = stack_at(seed, e, t, episode_len, obs_shape).reshape(-1)
    obs[k, 1] = stack_at(seed, e, t + 1, episode_len, obs_shape).reshape(-1)
  _, a, r, d = replay_oracle.synthetic_rows(seed, rows, 8, num_actions, discount)
  return obs, a, r, d


class _TimeStep:
  """Minimal dm_env.TimeStep stand-in (FIRST=0, MID=1, LAST=2) for the accumulators."""

  def __init__(self, step_type, reward, discount, observation):
    self.step_type, self.reward, self.discount, self.observation = step_type, reward, discount, observation

  def first(self):
    return self.step_type == 0

  def mid(self):
    return self.step_type == 1

  def last(self):
    return self.step_type == 2


def stacked_episode(rs, length, obs_shape, static=False):
  """Timesteps of one episode of `length` transitions whose observations are frame stacks as `processors.atari()`
  builds them (trailing-zero padded at the start); `static`: every frame is the same screen."""
  h, w, c = obs_shape
  frames = rs.randint(0, 256, size=(length + 1, h, w)).astype(np.uint8)
  if static:
    frames[:] = frames[0]
  stack = np.zeros((h, w, c), dtype=np.uint8)
  out = []
  for t in range(length + 1):
    if t < c:
      stack[:, :, t] = frames[t]
    else:
      stack = np.concatenate([stack[:, :, 1:], frames[t][:, :, None]], axis=-1)
    kind = 0 if t == 0 else (2 if t == length else 1)
    out.append(_TimeStep(kind, None if t == 0 else float(rs.randint(-1, 2)), None if t == 0 else 0.99, stack.copy()))
  return out


def interleave_episodes(rs, accumulators, episodes):
  """Round-robin over actor streams: stream k plays `episodes[k]` (a list of timestep lists) through
  `accumulators[k]`; returns the transitions in the order they would be added, with the action of each step drawn
  from `rs`."""
  cursors = [[ts for ep in eps for ts in ep] for eps in episodes]
  pos = [0] * len(cursors)
  out = []
  while any(p < len(c) for p, c in zip(pos, cursors)):
    for k, c in enumerate(cursors):
      if pos[k] < len(c):
        out.extend(accumulators[k].step(c[pos[k]], int(rs.randint(0, 6))))
        pos[k] += 1
  return out
