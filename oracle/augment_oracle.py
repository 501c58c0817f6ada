"""CPU definition of the learner's random-shift augmentation (DrQ: Kostrikov, Yarats & Fergus, ICLR 2021; DESIGN.md
§18).  TEST INFRASTRUCTURE ONLY (imported by tests/).

Pad p is an integer in [0, 16], less than min(H, W); p = 0 is off.  Each sampled example b gets two independent shifts,
(dy0, dx0) for s_tm1 and (dy1, dx1) for s_t, each component uniform on {0, ..., 2p}.  An observation [H][W][C] uint8
becomes

    out[y][x][c] = in[clamp(y + dy - p, 0, H - 1)][clamp(x + dx - p, 0, W - 1)][c]

i.e. edge ("replicate") padding by p followed by an H x W crop at offset (dy, dx); one shift moves all C stacked
channels of an observation together.

The draws come from the learner's Philox generator (oracle/philox_oracle.py) at its current counter on stream id 3:
example b takes the block at counter (b, 0, ctr low, ctr high ^ (3 << 24)), key = seed, and its four words w give
(dy0, dx0, dy1, dx1) in that order as floor(w * (2p + 1) / 2^32).  That is `philox_oracle.words(4 B, seed, ctr, 3)`
reshaped to [B][4]."""

import numpy as np

from oracle import philox_oracle

STREAM_SHIFTS = 3
MAX_PAD = 16


def check_pad(pad, H, W):
  """ValueError unless pad is an integer in [0, 16] and less than min(H, W)."""
  if isinstance(pad, (bool, np.bool_)) or int(pad) != pad:
    raise ValueError('random_shift_pad must be an integer, got %r' % (pad,))
  pad = int(pad)
  if pad < 0 or pad > MAX_PAD:
    raise ValueError('random_shift_pad must be in [0, %d], got %d' % (MAX_PAD, pad))
  if pad >= min(H, W):
    raise ValueError('random_shift_pad must be less than min(H, W) = %d, got %d' % (min(H, W), pad))
  return pad


def shift_one(obs, dy, dx, pad):
  """One observation [H, W, C] (or [H, W]) shifted by (dy, dx) with edge padding `pad`."""
  obs = np.asarray(obs)
  H, W = obs.shape[:2]
  ys = np.clip(np.arange(H) + int(dy) - pad, 0, H - 1)
  xs = np.clip(np.arange(W) + int(dx) - pad, 0, W - 1)
  return obs[ys][:, xs]


def shift(obs, shifts, pad, which):
  """A batch [B, H, W, C] shifted example by example: `which` 0 takes (dy0, dx0) of `shifts` [B, 4] (s_tm1), 1 takes
  (dy1, dx1) (s_t)."""
  obs = np.asarray(obs)
  shifts = np.asarray(shifts).reshape(-1, 4)
  assert obs.shape[0] == shifts.shape[0], (obs.shape, shifts.shape)
  return np.stack([shift_one(obs[b], shifts[b, 2 * which], shifts[b, 2 * which + 1], pad) for b in range(obs.shape[0])])


def shift_batch(s_tm1, s_t, shifts, pad):
  """(shifted s_tm1, shifted s_t): what the learner's passes read for the batch (s_tm1, s_t)."""
  return shift(s_tm1, shifts, pad, 0), shift(s_t, shifts, pad, 1)


def draws(B, seed, ctr, pad):
  """int32 [B, 4]: (dy0, dx0, dy1, dx1) of each example, bit for bit what the device draws."""
  w = philox_oracle.words(4 * B, seed, ctr, STREAM_SHIFTS).astype(np.uint64).reshape(B, 4)
  return ((w * np.uint64(2 * pad + 1)) >> np.uint64(32)).astype(np.int32)
