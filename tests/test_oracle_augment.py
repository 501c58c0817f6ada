"""CPU: the random-shift augmentation's definition (oracle/augment_oracle.py, DESIGN.md §18) against hand-built
arrays, and its draw mapping against the Philox restatement."""

import numpy as np
import pytest

from oracle import augment_oracle as ao
from oracle import philox_oracle


def _ramp(H, W, C):
  """An observation whose every byte names its position: (y * 7 + x * 3 + c * 50) mod 256."""
  y, x, c = np.meshgrid(np.arange(H), np.arange(W), np.arange(C), indexing='ij')
  return ((y * 7 + x * 3 + c * 50) % 256).astype(np.uint8)


@pytest.mark.parametrize('H,W', [(84, 84), (84, 92), (84, 88), (44, 44)])
@pytest.mark.parametrize('C', [1, 4])
@pytest.mark.parametrize('p', [1, 4, 16])
def test_extreme_shifts_replicate_corners_and_edges(H, W, C, p):
  obs = _ramp(H, W, C)
  # (p, p) is the identity
  assert np.array_equal(ao.shift_one(obs, p, p, p), obs)
  for dy in (0, 2 * p):
    for dx in (0, 2 * p):
      out = ao.shift_one(obs, dy, dx, p)
      assert out.shape == obs.shape and out.dtype == np.uint8
      # the corner the image moved away from is replicated over a (p + 1) x (p + 1) block
      cy = 0 if dy == 0 else H - 1
      cx = 0 if dx == 0 else W - 1
      ys = slice(0, p + 1) if dy == 0 else slice(H - p - 1, H)
      xs = slice(0, p + 1) if dx == 0 else slice(W - p - 1, W)
      assert np.array_equal(out[ys, xs], np.broadcast_to(obs[cy, cx], out[ys, xs].shape))
      # the edge rows / columns replicate the input's edge, and the rest is the input moved by (dy - p, dx - p)
      sy, sx = dy - p, dx - p
      for y in range(H):
        for x in (0, W // 2, W - 1):
          assert np.array_equal(out[y, x], obs[min(max(y + sy, 0), H - 1), min(max(x + sx, 0), W - 1)])
      inner = out[max(-sy, 0):H - max(sy, 0), max(-sx, 0):W - max(sx, 0)]
      assert np.array_equal(inner, obs[max(sy, 0):H + min(sy, 0), max(sx, 0):W + min(sx, 0)])


def test_one_shift_moves_every_channel_together():
  obs = _ramp(84, 84, 4)
  out = ao.shift_one(obs, 1, 7, 4)
  for c in range(4):
    assert np.array_equal(out[..., c], ao.shift_one(obs[..., c], 1, 7, 4))


@pytest.mark.parametrize('H,W', [(84, 84), (84, 92)])
def test_a_shift_then_its_opposite_is_the_identity_on_the_interior(H, W):
  p = 4
  rs = np.random.RandomState(0)
  obs = rs.randint(0, 256, size=(H, W, 4)).astype(np.uint8)
  for dy, dx in [(0, 8), (3, 5), (8, 0), (2, 2)]:
    back = ao.shift_one(ao.shift_one(obs, dy, dx, p), 2 * p - dy, 2 * p - dx, p)
    # rows / columns that the clamps never touched on either pass
    assert np.array_equal(back[p:H - p, p:W - p], obs[p:H - p, p:W - p])


def test_batch_shift_takes_each_examples_own_pair():
  rs = np.random.RandomState(1)
  s_tm1 = rs.randint(0, 256, size=(3, 44, 44, 4)).astype(np.uint8)
  s_t = rs.randint(0, 256, size=(3, 44, 44, 4)).astype(np.uint8)
  shifts = np.array([[0, 8, 4, 4], [8, 0, 1, 7], [2, 3, 8, 8]], np.int32)
  a, b = ao.shift_batch(s_tm1, s_t, shifts, 4)
  for i in range(3):
    assert np.array_equal(a[i], ao.shift_one(s_tm1[i], shifts[i, 0], shifts[i, 1], 4))
    assert np.array_equal(b[i], ao.shift_one(s_t[i], shifts[i, 2], shifts[i, 3], 4))


@pytest.mark.parametrize('seed', [0, 7, 2 ** 32 - 1, 2 ** 32, 2 ** 63 + 12345])
@pytest.mark.parametrize('ctr', [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 40 + 3])
@pytest.mark.parametrize('p', [1, 4, 16])
def test_draws_are_the_philox_words_scaled_to_the_shift_range(seed, ctr, p):
  B = 33
  d = ao.draws(B, seed, ctr, p)
  w = philox_oracle.words(4 * B, seed, ctr, ao.STREAM_SHIFTS).reshape(B, 4)
  assert d.dtype == np.int32 and d.shape == (B, 4)
  want = np.array([[int(v) * (2 * p + 1) >> 32 for v in row] for row in w], np.int32)
  assert np.array_equal(d, want)
  assert d.min() >= 0 and d.max() <= 2 * p
  # example b is the Philox block at counter (b, 0, ctr low, ctr high ^ (3 << 24))
  blk = philox_oracle.philox4x32_10((np.arange(B), 0, ctr & 0xFFFFFFFF, ((ctr >> 32) ^ (3 << 24)) & 0xFFFFFFFF),
                                    (seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF))
  assert np.array_equal(blk, w)


def test_draws_use_a_stream_of_their_own():
  w3 = philox_oracle.words(64, 5, 9, 3)
  assert not np.array_equal(w3, philox_oracle.words(64, 5, 9, philox_oracle.STREAM_TAUS))
  assert not np.array_equal(w3, philox_oracle.words(64, 5, 9, philox_oracle.STREAM_NOISE))


@pytest.mark.parametrize('pad,H,W', [(-1, 84, 84), (17, 84, 84), (84, 84, 84), (44, 84, 44), (1.5, 84, 84), (True, 84, 84)])
def test_bad_pads_are_rejected(pad, H, W):
  with pytest.raises(ValueError):
    ao.check_pad(pad, H, W)


def test_good_pads_pass():
  assert ao.check_pad(0, 84, 84) == 0
  assert ao.check_pad(16, 84, 84) == 16
  assert ao.check_pad(4, 84, 92) == 4
  assert ao.check_pad(16, 17, 17) == 16
