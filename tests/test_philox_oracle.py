"""CPU: the numpy Philox4x32-10 of oracle/philox_oracle.py against the Random123 known-answer vectors, and the
restated counter layout / output transforms of the device generator (tests/test_gpu_randomness.py compares the device
with them)."""

import numpy as np
import pytest
import scipy.special
import scipy.stats

from oracle import philox_oracle as po

# Random123 kat_vectors, philox4x32 10: counter, key -> output
KATS = [((0x0, 0x0, 0x0, 0x0), (0x0, 0x0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
        ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
        ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
         (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]


def _scalar_philox(counter, key):
  """The same ten rounds over Python integers: shares no arithmetic with the vectorised uint64 version."""
  c, k = list(counter), list(key)
  for _ in range(10):
    p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
    c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k[1], p0 & 0xFFFFFFFF]
    k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
  return tuple(c)


@pytest.mark.parametrize('counter,key,want', KATS)
def test_philox_known_answers(counter, key, want):
  assert tuple(int(w) for w in po.philox4x32_10(counter, key)) == want
  assert _scalar_philox(counter, key) == want


def test_vectorised_blocks_equal_scalar_blocks():
  rs = np.random.RandomState(0)
  ctr = rs.randint(0, 2 ** 32, size=(64, 4), dtype=np.uint64)
  key = (0x12345678, 0x9abcdef0)
  got = po.philox4x32_10(tuple(ctr[:, j] for j in range(4)), key)
  assert got.shape == (64, 4) and got.dtype == np.uint32
  for i in range(64):
    assert tuple(int(w) for w in got[i]) == _scalar_philox([int(x) for x in ctr[i]], key)


@pytest.mark.parametrize('seed,ctr', [(0, 0), (7, 3), (2 ** 32 + 5, 1), (11, 2 ** 32 + 9), (2 ** 63 + 1, 2 ** 40)])
def test_counter_layout(seed, ctr):
  """Element 4 * i4 + j is word j of the block (i4 low, i4 high, ctr low, ctr high ^ stream << 24) under the key (seed
  low, seed high); a length that is not a multiple of 4 is a prefix of the next multiple."""
  n = 4 * 5 + 3
  for stream in (po.STREAM_TAUS, po.STREAM_NOISE):
    w = po.words(n, seed, ctr, stream)
    assert w.shape == (n,)
    np.testing.assert_array_equal(w, po.words(n + 1, seed, ctr, stream)[:n])
    for i4 in (0, 3, 5):
      block = _scalar_philox([i4, 0, ctr & 0xFFFFFFFF, (ctr >> 32) ^ (stream << 24)], [seed & 0xFFFFFFFF, seed >> 32])
      for j in range(4):
        if 4 * i4 + j < n:
          assert int(w[4 * i4 + j]) == block[j]
  assert np.any(po.words(n, seed, ctr, 1) != po.words(n, seed, ctr, 2))
  assert np.any(po.words(n, seed, ctr, 1) != po.words(n, seed, ctr + 1, 1))
  assert np.any(po.words(n, seed, ctr, 1) != po.words(n, seed + 1, ctr, 1))


def test_distribution_bars_tell_a_truncated_normal_from_a_clipped_one():
  """The bars tests/test_gpu_randomness.py puts on the device's draws pass on the oracle's own draws and on scipy's
  truncated normal, and fail on a clipped normal, an untruncated one and a uniform on [-2, 2]."""
  n = 1 << 20
  tn = scipy.stats.truncnorm(-2, 2)
  assert abs(tn.var() - po.TRUNCNORM_VAR) < 1e-12
  assert np.sqrt(tn.moment(4) - tn.var() ** 2) < 1.1
  rs = np.random.RandomState(1)
  assert po.truncnorm_report_ok(po.truncnorm_report(po.truncated_normal(n, 9, 4)), n)
  assert po.truncnorm_report_ok(po.truncnorm_report(tn.rvs(n, random_state=rs)), n)
  clipped = po.truncnorm_report(np.clip(rs.standard_normal(n), -2, 2))
  assert not po.truncnorm_report_ok(clipped, n) and clipped['at_bound'] > 0.04 and clipped['ks'] > 0.02
  assert not po.truncnorm_report_ok(po.truncnorm_report(rs.standard_normal(n)), n)
  assert not po.truncnorm_report_ok(po.truncnorm_report(rs.uniform(-2, 2, n)), n)


def test_output_transforms():
  n = 1 << 16
  t = po.taus(n, 5, 2)
  assert t.dtype == np.float32 and t.min() >= 0.0 and t.max() < 1.0
  np.testing.assert_array_equal(t.astype(np.float64) * 2 ** 24, po.words(n, 5, 2, po.STREAM_TAUS) >> np.uint32(8))
  x = po.truncated_normal(n, 5, 2)
  assert np.abs(x).max() < 2.0
  # the inversion is the truncated normal's quantile function at the cell midpoints
  u = ((po.words(n, 5, 2, po.STREAM_NOISE) >> np.uint32(8)).astype(np.float64) + 0.5) * 2.0 ** -24
  np.testing.assert_allclose(x, scipy.stats.truncnorm(-2, 2).ppf(u), rtol=0, atol=1e-9)
  g = po.noise(n, 5, 2)
  np.testing.assert_allclose(np.sign(g) * g * g, x, rtol=1e-14, atol=0)
  assert np.abs(g).max() < np.sqrt(2.0)
  assert abs(x.var() - scipy.stats.truncnorm(-2, 2).var()) < 0.02 and abs(x.mean()) < 0.02
