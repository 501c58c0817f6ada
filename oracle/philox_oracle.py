"""CPU restatement of the learner's device generator (`randomness_kernel` in csrc/dz_learner.cu).
TEST INFRASTRUCTURE ONLY (imported by tests/).

Philox4x32-10 is written from its published definition (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy
as 1, 2, 3", SC'11; the Random123 round function): per round

    hi0, lo0 = mulhilo(0xD2511F53, c0);  hi1, lo1 = mulhilo(0xCD9E8D57, c2)
    (c0, c1, c2, c3) = (hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0)

with the key bumped by the Weyl constants (0x9E3779B9, 0xBB67AE85) between rounds, ten rounds.  It is pinned to the
three Random123 known-answer vectors in tests/test_philox_oracle.py.  Vectorised numpy over uint64 (products of two
32-bit words fit), so it shares no code with the product.

The kernel's use of it, restated from its comments and include/dqn_zoo_b200.h: one Philox block per four consecutive
output elements,

    counter = (i4 low, i4 high, ctr low, ctr high ^ (stream_id << 24)),   key = (seed low, seed high)

where i4 is the index of the quadruple, `ctr` the generator counter (d_counters[1]; a frozen actor's own), stream_id 1
for IQN's taus and 2 for rainbow's noise; element 4 * i4 + j comes from word j:

    tau   = (r >> 8) * 2^-24                                             in [0, 1)
    noise = sign(x) * sqrt|x|,  x = sqrt(2) * erfinv(lo + (-2 lo) * ((r >> 8) + 0.5) * 2^-24),  lo = erf(-sqrt 2)

i.e. x is the inverse-CDF draw of a standard normal truncated to [-2, 2] (networks.py:142-144), evaluated here in
float64 with scipy.special.erfinv."""

import numpy as np

M32 = np.uint64(0xFFFFFFFF)
MUL0, MUL1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
WEYL0, WEYL1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
STREAM_TAUS, STREAM_NOISE = 1, 2


def philox4x32_10(counter, key):
  """counter: four arrays (or ints) of 32-bit words, key: two.  Returns a uint32 array [..., 4]."""
  c0, c1, c2, c3 = np.broadcast_arrays(*[np.asarray(c, dtype=np.uint64) & M32 for c in counter])
  k0, k1 = (np.uint64(int(k) & 0xFFFFFFFF) for k in key)
  for _ in range(10):
    p0, p1 = MUL0 * c0, MUL1 * c2            # 32 x 32 -> 64 bits: exact in uint64
    c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
    k0, k1 = (k0 + WEYL0) & M32, (k1 + WEYL1) & M32
  return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def words(n, seed, ctr, stream_id):
  """The first n 32-bit words of the generator's output for (seed, counter, stream)."""
  seed, ctr = int(seed) & (2 ** 64 - 1), int(ctr) & (2 ** 64 - 1)
  i4 = np.arange((n + 3) // 4, dtype=np.uint64)
  out = philox4x32_10((i4 & M32, i4 >> np.uint64(32), ctr & 0xFFFFFFFF, (ctr >> 32) ^ ((stream_id << 24) & 0xFFFFFFFF)),
                      (seed & 0xFFFFFFFF, seed >> 32))
  return out.reshape(-1)[:n]


def taus(n, seed, ctr):
  """float32 [n], bit for bit what the device writes: a 24-bit integer times 2^-24 is exact in float32."""
  return ((words(n, seed, ctr, STREAM_TAUS) >> np.uint32(8)).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def truncated_normal(n, seed, ctr):
  """float64 [n]: x ~ Normal(0, 1) truncated to [-2, 2], by inversion at the midpoint of the 24-bit cell."""
  from scipy.special import erf, erfinv
  lo = erf(-np.sqrt(2.0))
  u = ((words(n, seed, ctr, STREAM_NOISE) >> np.uint32(8)).astype(np.float64) + 0.5) * 2.0 ** -24
  return np.sqrt(2.0) * erfinv(lo + (-2.0 * lo) * u)


def noise(n, seed, ctr):
  """float64 [n]: the factorised-noise transform sign(x) sqrt|x| of `truncated_normal`."""
  x = truncated_normal(n, seed, ctr)
  return np.sign(x) * np.sqrt(np.abs(x))


TRUNCNORM_VAR = 0.7737413035499232   # variance of Normal(0, 1) truncated to [-2, 2]


def truncnorm_report(x):
  """What tells a truncated normal from a clipped one (np.clip(normal, -2, 2) puts 2.3 % of its mass on each bound
  and has variance 0.92), for n >= 2^20 draws x: the Kolmogorov-Smirnov distance to truncnorm(-2, 2), mean, variance,
  the fraction sitting exactly on a bound and the fraction of positive draws."""
  import scipy.stats
  x = np.asarray(x, dtype=np.float64)
  return {'ks': float(scipy.stats.kstest(x, scipy.stats.truncnorm(-2, 2).cdf).statistic), 'mean': float(x.mean()),
          'var': float(x.var()), 'at_bound': float(np.mean(np.abs(x) >= 2.0)), 'positive': float(np.mean(x > 0))}


def truncnorm_report_ok(rep, n):
  """The bars on `truncnorm_report`: KS distance below 3e-3 (about three times the 1e-6 critical value at n = 2^20),
  mean and variance within five standard errors, fewer than 1e-5 of the draws on a bound, signs balanced to five
  standard errors."""
  se = 1.0 / np.sqrt(n)
  return (rep['ks'] < 3e-3 and abs(rep['mean']) < 5 * np.sqrt(TRUNCNORM_VAR) * se
          and abs(rep['var'] - TRUNCNORM_VAR) < 5 * 1.1 * se       # sd of x^2 under the truncated normal is 0.73 < 1.1
          and rep['at_bound'] < 1e-5 and abs(rep['positive'] - 0.5) < 2.5 * se)
