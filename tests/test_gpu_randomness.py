"""GPU: the device generator's draws against float64 (oracle/philox_oracle.py).

The other tests of `randomness_kernel` compare two call paths with each other; here the draws themselves are checked:
the words are Philox4x32-10 under the documented counter layout (taus bit for bit), the noise is the inverse-CDF draw
of a normal TRUNCATED to [-2, 2] (a clipped one puts 2.3 % of its mass on each bound) passed through sign(x) sqrt|x|,
and applies, streams, counters and the two stream ids are independent of each other.  Every entry point that launches
the kernel is called through the C interface into a buffer of the test's own with a canary border.

Tolerance of the noise.  The device forms v = lo + (-2 lo) (k + 0.5) 2^-24 in float32: k + 0.5 is not representable
for k >= 2^23 (half a 24-bit cell, (-2 lo) 2^-25 = 5.7e-8 in v) and the product and the sum round once each (<= 3e-8
each for |v| < 1), so |dv| <= 1.2e-7.  x = sqrt(2) erfinv(v) has dx/dv = sqrt(pi / 2) exp(x^2 / 2) (1.25 at 0, 9.3
at the bounds), erfinvf is documented at 2 ulp, and the multiply, the square root and squaring the float32 result back
add under 2e-7 relative: |dx| <= 1.2e-7 sqrt(pi / 2) exp(x^2 / 2) + 5e-7 |x|.  The comparison is made on x = sign(g)
g^2, where that bound holds everywhere.  On g = sign(x) sqrt|x| itself an absolute bar cannot hold near x = 0, where
the square root is infinitely steep (dg = dx / (2 sqrt|x|)): 1e-6 is asserted for |x| >= 0.01 and the worst element is
printed.
"""

import numpy as np
import pytest
import torch

from oracle import philox_oracle as po

pytestmark = pytest.mark.gpu

CANARY = -7.25
BORDER = 32
SEEDS = [(0, 0), (7, 3), (2 ** 32 + 5, 11), (13, 2 ** 32 + 9), (2 ** 63 + 12345, 2 ** 40 + 1)]   # (seed, counter)

_CACHE = {}


@pytest.fixture(scope='module', autouse=True)
def _release():
  yield
  _CACHE.clear()


def _learner(kind):
  """rainbow: 84x84, batch 32 (a noise apply is 8680 floats).  iqn: 44x44, batch 31, taus (33, 40, 36): 3379 taus per
  update, three past a multiple of 4."""
  if kind not in _CACHE:
    from dqn_zoo_b200 import learner as dl
    if kind == 'rainbow':
      _CACHE[kind] = dl.Learner(dl.NetworkSpec('rainbow', 6), batch_size=32)
    else:
      net = dl.NetworkSpec('iqn', 6, obs_shape=(44, 44, 4), tau_samples_s_tm1=33, tau_samples_policy=40, tau_samples_s_t=36)
      _CACHE[kind] = dl.Learner(net, batch_size=31)
    _CACHE[kind].init_params(1)
  return _CACHE[kind]


def _stream():
  return torch.cuda.current_stream().cuda_stream


def _draw(n, call):
  """Runs call(pointer) on n floats inside a canary border; returns them after checking the border is intact."""
  buf = torch.full((n + 2 * BORDER,), CANARY, dtype=torch.float32, device='cuda')
  call(buf.data_ptr() + 4 * BORDER)
  torch.cuda.synchronize()
  out = buf.cpu().numpy()
  assert np.all(out[:BORDER] == CANARY) and np.all(out[BORDER + n:] == CANARY), 'the generator wrote outside its n floats'
  assert not np.any(out[BORDER:BORDER + n] == CANARY)
  return out[BORDER:BORDER + n].copy()


def _learner_taus(L, seed, ctr):
  from dqn_zoo_b200 import _lib
  net = L.net
  n = L.batch_size * (net.tau_samples_s_tm1 + net.tau_samples_policy + net.tau_samples_s_t)
  L.counters[1] = ctr
  out = _draw(n, lambda p: _lib.call('dz_learner_generate_randomness', L._h, seed, p, 0, _stream()))
  assert int(L.counters[1]) == ctr + 1, 'one counter step per call'
  return out


def _learner_noise(L, seed, ctr, streams=None):
  """streams None: the three applies of one update (dz_learner_generate_randomness); else E per-stream applies."""
  from dqn_zoo_b200 import _lib
  L.counters[1] = ctr
  if streams is None:
    out = _draw(3 * L.noise_stride, lambda p: _lib.call('dz_learner_generate_randomness', L._h, seed, 0, p, _stream()))
  else:
    out = _draw(streams * L.noise_stride,
                lambda p: _lib.call('dz_learner_generate_stream_noise', L._h, seed, streams, p, _stream()))
  assert int(L.counters[1]) == ctr + 1, 'one counter step per call'
  return out


def _actor_draw(L, actor, n, seed, ctr, per_stream):
  from dqn_zoo_b200 import _lib
  if actor.frozen:
    actor.counter = ctr
  else:
    L.counters[1] = ctr
  before = L.counters.clone()
  out = _draw(n, lambda p: _lib.call('dz_actor_generate_randomness', actor._h, seed, 1 if per_stream else 0, p, _stream()))
  if actor.frozen:
    assert actor.counter == ctr + 1 and torch.equal(L.counters, before), 'a frozen actor draws from its own counter'
  else:
    assert int(L.counters[1]) == ctr + 1
  return out


def _x_bound(x):
  return 1.2e-7 * np.sqrt(np.pi / 2) * np.exp(0.5 * x * x) + 5e-7 * np.abs(x)


def _check_noise(got, seed, ctr, where):
  """Device noise g (float32) against the float64 oracle; returns (worst |dg| over |x| >= 0.01, worst dx / bound)."""
  n = got.size
  x_ref = po.truncated_normal(n, seed, ctr)
  g_ref = np.sign(x_ref) * np.sqrt(np.abs(x_ref))
  g = got.astype(np.float64)
  assert np.all(np.isfinite(g)) and np.abs(g).max() <= np.sqrt(2.0), where
  x_dev = np.sign(g) * g * g
  ratio = np.abs(x_dev - x_ref) / _x_bound(x_ref)
  i = int(np.argmax(ratio))
  assert ratio[i] <= 1.0, (where, 'element', i, 'x', x_ref[i], 'device', x_dev[i], 'error / bound', ratio[i])
  away = np.abs(x_ref) >= 0.01
  dg = np.abs(g - g_ref)
  j = int(np.argmax(np.where(away, dg, 0)))
  assert dg[j] <= 1e-6, (where, 'element', j, 'x', x_ref[j], 'noise', g[j], g_ref[j])
  k = int(np.argmax(dg))
  return dg[j], x_ref[j], ratio[i], dg[k], x_ref[k]


# ---- the words and the transforms -------------------------------------------------------------------------------------

@pytest.mark.parametrize('seed,ctr', SEEDS)
def test_learner_taus_are_philox_bit_for_bit(seed, ctr):
  L = _learner('iqn')
  got = _learner_taus(L, seed, ctr)
  assert got.size % 4 == 3                      # the last block writes three of its four words
  np.testing.assert_array_equal(got, po.taus(got.size, seed, ctr))
  assert got.min() >= 0.0 and got.max() < 1.0


@pytest.mark.parametrize('frozen', [False, True])
def test_actor_taus_are_philox_bit_for_bit(frozen):
  L = _learner('iqn')
  for E in (1, 5, 131):                          # 40, 200 and 5240 taus
    actor = L.actor(E, frozen=frozen)
    for seed, ctr in SEEDS[1:4]:
      got = _actor_draw(L, actor, E * L.net.tau_samples_policy, seed, ctr, False)
      np.testing.assert_array_equal(got, po.taus(got.size, seed, ctr))


def test_a_ragged_tail_of_one_and_two_words():
  """Tau counts 1 and 2 past a multiple of 4 (batch 31 x (33, 40, 36) covers 3): the last block is cut where it should be."""
  from dqn_zoo_b200 import learner as dl
  for taus in ((3, 2, 2), (2, 2, 2)):            # 7 * 3 = 21 and 6 * 3 = 18 taus
    net = dl.NetworkSpec('iqn', 6, obs_shape=(44, 44, 4), tau_samples_s_tm1=taus[0], tau_samples_policy=taus[1],
                         tau_samples_s_t=taus[2])
    L = dl.Learner(net, batch_size=3)
    got = _learner_taus(L, 21, 6)
    assert got.size % 4 == sum(taus) * 3 % 4 and got.size % 4 in (1, 2)
    np.testing.assert_array_equal(got, po.taus(got.size, 21, 6))


@pytest.mark.parametrize('seed,ctr', SEEDS)
def test_learner_noise_against_float64(seed, ctr):
  L = _learner('rainbow')
  got = _learner_noise(L, seed, ctr)
  worst_g, at_x, worst_ratio, worst_any, any_x = _check_noise(got, seed, ctr, 'update noise')
  print('noise seed %d counter %d: worst |dg| %.2e at x = %.4f (|x| >= 0.01), anywhere %.2e at x = %.2e; worst dx / bound '
        '%.2f' % (seed, ctr, worst_g, at_x, worst_any, any_x, worst_ratio))
  rows = _learner_noise(L, seed, ctr, streams=32)
  _check_noise(rows, seed, ctr, 'stream noise')
  np.testing.assert_array_equal(rows[:got.size], got)   # the first three applies are the update's


@pytest.mark.parametrize('frozen', [False, True])
def test_actor_noise_against_float64(frozen):
  L = _learner('rainbow')
  S = L.noise_stride
  actor = L.actor(40, frozen=frozen)                     # more streams than the learner's batch
  for seed, ctr in SEEDS[2:4]:
    _check_noise(_actor_draw(L, actor, S, seed, ctr, False), seed, ctr, 'actor noise')
    _check_noise(_actor_draw(L, actor, 40 * S, seed, ctr, True), seed, ctr, 'actor stream noise')


# ---- distribution -----------------------------------------------------------------------------------------------------

def test_tau_distribution():
  """2^20 taus over 64 counters (an actor of 256 streams x 64 taus): uniform on [0, 1)."""
  import scipy.stats
  from dqn_zoo_b200 import learner as dl
  L = dl.Learner(dl.NetworkSpec('iqn', 6, obs_shape=(44, 44, 4)), batch_size=4)
  actor = L.actor(256)
  t = np.concatenate([_actor_draw(L, actor, 256 * 64, 5, ctr, False) for ctr in range(64)]).astype(np.float64)
  n = t.size
  assert n == 1 << 20
  ks = scipy.stats.kstest(t, 'uniform').statistic
  print('taus: n %d KS %.2e mean %.6f var %.6f min %.3g max %.9f' % (n, ks, t.mean(), t.var(), t.min(), t.max()))
  assert ks < 3e-3
  assert t.min() >= 0.0 and t.max() < 1.0
  se = 1 / np.sqrt(n)
  assert abs(t.mean() - 0.5) < 5 * np.sqrt(1 / 12) * se and abs(t.var() - 1 / 12) < 5 * np.sqrt(1 / 180) * se
  counts = np.bincount((t * 16).astype(int), minlength=16)         # chi-square over 16 cells, 15 degrees of freedom
  chi2 = float(((counts - n / 16) ** 2 / (n / 16)).sum())
  assert chi2 < 50.0, chi2                                          # P(chi2_15 > 50) = 1.2e-5
  # the low byte of the 24 kept bits is as uniform as the high ones
  low = np.bincount((t * 2 ** 24).astype(np.int64) & 0xFF, minlength=256)
  assert float(((low - n / 256) ** 2 / (n / 256)).sum()) < 400.0    # P(chi2_255 > 400) = 1e-8


def test_noise_distribution():
  """1.1 M noise draws over four counters: x = sign(g) g^2 is a normal truncated (not clipped) to [-2, 2]."""
  L = _learner('rainbow')
  g = np.concatenate([_learner_noise(L, 77, ctr, streams=32) for ctr in range(4)]).astype(np.float64)
  n = g.size
  assert n >= 1 << 20
  x = np.sign(g) * g * g
  rep = po.truncnorm_report(x)
  print('noise: n %d KS %.2e mean %.2e var %.5f (truncated normal %.5f) on a bound %.1e positive %.5f'
        % (n, rep['ks'], rep['mean'], rep['var'], po.TRUNCNORM_VAR, rep['at_bound'], rep['positive']))
  assert po.truncnorm_report_ok(rep, n), rep


# ---- independence -----------------------------------------------------------------------------------------------------

def _corr(a, b):
  a = a - a.mean()
  b = b - b.mean()
  return float((a * b).sum() / np.sqrt((a * a).sum() * (b * b).sum()))


def _assert_independent(rows, what):
  """rows [k, n]: every pair uncorrelated to five standard errors, and no two rows with a common 64-element prefix."""
  k, n = rows.shape
  worst = 0.0
  for i in range(k):
    for j in range(i):
      worst = max(worst, abs(_corr(rows[i], rows[j])))
  assert worst < 5 / np.sqrt(n), (what, worst, 5 / np.sqrt(n))
  assert len({row[:64].tobytes() for row in rows}) == k, what
  return worst


def test_applies_streams_counters_and_stream_ids_are_independent():
  R, Q = _learner('rainbow'), _learner('iqn')
  S = R.noise_stride
  sq = lambda g: np.sign(g) * g.astype(np.float64) ** 2
  three = sq(_learner_noise(R, 41, 8)).reshape(3, S)
  w3 = _assert_independent(three, 'the three applies of one update')
  streams = sq(_learner_noise(R, 41, 8, streams=32)).reshape(32, S)
  w32 = _assert_independent(streams, '32 per-stream applies')
  nt = Q.batch_size * (33 + 40 + 36)
  by_counter = np.stack([_learner_taus(Q, 41, c).astype(np.float64) for c in (8, 9, 10, 11)])
  wc = _assert_independent(by_counter, 'taus of consecutive counters')
  noise_by_counter = np.stack([sq(_learner_noise(R, 41, c))[:S] for c in (8, 9, 10, 11)])
  wn = _assert_independent(noise_by_counter, 'noise of consecutive counters')
  by_seed = np.stack([_learner_taus(Q, s, 8).astype(np.float64) for s in (41, 42, 41 + 2 ** 32)])
  ws = _assert_independent(by_seed, 'taus of neighbouring seeds')
  # same seed, same counter: only the stream id separates the taus from the noise.  The noise is a monotone function
  # of its word, so taus drawn from the SAME words would correlate at 0.97.
  pair = np.stack([by_counter[0], three.reshape(-1)[:nt]])
  wi = _assert_independent(pair, 'taus against noise at one seed and counter')
  same_words = (po.words(nt, 41, 8, po.STREAM_NOISE) >> np.uint32(8)).astype(np.float64)
  assert _corr(same_words, three.reshape(-1)[:nt]) > 0.9
  print('worst |r|: applies %.4f streams %.4f tau counters %.4f noise counters %.4f seeds %.4f taus/noise %.4f'
        % (w3, w32, wc, wn, ws, wi))
