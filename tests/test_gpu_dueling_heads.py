"""GPU: the dueling head kernels (DESIGN.md §16, §17), plain and noisy, launch by launch against float64.

`dz_test_dueling_head_fwd` / `dz_test_dueling_head_bwd` run the learner's own launch functions (launch_dueling_head_fwd
and launch_dueling_head_bwd: dueling_head_fwd_kernel, dueling_head_bwd_kernel and their noisy_ variants) with a dueling
learner's offsets and noise layout on h1 streams, parameter blobs and noise applies given here.  The references restate
the head in numpy float64 on the same fp32 inputs: adv = h1_adv W_adv + b_adv, v = h1_val W_val + b_val, q = v + adv -
mean_a adv, the factorised weight W = mu + sigma (eps_in eps_out^T) and bias mu_b + sigma_b eps_out; the backward dadv =
dq - mean_a dq, dval = sum_a dq, dh1_adv = [h1_adv > 0] dadv W_adv^T, dh1_val = [h1_val > 0] dval W_val^T.

Exact: the ReLU masks (h1 = +0, -0 give exactly 0, the smallest denormal passes the gradient), dadv = 0 and dval = dq at
A = 1, q independent of the advantage stream at A = 1, the tf32 hi/lo pair (hi = rna(x), lo = rna(x - hi) of the
kernel's own dh1, rna the round-to-nearest-away of cvt.rna.tf32.f32), noisy with sigma = 0 bitwise the plain kernels,
and a row's bits at every row count and position.  Continuous outputs get a float32 budget per element, u = 2^-24:
  head output  a lane sums 16 fmaf terms, 5 butterfly levels add the lanes, the bias is added last; a noisy weight
               fmaf(sigma, ein * eout, mu) rounds twice and its bias fmaf(sigma_b, eout, t + mu_b) twice:
               e_o = 25 u S_o,  S_o = sum_k |x_k| (|mu_ko| + |sigma_ko ein_k eout_o|) + |mu_b| + |sigma_b eout_o|
  aggregation  q_a = v + (adv_a - m), m = (serial sum) / A:  e_q = e_v + e_adv_a + (sum_a e_adv + A u sum |adv|) / A
               + 3 u (|adv_a| + |m| + |v|)
  transpose    dval = serial sum over A: A u sum |dq|;  dadv = dq - dval / A: u sum |dq| + u |dval / A| + u |dadv|
  dh1          from the kernel's own dadv / dval: (A + 3) u sum_a |dadv_a| (|mu_ka| + |sigma_ka ein_k eout_a|), and
               3 u |dval| (|mu_k| + |sigma_k ein_k eout|) for the value stream.
Every budget carries 1e-12 of its operands for float64's own rounding.  `-s` prints worst error / budget per case.
"""

import ctypes as C

import numpy as np
import pytest
import torch

import test_gpu_loss_kernels as lk

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ACTIONS = [1, 2, 3, 4, 5, 7, 18, 33, 63, 64]
ROWS = [1, 7, 8, 9, 33]
BIG = 1024
f32, dev, within = lk.f32, lk.dev, lk.within

_LEARNERS = {}


def learner(A, noisy):
  from dqn_zoo_b200 import learner as dl
  if (A, noisy) not in _LEARNERS:
    _LEARNERS[A, noisy] = dl.Learner(dl.NetworkSpec('dqn', A, obs_shape=(44, 44, 4), dueling=True, noisy=noisy),
                                     batch_size=4)
  return _LEARNERS[A, noisy]


@pytest.fixture(scope='module', autouse=True)
def _free_learners():
  yield
  _LEARNERS.clear()


def stream():
  return torch.cuda.current_stream().cuda_stream


def nan(*shape):
  return torch.full(shape, float('nan'), dtype=torch.float32, device='cuda')


def ptrs(ts):
  return (C.c_void_p * len(ts))(*[None if t is None else (t if isinstance(t, int) else t.data_ptr()) for t in ts])


def noise_offsets(L):
  """The offsets of the heads' eps_in / eps_out in one noise apply (DESIGN.md §17: a1i, a1o, a2i, a2o, v1i, v1o, v2i,
  v2o, each padded to 4 floats), checked against the library's stride."""
  D, A = L.tensors['adv1/mu/w'][1][0], L.net.num_actions
  r4 = lambda n: (n + 3) // 4 * 4
  a2i = D + 512
  a2o = a2i + 512
  v2i = a2o + r4(A) + D + 512
  v2o = v2i + 512
  assert v2o + 4 == L.noise_stride
  return a2i, a2o, v2i, v2o


class Head:
  """A parameter blob of learner L with random head weights: per stream (mu, sigma, mu_b, sigma_b) as float32 numpy."""

  def __init__(self, L, rs, sigma_scale=1.0, adv_bias=None):
    self.noisy = L.net.noisy
    A = L.net.num_actions
    self.blob = torch.full((L.plan.param_count,), float('nan'), dtype=torch.float32, device='cuda')
    s = 1 / np.sqrt(512)
    self.p = {}
    for name, n in (('adv2', A), ('val2', 1)):
      mu, mub = f32(rs.uniform(-s, s, (512, n))), f32(rs.uniform(-s, s, n))
      if name == 'adv2' and adv_bias is not None:
        mub = f32(adv_bias)
      sg, sgb = f32(rs.uniform(0, 0.5 * s, (512, n)) * sigma_scale), f32(rs.uniform(0, 0.5 * s, n) * sigma_scale)
      if not self.noisy:
        sg, sgb = np.zeros_like(sg), np.zeros_like(sgb)
      self.p[name] = (mu, sg, mub, sgb)
      names = ((name + '/mu/w', mu), (name + '/sigma/w', sg), (name + '/mu/b', mub), (name + '/sigma/b', sgb)) \
          if self.noisy else ((name + '/w', mu), (name + '/b', mub))
      for key, v in names:
        L.view(self.blob, key).copy_(torch.as_tensor(v))


def h1_rows(rows, rs):
  """Post-ReLU activations with exact zeros of both signs and the smallest denormal among the positives."""
  x = f32(np.maximum(rs.standard_normal((rows, 512)), 0.0))
  x[rs.uniform(size=x.shape) < 0.1] = -0.0
  x[rs.uniform(size=x.shape) < 0.05] = np.float32(2.0 ** -149)
  return x


def noise_rows(L, rows, rs):
  """Noise applies [rows][stride]: eps values of the factorised form sign(e) sqrt|e|."""
  e = rs.standard_normal((rows, L.noise_stride))
  return f32(np.sign(e) * np.sqrt(np.abs(e)))


def eps_of(L, noise):
  """(ein_adv [R][512], eout_adv [R][A], ein_val [R][512], eout_val [R][1]) of noise applies [R][stride]."""
  a2i, a2o, v2i, v2o = noise_offsets(L)
  A = L.net.num_actions
  n = noise.astype(np.float64)
  return n[:, a2i:a2i + 512], n[:, a2o:a2o + A], n[:, v2i:v2i + 512], n[:, v2o:v2o + 1]


def stream_out(x, p, ei, eo):
  """x W + b of one stream with the factorised noise (ei [R][512], eo [R][n]; zeros for the plain head), and S_o."""
  mu, sg, mub, sgb = (v.astype(np.float64) for v in p)
  ax = np.abs(x)
  out = x @ mu + ((x * ei) @ sg) * eo + mub + sgb * eo
  S = ax @ np.abs(mu) + ((ax * np.abs(ei)) @ sg) * np.abs(eo) + np.abs(mub) + sgb * np.abs(eo)
  return out, S


def forward_ref(L, head, xa, xv, noise):
  """float64 q [R][A] and its budget; noise [R][stride] or None."""
  A = L.net.num_actions
  R = xa.shape[0]
  if noise is None:
    eia, eoa, eiv, eov = np.zeros((R, 512)), np.zeros((R, A)), np.zeros((R, 512)), np.zeros((R, 1))
  else:
    eia, eoa, eiv, eov = eps_of(L, noise)
  adv, Sa = stream_out(xa.astype(np.float64), head.p['adv2'], eia, eoa)
  v, Sv = stream_out(xv.astype(np.float64), head.p['val2'], eiv, eov)
  m = adv.mean(1, keepdims=True)
  q = v + adv - m
  e_adv, e_v = 25 * U * Sa, 25 * U * Sv
  e_q = e_v + e_adv + (e_adv.sum(1, keepdims=True) + A * U * np.abs(adv).sum(1, keepdims=True)) / A \
      + 3 * U * (np.abs(adv) + np.abs(m) + np.abs(v))
  return q, e_q, v, e_v


def run_fwd(L, rows, h1, blobs, noise, noise_ld=0):
  """h1: per pass (adv, val) device tensors or pointers; noise: per pass device pointers or None."""
  from dqn_zoo_b200 import _lib
  np_ = len(blobs)
  A = L.net.num_actions
  out = [nan(rows + 1, A) for _ in range(np_)]
  _lib.call('dz_test_dueling_head_fwd', L._h, rows, np_, ptrs([t for pair in h1 for t in pair]), ptrs(blobs),
            None if noise is None else ptrs(noise), noise_ld, ptrs(out), stream())
  torch.cuda.synchronize()
  res = [o.cpu().numpy() for o in out]
  for o in res:
    assert np.isnan(o[rows]).all(), 'a row past the last was written'
  return [o[:rows] for o in res]


@pytest.mark.parametrize('noisy', [False, True], ids=['plain', 'noisy'])
@pytest.mark.parametrize('A', ACTIONS)
def test_dueling_head_forward(A, noisy):
  """Three passes with distinct blobs (and noise applies) over 1024 rows, one pass with large advantage biases of mixed
  sign that cancel in the mean; then 1 to 3 passes at 1, 7, 8, 9 and 33 rows from other positions, bit for bit; noisy:
  every row its own apply (noise_ld = stride) and sigma = 0 against the plain kernel."""
  L = learner(A, noisy)
  rs = np.random.RandomState(A * 2 + noisy)
  big_bias = np.where(np.arange(A) % 2 == 0, 3.0e3, -3.0e3) + rs.uniform(-1, 1, A) if A > 1 else None
  heads = [Head(L, rs), Head(L, rs, adv_bias=big_bias), Head(L, rs, sigma_scale=4.0)]
  xs = [(h1_rows(BIG, rs), h1_rows(BIG, rs)) for _ in range(3)]
  h1 = [(dev(a), dev(v)) for a, v in xs]
  noise = [f32(noise_rows(L, 1, rs)) for _ in range(3)] if noisy else None
  nd = [dev(n) for n in noise] if noisy else None
  big = run_fwd(L, BIG, h1, [h.blob for h in heads], nd)
  worst = 0.0
  for i in range(3):
    q, e_q, _, _ = forward_ref(L, heads[i], *xs[i], None if not noisy else np.repeat(noise[i], BIG, 0))
    worst = max(worst, within('q pass %d' % i, big[i], q, e_q, np.abs(q) + 1))
  for rows in ROWS:
    start = rs.randint(0, BIG - rows + 1)
    np_ = 1 + rows % 3
    sub = [(h1[i][0].data_ptr() + 4 * 512 * start, h1[i][1].data_ptr() + 4 * 512 * start) for i in range(np_)]
    got = run_fwd(L, rows, sub, [h.blob for h in heads[:np_]], nd[:np_] if noisy else None)
    for i in range(np_):
      np.testing.assert_array_equal(got[i], big[i][start:start + rows], err_msg='rows=%d pass %d' % (rows, i))
  if A == 1:   # q = v exactly: the advantage stream cannot move a bit
    other = Head(L, rs)
    names = ('/mu/w', '/sigma/w', '/mu/b', '/sigma/b') if noisy else ('/w', None, '/b', None)
    for name, v in zip(names, heads[0].p['val2']):
      if name:
        L.view(other.blob, 'val2' + name).copy_(torch.as_tensor(v))
    alt = run_fwd(L, BIG, [(dev(h1_rows(BIG, rs)), h1[0][1])], [other.blob], nd[:1] if noisy else None)
    np.testing.assert_array_equal(alt[0], big[0])
    _, _, v, e_v = forward_ref(L, heads[0], *xs[0], None if not noisy else np.repeat(noise[0], BIG, 0))
    worst = max(worst, within('q = v', big[0], v, e_v, np.abs(v) + 1))
  if noisy:
    stride = L.noise_stride
    per_row = [noise_rows(L, BIG, rs) for _ in range(2)]
    pd = [dev(n) for n in per_row]
    got = run_fwd(L, BIG, h1[:2], [h.blob for h in heads[:2]], pd, noise_ld=stride)
    for i in range(2):
      q, e_q, _, _ = forward_ref(L, heads[i], *xs[i], per_row[i])
      worst = max(worst, within('q per-row noise pass %d' % i, got[i], q, e_q, np.abs(q) + 1))
    start, rows = 517, 33
    sub = run_fwd(L, rows, [(h1[0][0].data_ptr() + 4 * 512 * start, h1[0][1].data_ptr() + 4 * 512 * start)],
                  [heads[0].blob], [pd[0].data_ptr() + 4 * stride * start], noise_ld=stride)
    np.testing.assert_array_equal(sub[0], got[0][start:start + rows])
    # sigma = 0: fmaf(0, ., mu) is mu, so the noisy kernel gives the plain kernel's bits
    P = learner(A, False)
    zero = Head(L, rs, sigma_scale=0.0)
    plain = Head(P, rs)
    for k in ('adv2', 'val2'):
      P.view(plain.blob, k + '/w').copy_(torch.as_tensor(zero.p[k][0]))
      P.view(plain.blob, k + '/b').copy_(torch.as_tensor(zero.p[k][2]))
    got_n = run_fwd(L, BIG, h1[:1], [zero.blob], nd[:1])
    got_p = run_fwd(P, BIG, h1[:1], [plain.blob], None)
    np.testing.assert_array_equal(got_n[0], got_p[0])
  print('dueling head fwd A=%d %s: worst error / budget %.3f' % (A, 'noisy' if noisy else 'plain', worst))


# ---- backward ---------------------------------------------------------------------------------------------------------

def rna_tf32(x):
  """cvt.rna.tf32.f32 on finite float32: round to 10 mantissa bits, ties away from zero (on the magnitude's bits)."""
  b = np.asarray(x, np.float32).view(np.uint32)
  return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def run_bwd(L, rows, dq, h1, blob, noise, with_hilo):
  from dqn_zoo_b200 import _lib
  A = L.net.num_actions
  dq_d = dev(np.concatenate([dq, np.full((1, A), np.nan, np.float32)]))
  dval = nan(rows + 1)
  dh1 = [nan(rows + 1, 512) for _ in range(2)]
  hi = [nan(rows + 1, 512) for _ in range(2)] if with_hilo else None
  lo = [nan(rows + 1, 512) for _ in range(2)] if with_hilo else None
  _lib.call('dz_test_dueling_head_bwd', L._h, rows, dq_d.data_ptr(), dval.data_ptr(), ptrs(h1), blob.data_ptr(),
            None if noise is None else (noise if isinstance(noise, int) else noise.data_ptr()), ptrs(dh1),
            None if hi is None else ptrs(hi), None if lo is None else ptrs(lo), stream())
  torch.cuda.synchronize()
  out = dict(dadv=dq_d.cpu().numpy(), dval=dval.cpu().numpy(), dh1=[t.cpu().numpy() for t in dh1])
  if with_hilo:
    out['hi'], out['lo'] = [t.cpu().numpy() for t in hi], [t.cpu().numpy() for t in lo]
  for k, v in out.items():
    for t in (v if isinstance(v, list) else [v]):
      assert np.isnan(t[rows]).all(), (k, 'a row past the last was written')
  return {k: [t[:rows] for t in v] if isinstance(v, list) else v[:rows] for k, v in out.items()}


@pytest.mark.parametrize('noisy', [False, True], ids=['plain', 'noisy'])
@pytest.mark.parametrize('A', ACTIONS)
def test_dueling_head_backward(A, noisy):
  """1024 rows against float64 with exact masks and the tf32 pair, the same bits without hi / lo and at other row
  counts and positions; A = 1: dadv = 0 and dval = dq exactly; noisy with sigma = 0: the plain kernel's bits."""
  L = learner(A, noisy)
  rs = np.random.RandomState(100 + A * 2 + noisy)
  head = Head(L, rs)
  xa, xv = h1_rows(BIG, rs), h1_rows(BIG, rs)
  h1 = [dev(xa), dev(xv)]
  dq = f32(rs.standard_normal((BIG, A)))
  dq[::5] *= 1e3
  noise = noise_rows(L, 1, rs) if noisy else None
  nd = dev(noise) if noisy else None
  got = run_bwd(L, BIG, dq, h1, head.blob, nd, True)
  dq64 = dq.astype(np.float64)
  s = dq64.sum(1)
  worst = within('dval', got['dval'], s, A * U * np.abs(dq64).sum(1), np.abs(s) + 1)
  dadv = dq64 - s[:, None] / A
  e_dadv = U * np.abs(dq64).sum(1, keepdims=True) + U * np.abs(s[:, None] / A) + U * np.abs(dadv)
  worst = max(worst, within('dadv', got['dadv'], dadv, e_dadv, np.abs(dadv) + 1))
  if A == 1:
    assert (got['dadv'] == 0).all() and (got['dval'] == dq[:, 0]).all()
  if noisy:
    eia, eoa, eiv, eov = (e[0] for e in eps_of(L, noise))
  else:
    eia, eoa, eiv, eov = np.zeros(512), np.zeros(A), np.zeros(512), np.zeros(1)
  mu, sg = (v.astype(np.float64) for v in head.p['adv2'][:2])
  Wa, Wa_abs = mu + sg * np.outer(eia, eoa), np.abs(mu) + sg * np.abs(np.outer(eia, eoa))
  muv, sgv = (v.astype(np.float64)[:, 0] for v in head.p['val2'][:2])
  Wv, Wv_abs = muv + sgv * eiv * eov[0], np.abs(muv) + sgv * np.abs(eiv * eov[0])
  da, dv = got['dadv'].astype(np.float64), got['dval'].astype(np.float64)
  refs = [(xa, da @ Wa.T, (A + 3) * U * (np.abs(da) @ Wa_abs.T)),
          (xv, dv[:, None] * Wv[None, :], 3 * U * np.abs(dv)[:, None] * Wv_abs[None, :])]
  for s_, (x, want, bud) in enumerate(refs):
    g = got['dh1'][s_]
    off = ~(x > 0)
    assert (g[off] == 0).all() and not np.signbit(g[off]).any(), 'stream %d: a masked gradient is not +0' % s_
    if A == 1 and s_ == 0:
      assert (g == 0).all(), 'A = 1: dadv = 0 leaves the advantage stream no gradient'
    else:
      live = (x == np.float32(2.0 ** -149)) & (np.abs(want) > bud)   # the smallest denormal passes the gradient
      assert live.any() and (g[live] != 0).all(), 'stream %d: a denormal h1 masked the gradient' % s_
    worst = max(worst, within('dh1 stream %d' % s_, np.where(off, 0.0, g), np.where(off, 0.0, want), bud,
                              np.abs(want) + 1))
    hi = rna_tf32(g)
    lo = rna_tf32((g - hi).astype(np.float32))
    assert (got['hi'][s_].view(np.uint32) == hi.view(np.uint32)).all(), 'stream %d: tf32 hi' % s_
    assert (got['lo'][s_].view(np.uint32) == lo.view(np.uint32)).all(), 'stream %d: tf32 lo' % s_
  bare = run_bwd(L, BIG, dq, h1, head.blob, nd, False)
  for k in ('dadv', 'dval'):
    np.testing.assert_array_equal(bare[k], got[k])
  for s_ in range(2):
    np.testing.assert_array_equal(bare['dh1'][s_], got['dh1'][s_])
  for rows in ROWS:
    start = rs.randint(0, BIG - rows + 1)
    sub = run_bwd(L, rows, dq[start:start + rows], [t.data_ptr() + 4 * 512 * start for t in h1], head.blob, nd,
                  rows % 2 == 1)
    for k in ('dadv', 'dval'):
      np.testing.assert_array_equal(sub[k], got[k][start:start + rows], err_msg='%s rows=%d' % (k, rows))
    for s_ in range(2):
      np.testing.assert_array_equal(sub['dh1'][s_], got['dh1'][s_][start:start + rows])
      if 'hi' in sub:
        np.testing.assert_array_equal(sub['hi'][s_], got['hi'][s_][start:start + rows])
        np.testing.assert_array_equal(sub['lo'][s_], got['lo'][s_][start:start + rows])
  if noisy:
    P = learner(A, False)
    zero = Head(L, rs, sigma_scale=0.0)
    plain = Head(P, rs)
    for k in ('adv2', 'val2'):
      P.view(plain.blob, k + '/w').copy_(torch.as_tensor(zero.p[k][0]))
      P.view(plain.blob, k + '/b').copy_(torch.as_tensor(zero.p[k][2]))
    got_n = run_bwd(L, BIG, dq, h1, zero.blob, nd, True)
    got_p = run_bwd(P, BIG, dq, h1, plain.blob, None, True)
    for k in ('dadv', 'dval'):
      np.testing.assert_array_equal(got_n[k], got_p[k])
    for k in ('dh1', 'hi', 'lo'):
      for s_ in range(2):
        np.testing.assert_array_equal(got_n[k][s_], got_p[k][s_])
  print('dueling head bwd A=%d %s: worst error / budget %.3f' % (A, 'noisy' if noisy else 'plain', worst))
