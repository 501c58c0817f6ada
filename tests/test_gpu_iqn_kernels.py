"""GPU: the kernels of IQN's network (iqn, munchausen_iqn and fqf; networks.py:264-292), launch by launch against float64.

The hooks run the learner's own launch functions on buffers given here: `dz_test_iqn_cos` (launch_iqn_cos:
iqn_cos_kernel), `dz_test_iqn_head_fwd` / `dz_test_iqn_head_dgrad` (launch_iqn_head_fwd / launch_iqn_head_dgrad, with an
IQN learner's offsets of head/w and head/b), `dz_test_iqn_hadamard_bwd` (launch_iqn_hadamard_bwd, unpacked and packed)
and `dz_test_iqn_embed_packed` (the learner's embedding problem, pk_embed_problem, on tc_pgemm_kernel's EPI = 1 epilogue).

Exact, asserted bit for bit: cos(0) = 1; every ReLU mask at +0, -0 and +-2^-149 (a masked output is +0, the smallest
positive denormal passes); the Hadamard backward's dE = fl(g f), and the packed kernel's transposed image equals the tf32
split of the unpacked kernel's dE at pk_index(k, b 64 + n); the embedding epilogue's images hold hi = rna(h), lo =
rna(h - hi) of the kernel's own h = fl(E0 act3[i / mul_div]) (rna: cvt.rna.tf32.f32), the transposed image is the plain
image transposed, and image padding (zeroed here, as the learner zeroes it once) stays zero, the ones row included;
the value head's and its input gradient's rows do not depend on the row count, the row's position or the other applies
of the launch.  Every output starts as NaN and the element past the end must stay NaN.

Continuous outputs get a per-element float32 budget, u = 2^-24, from each kernel's operation order; a path of n
roundings costs (1 + u)^n - 1 < (n + 1) u of the magnitudes it carries:
  cos          CUDA's cosf is within 2 ulp of cos of its float32 argument (CUDA C++ Programming Guide, Mathematical
               Functions); the argument fl(fl((j + 1) pi_f) tau) is formed here in float32 the same way:
               e = 2 ulp_32(cos x).
  head fwd     a lane chains 16 fmaf, 5 butterfly levels add the lanes, the bias is added last, 22 roundings:
               e = 23 u (sum_k |h1_k W_ka| + |b_a|).
  head dgrad   a chain of A fmaf over the actions: e = (A + 1) u sum_a |dout_a W_ka|.
  dfeat        unpacked: a serial sum over N (fused or not, N roundings per term): (N + 1) u sum_n |g e|; packed: 4
               fmaf per thread then a serial sum of 16 partials, 19 roundings: 20 u sum_n |g e|.
  embed E0     3xTF32: the dropped lo*lo product and both split residuals leave 3 * 2^-22 = 12 u of each |cos W|; each
               of the three MMAs of a k-step truncates its sum (budgeted 4 u each, a truncation of 2 bits); the k-steps'
               partial sums are added with K/8 round-to-nearest adds (K = latent rounded up to 16) and the bias with one:
               e = (25 + K/8) u (sum_r |cos_r W_rj| + |b_j|).
  embed h      hi + lo against float64 E0 act3: e_E0 |act3| + 5 u |E0 act3| (the product rounds once, the split leaves
               at most 2^-22 = 4 u).
Every budget carries 1e-12 of its operands for float64's own rounding.  `-s` prints worst error / budget per case.
"""

import ctypes as C

import numpy as np
import pytest
import torch

import test_gpu_loss_kernels as lk
from test_gpu_dueling_heads import rna_tf32
from test_gpu_packed_gemm import pk_index

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
DENORM = np.float32(2.0 ** -149)
PI32 = np.float32(np.pi)
f32, dev, within = lk.f32, lk.dev, lk.within
ROWS = [1, 7, 8, 9, 511, 512, 2112, 2113, 4096]   # 2112 = 264 blocks x 8 warps: one sweep of the value head's grid
BIG = 4096
ACTIONS = [1, 2, 6, 17, 18]

_LEARNERS = {}


def learner(A):
  from dqn_zoo_b200 import learner as dl
  if A not in _LEARNERS:
    _LEARNERS[A] = dl.Learner(dl.NetworkSpec('iqn', A, obs_shape=(44, 44, 4)), batch_size=4)
  return _LEARNERS[A]


@pytest.fixture(scope='module', autouse=True)
def _free_learners():
  yield
  _LEARNERS.clear()


def stream():
  return torch.cuda.current_stream().cuda_stream


def nan(*shape):
  return torch.full(shape, float('nan'), dtype=torch.float32, device='cuda')


def ptrs(ts):
  return (C.c_void_p * len(ts))(*[t if isinstance(t, int) else t.data_ptr() for t in ts])


def ratio(got, want, budget):
  """Worst error / budget without asserting (the mutation test)."""
  err = np.abs(np.asarray(got, np.float64) - want)
  return float((err / (np.asarray(budget, np.float64) + 1e-30)).max())


def bits(x):
  return np.asarray(x, np.float32).view(np.uint32)


def post_relu(shape, rs):
  """Post-ReLU activations with exact zeros of both signs and the smallest denormal among the positives."""
  x = f32(np.maximum(rs.standard_normal(shape), 0.0))
  x[rs.uniform(size=shape) < 0.1] = -0.0
  x[rs.uniform(size=shape) < 0.05] = DENORM
  return x


def split(x):
  hi = rna_tf32(x)
  return hi, rna_tf32(f32(x - hi))


def ceil_to(n, k):
  return -(-n // k) * k


# ---- cosine features ------------------------------------------------------------------------------------------------

def cos_arg(taus, latent):
  """fl(fl((j + 1) pi_f) tau) in float32, as networks.py:277-278 forms it."""
  pim = f32(np.arange(1, latent + 1, dtype=np.float32) * PI32)
  return f32(taus[:, None] * pim[None, :])


def ulp32(x):
  a = np.maximum(np.abs(np.asarray(x, np.float64)), 2.0 ** -126)
  return 2.0 ** (np.floor(np.log2(a)) - 23)


def run_cos(taus, latent):
  from dqn_zoo_b200 import _lib
  rows = len(taus)
  out, t = nan(rows * latent + 1), dev(taus)
  _lib.call('dz_test_iqn_cos', t.data_ptr(), rows, latent, out.data_ptr(), stream())
  torch.cuda.synchronize()
  o = out.cpu().numpy()
  assert np.isnan(o[-1]), 'an element past the last was written'
  return o[:-1].reshape(rows, latent)


def cos_taus(rows, rs):
  special = f32([0.0, 2.0 ** -24, 0.5, 1.0 - 2.0 ** -24])
  return f32(np.concatenate([special, rs.uniform(0, 1, max(rows - 4, 0))])[:rows])


@pytest.mark.parametrize('latent', [1, 16, 63, 64, 128, 144])
def test_cos(latent):
  """tau at 0, 2^-24, 0.5 and 1 - 2^-24 plus uniforms; row counts that fill the last 256-thread block and that do not.
  At latent 128 the largest argument is 128 pi_f (1 - 2^-24), about 402 rad."""
  rs = np.random.RandomState(latent)
  q = 256 // np.gcd(256, latent)         # rows * latent % 256 == 0 at multiples of q
  worst = 0.0
  for rows in sorted({1, 4, q, q + 1, 2 * q + 3, 2053}):
    taus = cos_taus(rows, rs)
    got = run_cos(taus, latent)
    want = np.cos(cos_arg(taus, latent).astype(np.float64))
    worst = max(worst, within('cos rows=%d' % rows, got, want, 2 * ulp32(want), 1.0))
    assert (got[0] == 1.0).all(), 'cos(0) must be exactly 1'
  print('iqn cos latent=%d: worst error / budget %.3f' % (latent, worst))


# ---- value head -----------------------------------------------------------------------------------------------------

class Head:
  """A NaN parameter blob of learner L with a random value head W [512][A], b [A]."""

  def __init__(self, L, rs):
    A = L.net.num_actions
    s = 1 / np.sqrt(512)
    self.W, self.b = f32(rs.uniform(-s, s, (512, A))), f32(rs.uniform(-s, s, A))
    self.blob = torch.full((L.plan.param_count,), float('nan'), dtype=torch.float32, device='cuda')
    L.view(self.blob, 'head/w').copy_(torch.as_tensor(self.W))
    L.view(self.blob, 'head/b').copy_(torch.as_tensor(self.b))


def head_ref(head, x):
  x = x.astype(np.float64)
  W, b = head.W.astype(np.float64), head.b.astype(np.float64)
  return x @ W + b, 23 * U * (np.abs(x) @ np.abs(W) + np.abs(b))


def run_head_fwd(L, Ms, h1, blobs):
  """h1: per apply a device pointer to [M][512]; returns per apply q [M][A]."""
  from dqn_zoo_b200 import _lib
  A = L.net.num_actions
  n = len(Ms)
  out = [nan(M + 1, A) for M in Ms]
  _lib.call('dz_test_iqn_head_fwd', L._h, n, (C.c_int32 * n)(*Ms), ptrs(h1), ptrs(blobs), ptrs(out), stream())
  torch.cuda.synchronize()
  res = [o.cpu().numpy() for o in out]
  for o in res:
    assert np.isnan(o[-1]).all(), 'a row past the last was written'
  return [o[:-1] for o in res]


@pytest.mark.parametrize('A', ACTIONS)
def test_head_forward(A):
  """Three blobs over 4096 rows each against float64; then three applies of different row counts per launch from other
  positions, and single rows alone, bit for bit against the 4096-row outputs."""
  L = learner(A)
  rs = np.random.RandomState(10 + A)
  heads = [Head(L, rs) for _ in range(3)]
  xs = [post_relu((BIG, 512), rs) for _ in range(3)]
  h1 = [dev(x) for x in xs]
  full = [run_head_fwd(L, [BIG], [h1[i]], [heads[i].blob])[0] for i in range(3)]
  worst = 0.0
  for i in range(3):
    want, bud = head_ref(heads[i], xs[i])
    worst = max(worst, within('q apply %d' % i, full[i], want, bud, np.abs(want) + 1))
  for k, M in enumerate(ROWS):
    Ms = [M, ROWS[(k + 3) % len(ROWS)], ROWS[(k + 6) % len(ROWS)]]
    starts = [rs.randint(0, BIG - m + 1) for m in Ms]
    got = run_head_fwd(L, Ms, [h1[i].data_ptr() + 4 * 512 * starts[i] for i in range(3)], [h.blob for h in heads])
    for i in range(3):
      assert (bits(got[i]) == bits(full[i][starts[i]:starts[i] + Ms[i]])).all(), ('Ms', Ms, 'apply', i)
  for r in (0, BIG - 1, rs.randint(BIG), rs.randint(BIG)):
    alone = run_head_fwd(L, [1], [h1[1].data_ptr() + 4 * 512 * r], [heads[1].blob])[0]
    assert (bits(alone[0]) == bits(full[1][r])).all(), ('row alone', r)
  print('iqn head fwd A=%d: worst error / budget %.3f' % (A, worst))


def run_head_dgrad(L, M, dout, blob, h1):
  """dout: device [M][A] (pointer or tensor); h1: device pointer or tensor [M][512]."""
  from dqn_zoo_b200 import _lib
  dh1 = nan(M + 1, 512)
  _lib.call('dz_test_iqn_head_dgrad', L._h, M, dout if isinstance(dout, int) else dout.data_ptr(), blob.data_ptr(),
            h1 if isinstance(h1, int) else h1.data_ptr(), dh1.data_ptr(), stream())
  torch.cuda.synchronize()
  o = dh1.cpu().numpy()
  assert np.isnan(o[-1]).all(), 'a row past the last was written'
  return o[:-1]


def dgrad_inputs(A, rs):
  x = post_relu((BIG, 512), rs)
  x[rs.uniform(size=x.shape) < 0.05] = -DENORM
  dout = f32(rs.standard_normal((BIG, A)))
  dout[::5] *= 1e3
  return x, dout


def dgrad_ref(head, dout):
  A = dout.shape[1]
  d, W = dout.astype(np.float64), head.W.astype(np.float64)
  return d @ W.T, (A + 1) * U * (np.abs(d) @ np.abs(W).T)


@pytest.mark.parametrize('A', ACTIONS)
def test_head_dgrad(A):
  """4096 rows against float64 with h1 at +0, -0 and +-2^-149; the mask exactly; then every row count from other
  positions bit for bit."""
  L = learner(A)
  rs = np.random.RandomState(20 + A)
  head = Head(L, rs)
  x, dout = dgrad_inputs(A, rs)
  h1, dd = dev(x), dev(dout)
  got = run_head_dgrad(L, BIG, dd, head.blob, h1)
  want, bud = dgrad_ref(head, dout)
  off = ~(x > 0)
  assert (bits(got[off]) == 0).all(), 'a masked gradient is not +0'
  live = (x == DENORM) & (np.abs(want) > bud)
  assert live.any() and (got[live] != 0).all(), 'the smallest denormal h1 masked the gradient'
  worst = within('dh1', np.where(off, 0.0, got), np.where(off, 0.0, want), bud, np.abs(want) + 1)
  for M in ROWS:
    s = rs.randint(0, BIG - M + 1)
    sub = run_head_dgrad(L, M, dd.data_ptr() + 4 * A * s, head.blob, h1.data_ptr() + 4 * 512 * s)
    assert (bits(sub) == bits(got[s:s + M])).all(), ('M', M)
  print('iqn head dgrad A=%d: worst error / budget %.3f' % (A, worst))


# ---- Hadamard backward ----------------------------------------------------------------------------------------------

def hadamard_inputs(B, N, D, rs):
  E = post_relu((B, N, D), rs)
  F = post_relu((B, D), rs)
  G = f32(rs.standard_normal((B, N, D)))
  G[:, ::3] *= 1e2
  return G, E, F


def run_hadamard(packed, G, E, F, img_rows_pad=0):
  """Returns (dhi after the call, dfeat, img_hi, img_lo); every buffer carries one NaN element past its end."""
  from dqn_zoo_b200 import _lib
  B, N, D = G.shape
  dhi = dev(np.concatenate([G.reshape(-1), f32([np.nan] * 4)]))
  dfeat = nan(B * D + 4)
  hi = nan(img_rows_pad * B * N + 4) if packed else None
  lo = nan(img_rows_pad * B * N + 4) if packed else None
  dE, dF = dev(E), dev(F)
  _lib.call('dz_test_iqn_hadamard_bwd', int(packed), B, N, D, dhi.data_ptr(), dE.data_ptr(), dF.data_ptr(),
            dfeat.data_ptr(), hi.data_ptr() if packed else None, lo.data_ptr() if packed else None, img_rows_pad, stream())
  torch.cuda.synchronize()
  out = [t.cpu().numpy() for t in (dhi, dfeat)] + ([t.cpu().numpy() for t in (hi, lo)] if packed else [None, None])
  for t in out:
    if t is not None:
      assert np.isnan(t[-4:]).all(), 'an element past the last was written'
  dhi, dfeat = out[0][:-4].reshape(B, N, D), out[1][:-4].reshape(B, D)
  return dhi, dfeat, out[2] if out[2] is None else out[2][:-4], out[3] if out[3] is None else out[3][:-4]


def hadamard_ref(G, E, F):
  """dE exactly (float32 products), dfeat in float64 and sum_n |g e|."""
  dE = np.where(E > 0, f32(G * F[:, None, :]), f32(0.0))
  g, e = G.astype(np.float64), E.astype(np.float64)
  return dE, np.where(F > 0, (g * e).sum(1), 0.0), np.abs(g * e).sum(1)


def check_hadamard_exact(F, dE_got, dE_want, dfeat_got):
  assert (bits(dE_got) == bits(dE_want)).all(), 'dE is not fl(g f) under the E > 0 mask'
  assert (bits(dfeat_got[~(F > 0)]) == 0).all(), 'a masked dfeat is not +0'


@pytest.mark.parametrize('D', [256, 3136])
@pytest.mark.parametrize('N', [1, 5, 7, 8, 32, 33, 64, 201])
def test_hadamard_bwd(N, D):
  """dHI becomes dE in place, bit for bit; dfeat against float64 with E and F at +-0 and 2^-149."""
  B = 3
  rs = np.random.RandomState(N * 7 + D)
  G, E, F = hadamard_inputs(B, N, D, rs)
  dE, dfeat, _, _ = run_hadamard(False, G, E, F)
  dE_want, dfeat_want, S = hadamard_ref(G, E, F)
  check_hadamard_exact(F, dE, dE_want, dfeat)
  live = (E == DENORM) & (dE_want != 0)
  assert live.any() and (dE[live] != 0).all(), 'the smallest denormal E masked dE'
  worst = within('dfeat', dfeat, dfeat_want, (N + 1) * U * S, S)
  print('iqn hadamard bwd N=%d D=%d: worst error / budget %.3f' % (N, D, worst))


def image_index(rows, red, rg):
  r, m = np.meshgrid(np.arange(rows), np.arange(red), indexing='ij')
  return pk_index(r, m, rg)


@pytest.mark.parametrize('B', [16, 17, 32])
@pytest.mark.parametrize('D', [256, 3136])
def test_hadamard_bwd_packed(D, B):
  """N = 64: dfeat against float64 and the unpacked kernel; the dE^T image is the tf32 split of the unpacked kernel's dE
  bit for bit at pk_index(k, b 64 + n); dHI is left as it was and the image's padding rows untouched."""
  N = 64
  rs = np.random.RandomState(B * 3 + D)
  G, E, F = hadamard_inputs(B, N, D, rs)
  rows_pad = ceil_to(D, 128)
  dhi, dfeat, hi, lo = run_hadamard(True, G, E, F, rows_pad)
  dE_un, dfeat_un, _, _ = run_hadamard(False, G, E, F)
  _, dfeat_want, S = hadamard_ref(G, E, F)
  assert (bits(dhi) == bits(G)).all(), 'the packed kernel wrote dHI'
  assert (bits(dfeat[~(F > 0)]) == 0).all(), 'a masked dfeat is not +0'
  worst = within('dfeat', dfeat, dfeat_want, 20 * U * S, S)
  worst = max(worst, within('dfeat vs unpacked', dfeat, dfeat_un.astype(np.float64), (20 + N + 1) * U * S, S))
  idx = image_index(D, B * N, rows_pad // 8)
  want_hi, want_lo = split(dE_un.transpose(2, 0, 1).reshape(D, B * N))
  assert (bits(hi[idx]) == bits(want_hi)).all(), 'dE^T hi is not the split of the unpacked dE'
  assert (bits(lo[idx]) == bits(want_lo)).all(), 'dE^T lo is not the split of the unpacked dE'
  pad = np.ones(hi.size, bool)
  pad[idx.reshape(-1)] = False
  assert np.isnan(hi[pad]).all() and np.isnan(lo[pad]).all(), 'the image padding was written'
  print('iqn hadamard bwd packed D=%d B=%d: worst error / budget %.3f' % (D, B, worst))


# ---- embedding epilogue (EPI = 1) -----------------------------------------------------------------------------------

class Embed:
  """Inputs of one embedding problem: cos [M][latent] with four all-zero rows, W [latent][D] with zero columns, bias at
  +-0 and +-2^-149 among uniforms, act3 [ceil(M / mul_div)][mul_ld] post-ReLU (NaN past D)."""

  def __init__(self, M, latent, D, mul_div, mul_ld, rs):
    self.M, self.latent, self.D, self.mul_div, self.mul_ld = M, latent, D, mul_div, mul_ld
    self.cos = f32(np.cos(cos_arg(f32(rs.uniform(0, 1, M)), latent).astype(np.float64)))
    self.cos[rs.choice(M, 4, replace=False)] = 0.0
    s = 1 / np.sqrt(latent)
    self.W = f32(rs.uniform(-s, s, (latent, D)))
    self.W[:, np.arange(D) % 97 == 5] = 0.0
    b = f32(rs.uniform(-0.2, 0.2, D))
    j = np.arange(D)
    b[j % 13 == 0], b[j % 13 == 1], b[j % 13 == 2], b[j % 13 == 3] = 0.0, -0.0, DENORM, -DENORM
    self.b = b
    self.mul = np.full((-(-M // mul_div), mul_ld), np.nan, np.float32)
    self.mul[:, :D] = post_relu((self.mul.shape[0], D), rs)


def run_embed(e, keep=True):
  """Returns E0 [M][D] (None without keep), the images as flat float32 (img hi/lo, imgT hi/lo or None) and their
  extents.  keep: E0 and the transposed image, as the learner's online apply on s_tm1 writes them."""
  from dqn_zoo_b200 import _lib
  M, latent, D = e.M, e.latent, e.D
  work = nan(_lib.lib.dz_test_tc_pgemm_work(M, D, latent))
  e0 = nan(M + 1, D)
  rp, cp = ceil_to(M, 128), ceil_to(D, 16)
  rpT, cpT = ceil_to(D + 1, 128), ceil_to(M, 16)
  img = [torch.zeros(rp * cp, dtype=torch.float32, device='cuda') for _ in range(2)]
  onesT = np.zeros(rpT * cpT, np.float32)
  onesT[pk_index(D, np.arange(M), rpT // 8)] = 1.0       # the bias-gradient row, as the learner sets it once
  imgT = [dev(onesT), torch.zeros(rpT * cpT, dtype=torch.float32, device='cuda')] if keep else [None, None]
  ins = [dev(x) for x in (e.cos, e.W, e.b, e.mul)]
  _lib.call('dz_test_iqn_embed_packed', ins[0].data_ptr(), M, latent, ins[1].data_ptr(), D, ins[2].data_ptr(),
            ins[3].data_ptr(), e.mul_div, e.mul_ld, work.data_ptr(), e0.data_ptr() if keep else None, img[0].data_ptr(),
            img[1].data_ptr(), imgT[0].data_ptr() if keep else None, imgT[1].data_ptr() if keep else None, stream())
  torch.cuda.synchronize()
  E0 = e0.cpu().numpy()
  if keep:
    assert np.isnan(E0[-1]).all(), 'a row past the last was written'
  else:
    assert np.isnan(E0).all(), 'E0 was written without being asked for'
  out = [t.cpu().numpy() if t is not None else None for t in img + imgT]
  return E0[:-1] if keep else None, out, (rp, cp, rpT, cpT)


def embed_ref(e):
  c, W, b = e.cos.astype(np.float64), e.W.astype(np.float64), e.b.astype(np.float64)
  K = ceil_to(e.latent, 16)
  return np.maximum(c @ W + b, 0.0), (25 + K // 8) * U * (np.abs(c) @ np.abs(W) + np.abs(b))


def mul_rows(e):
  return e.mul[np.arange(e.M) // e.mul_div, :e.D]


EMBED_CASES = [   # M, latent, D, mul_div, mul_ld
    (1024, 16, 256, 8, 256), (1028, 64, 256, 33, 260), (1028, 128, 3136, 64, 3136), (2048, 128, 3136, 33, 3136),
    (4096, 64, 3136, 64, 3140), (4096, 16, 256, 33, 256), (2048, 16, 3136, 8, 3136), (1024, 128, 256, 64, 256),
    (1028, 16, 100, 8, 100)]


@pytest.mark.parametrize('M,latent,D,mul_div,mul_ld', EMBED_CASES)
def test_embed_packed(M, latent, D, mul_div, mul_ld):
  """E0 against float64 relu(cos W + b); the image pair against the kernel's own h and against float64; the transposed
  image bit for bit; the padding of both images zero and the ones row intact.  M = 1028 leaves 12 unwritten reduction
  columns in the transposed image, D = 100 4 in the plain one."""
  rs = np.random.RandomState(M + latent + D + mul_div)
  e = Embed(M, latent, D, mul_div, mul_ld, rs)
  E0, (hi, lo, hiT, loT), (rp, cp, rpT, cpT) = run_embed(e)
  want, bud = embed_ref(e)
  worst = within('E0', E0, want, bud, np.abs(want) + 1)
  zero_row = (e.cos == 0).all(1)
  assert zero_row.sum() == 4 and (E0[zero_row] == np.maximum(e.b, 0)).all(), 'relu(0 + b) is not exact'
  assert (E0[:, e.b == DENORM][zero_row] == DENORM).all(), 'relu let the smallest denormal bias through only inexactly'
  m = mul_rows(e)
  h = f32(E0 * m)
  idx = image_index(M, D, rp // 8)
  want_hi, want_lo = split(h)
  assert (bits(hi[idx]) == bits(want_hi)).all(), 'image hi is not rna(fl(E0 act3))'
  assert (bits(lo[idx]) == bits(want_lo)).all(), 'image lo is not rna(h - hi)'
  hw = want * m.astype(np.float64)
  worst = max(worst, within('hi + lo', hi[idx].astype(np.float64) + lo[idx], hw,
                            bud * np.abs(m) + 5 * U * np.abs(hw), np.abs(hw) + 1))
  idxT = image_index(D, M, rpT // 8)
  assert (bits(hiT[idxT]) == bits(hi[idx]).T).all(), 'the transposed image hi is not the image transposed'
  assert (bits(loT[idxT]) == bits(lo[idx]).T).all(), 'the transposed image lo is not the image transposed'
  ones = pk_index(D, np.arange(M), rpT // 8)
  assert (hiT[ones] == 1.0).all() and (bits(loT[ones]) == 0).all(), 'the ones row was overwritten'
  for name, flat, used in (('image', [hi, lo], [idx]), ('transposed image', [hiT, loT], [idxT, ones])):
    pad = np.ones(flat[0].size, bool)
    for u in used:
      pad[u.reshape(-1)] = False
    assert pad.sum() == flat[0].size - sum(u.size for u in used)
    for part in flat:
      assert (bits(part[pad]) == 0).all(), '%s padding was written' % name
  print('iqn embed packed M=%d latent=%d D=%d mul_div=%d: worst error / budget %.3f' % (M, latent, D, mul_div, worst))


def test_embed_packed_without_transposed_image():
  """The forward of the target network's applies: no transposed image and no E0, the same image bits."""
  rs = np.random.RandomState(5)
  e = Embed(1028, 64, 256, 33, 256, rs)
  _, full, _ = run_embed(e)
  _, bare, _ = run_embed(e, keep=False)
  for a, b in zip(full[:2], bare[:2]):
    assert (bits(a) == bits(b)).all()


# ---- preconditions --------------------------------------------------------------------------------------------------

def test_hooks_reject_shapes_outside_the_kernels():
  """Each hook returns DZ_EINVAL, and writes nothing, outside its kernel's preconditions: the value head's 18 actions
  and 1 to 3 applies, the packed Hadamard's N = 64 and D % 64 = 0, and EPI = 1's latent <= 128, M % 4 = D % 4 = 0."""
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  EINVAL = -1
  lib, s = _lib.lib, stream()
  x = nan(4 * 3200 * 64)
  p = x.data_ptr()
  assert lib.dz_test_iqn_hadamard_bwd(1, 2, 32, 256, p, p, p, p, p, p, 256, s) == EINVAL, 'packed N = 32'
  assert lib.dz_test_iqn_hadamard_bwd(1, 2, 64, 96, p, p, p, p, p, p, 128, s) == EINVAL, 'packed D % 64 != 0'
  assert lib.dz_test_iqn_hadamard_bwd(1, 2, 64, 256, p, p, p, p, p, p, 128, s) == EINVAL, 'image shorter than D'
  embed = lambda M, latent, D, mul_div, mul_ld: lib.dz_test_iqn_embed_packed(p, M, latent, p, D, p, p, mul_div, mul_ld,
                                                                             p, p, p, p, None, None, s)
  assert embed(1024, 144, 256, 8, 256) == EINVAL, 'latent > 128'
  assert embed(1026, 16, 256, 8, 256) == EINVAL, 'M % 4 != 0'
  assert embed(1024, 16, 258, 8, 258) == EINVAL, 'D % 4 != 0'
  assert embed(1024, 16, 256, 0, 256) == EINVAL, 'mul_div = 0'
  assert embed(1024, 16, 256, 8, 252) == EINVAL, 'mul_ld < D'
  one = (C.c_int32 * 3)(8, 8, 8)
  wide = dl.Learner(dl.NetworkSpec('iqn', 19, obs_shape=(44, 44, 4)), batch_size=4)
  assert lib.dz_test_iqn_head_fwd(wide._h, 1, one, ptrs([p]), ptrs([p]), ptrs([p]), s) == EINVAL, 'A = 19'
  assert lib.dz_test_iqn_head_dgrad(wide._h, 8, p, p, p, p, s) == EINVAL, 'A = 19'
  L = learner(6)
  four = ptrs([p] * 4)
  assert lib.dz_test_iqn_head_fwd(L._h, 4, (C.c_int32 * 4)(8, 8, 8, 8), four, four, four, s) == EINVAL, 'np = 4'
  assert lib.dz_test_iqn_head_fwd(L._h, 1, one, ptrs([p + 4]), ptrs([p]), ptrs([p]), s) == EINVAL, 'misaligned h1'
  torch.cuda.synchronize()
  assert np.isnan(x.cpu().numpy()).all(), 'a rejected call wrote its buffers'


# ---- the bars discriminate ------------------------------------------------------------------------------------------

def test_mutated_references_fail():
  """A plausibly wrong reference fails each comparison above on the kernels' real outputs, while the right one passes."""
  rs = np.random.RandomState(77)
  # cos: the argument formed in float64, or j instead of j + 1
  taus = cos_taus(64, rs)
  got = run_cos(taus, 128)
  want = np.cos(cos_arg(taus, 128).astype(np.float64))
  assert ratio(got, want, 2 * ulp32(want)) <= 1
  exact_arg = taus[:, None].astype(np.float64) * np.pi * np.arange(1, 129)
  assert ratio(got, np.cos(exact_arg), 2 * ulp32(want)) > 1, 'cos: float64 argument'
  shifted = np.cos(f32(taus[:, None] * f32(np.arange(0, 128, dtype=np.float32) * PI32)).astype(np.float64))
  assert ratio(got, shifted, 2 * ulp32(want)) > 1, 'cos: j pi tau'
  # value head: bias dropped, or apply 0's head for apply 1
  L = learner(6)
  heads = [Head(L, rs) for _ in range(2)]
  xs = [post_relu((512, 512), rs) for _ in range(2)]
  h1 = [dev(x) for x in xs]
  q = run_head_fwd(L, [512, 512], h1, [h.blob for h in heads])
  want, bud = head_ref(heads[1], xs[1])
  assert ratio(q[1], want, bud) <= 1
  assert ratio(q[1], want - heads[1].b, bud) > 1, 'head: bias dropped'
  assert ratio(q[1], head_ref(heads[0], xs[1])[0], bud) > 1, "head: apply 0's weights"
  # head input gradient: the mask on h1 >= 0
  x, dout = dgrad_inputs(6, rs)
  x, dout = x[:512], dout[:512]
  h1d, dd = dev(x), dev(dout)
  g = run_head_dgrad(L, 512, dd, heads[0].blob, h1d)
  want, bud = dgrad_ref(heads[0], dout)
  assert ratio(g, np.where(x > 0, want, 0.0), bud) <= 1
  assert ratio(g, np.where(x >= 0, want, 0.0), bud) > 1, 'dgrad: mask on h1 >= 0'
  # Hadamard: the mask on E >= 0, dfeat unmasked, and the dE image of the unpacked kernel one reduction column off
  G, E, F = hadamard_inputs(16, 64, 256, rs)
  dE, dfeat, _, _ = run_hadamard(False, G, E, F)
  dE_want, dfeat_want, S = hadamard_ref(G, E, F)
  assert (bits(dE) == bits(dE_want)).all() and ratio(dfeat, dfeat_want, 65 * U * S) <= 1
  assert (bits(dE) != bits(np.where(E >= 0, f32(G * F[:, None, :]), f32(0.0)))).any(), 'hadamard: mask on E >= 0'
  g64, e64 = G.astype(np.float64), E.astype(np.float64)
  assert ratio(dfeat, (g64 * e64).sum(1), 65 * U * S) > 1, 'hadamard: dfeat without the F > 0 mask'
  _, _, hi, _ = run_hadamard(True, G, E, F, 256)
  idx = image_index(256, 16 * 64, 32)
  want_hi = split(dE.transpose(2, 0, 1).reshape(256, -1))[0]
  assert (bits(hi[idx]) == bits(want_hi)).all()
  assert (bits(hi[idx]) != bits(np.roll(want_hi, 1, axis=1))).any(), 'packed hadamard: image one column off'
  # embedding epilogue: bias dropped, i % B instead of i / mul_div, the image one row off, the transpose not taken
  e = Embed(1028, 16, 256, 33, 256, rs)
  E0, (hi, lo, hiT, _), (rp, _, rpT, _) = run_embed(e)
  want, bud = embed_ref(e)
  assert ratio(E0, want, bud) <= 1
  c, W = e.cos.astype(np.float64), e.W.astype(np.float64)
  assert ratio(E0, np.maximum(c @ W, 0.0), bud) > 1, 'embed: bias dropped'
  idx = image_index(1028, 256, rp // 8)
  h = f32(E0 * mul_rows(e))
  assert (bits(hi[idx]) == bits(split(h)[0])).all()
  B = 1028 // 33
  wrong = f32(E0 * e.mul[np.arange(1028) % B, :256])
  assert (bits(hi[idx]) != bits(split(wrong)[0])).any(), 'embed: i % B for i / mul_div'
  assert (bits(hi[idx]) != bits(split(np.roll(h, 1, axis=0))[0])).any(), 'embed: image one row off'
  idxT = image_index(256, 1028, rpT // 8)
  assert (bits(hiT[idxT]) == bits(hi[idx]).T).all()
  assert (bits(hiT[image_index(256, 256, rpT // 8)]) != bits(hi[image_index(256, 256, rp // 8)])).any(), \
      'embed: transposed image not transposed'
