"""GPU: FQF's fraction, loss and acting kernels (DESIGN.md §15) kernel by kernel against float64.

`dz_test_fraction_forward` runs the learner's launch_fraction_forward (fraction_forward_kernel) on features and a
parameter blob given here, `dz_test_loss_fqf` runs launch_loss with fqf's fraction buffers (loss_fqf_kernel, then
loss_mean_kernel) and `dz_test_q_values_fqf` launch_q_values with the interval weights (q_values_fqf_kernel,
act_select_kernel).  No network runs, so the inputs can sit where these kernels make discrete choices: saturated
softmaxes (tied and zero-width fractions, a prefix sum that rounds above 1), tied weighted selections, quantile
differences of exactly 0 and +-kappa, importance weight 0 and terminal transitions.  The references are
oracle/fqf_oracle.py's `proposal`, `head_loss`, `tau_gradient` and `dlogits_of` in float64 on the same fp32 inputs.

Exact: the fraction invariant 0 = tau_0 <= ... <= tau_N = 1, w_i = tau_{i+1} - tau_i >= 0 and tau_i <= tau_hat_i <=
tau_{i+1}; the pass1 / pass2 layout; a row's bits at every E and position; the selected and acting actions; dlogits
exactly 0 where q_k = 0 or the importance weight is 0, and dout exactly 0 off a_tm1.  Continuous outputs get a float32
budget per element, with u = 2^-24:
  logit     l_c = sum_k x_k W_kc + b_c: 8 warps each add D/8 terms with fmaf, the 8 partials are added serially and the
            bias last: e_l = (D/8 + 9) u (sum_k |x_k W_kc| + |b_c|).
  fractions the host twin's budget of tests/test_oracle_fqf.py (R = max |l - max l|) with the logit errors on top: a
            softmax moves by at most 2 max_c e_l relative, so q: ((N + 4 + 2R) u + 2 E) q + 2^-147 (E = max_c e_l);
            tau: T = (2N + 4 + 2R) u + 2E + N 2^-147; tau_hat: T + u; w: 2T + u.
  loss      the quantile tail of tests/test_gpu_loss_kernels.py (budget_quantile) at tau = tau_hat, Nt = N.
  dlogits   the host twin's dlogits budget with exact q inputs: E_dq = (N + 2) u sum_i G_i, |dD| <= N u sum_j q_j |dq_j|
            + sum_j q_j E_dq, then cot (q_k (E_dq + |dD|) + 2 u q_k |dq_k - D|) + u |dlogit_k| for cot = w_b / B.
  q-values  Q = sum_i w_i Z_i (fmaf chain): (N + 1) u sum_i |w_i Z_i|.
Every budget carries 1e-12 of its operands for the oracle's own float64 rounding.  `-s` prints worst error / budget.
"""

import ctypes as C
import json
import os

import numpy as np
import pytest
import torch

from oracle import fqf_oracle as fo
import test_gpu_loss_kernels as lk
from test_oracle_fqf import assert_fraction_invariant

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'fqf_hand_vectors.json')
f32, dev, within = lk.f32, lk.dev, lk.within


def nan(*shape):
  return torch.full(shape, float('nan'), dtype=torch.float32, device='cuda')


def stream():
  return torch.cuda.current_stream().cuda_stream


_LEARNERS = {}


def learner(hw, N, A=4):
  from dqn_zoo_b200 import learner as dl
  key = (hw, N, A)
  if key not in _LEARNERS:
    _LEARNERS[key] = dl.Learner(dl.NetworkSpec('fqf', A, obs_shape=(hw, hw, 4), num_fractions=N), batch_size=4)
  return _LEARNERS[key]


@pytest.fixture(scope='module', autouse=True)
def _free_learners():
  yield
  _LEARNERS.clear()


# ---- fraction_forward_kernel ------------------------------------------------------------------------------------------

def patterns(N):
  """Logit patterns over N fractions, each exact in float32: near-uniform, a saturated middle fraction (a tau tie), a
  saturated last fraction at -30 (the prefix sum of the rest rounds above 1) and at -90, a saturated first fraction, all
  mass on one fraction, and logits of magnitude 80 and more."""
  p = []
  p.append(np.zeros(N))
  m = np.zeros(N); m[N // 2] = -90.0; p.append(m)
  s = np.zeros(N); s[-1] = -30.0; p.append(s)
  s = np.zeros(N); s[-1] = -90.0; p.append(s)
  f = np.zeros(N); f[0] = -90.0; p.append(f)
  o = np.full(N, -100.0); o[N // 3] = 0.0; p.append(o)
  p.append(np.round(np.linspace(-85.0, 85.0, N)))
  p.append(np.where(np.arange(N) % 2 == 0, 80.0, -81.0))
  return np.stack(p)


def fraction_inputs(N, D, E, rs):
  """features [E][D] and the fraction layer W [D][N], b [N]: features 0..P-1 are one-hot pattern selectors whose rows
  of W hold the patterns, the rest are torso-like features >= 0 with W at the default init scale.  Odd rows have no
  torso part, so their logits are exactly pattern + b."""
  pat = patterns(N)
  P = len(pat)
  assert D > P
  W = np.zeros((D, N), np.float32)
  W[:P] = pat
  W[P:] = rs.uniform(-0.01, 0.01, (D - P, N)) / np.sqrt(D)
  b = f32(np.round(rs.uniform(-0.5, 0.5, N) * 64) / 64)
  x = f32(rs.uniform(0.0, 2.0, (E, D)))
  x[:, :P] = 0.0
  x[np.arange(E), np.arange(E) % P] = 1.0
  x[1::2, P:] = 0.0
  return x, W, b


def blob_with(L, W, b):
  blob = torch.full((L.plan.param_count,), float('nan'), dtype=torch.float32, device='cuda')
  L.view(blob, 'fraction/w').copy_(torch.as_tensor(W))
  L.view(blob, 'fraction/b').copy_(torch.as_tensor(b))
  return blob


def run_fractions(L, feats, blob, outputs=('tau', 'tau_hat', 'w', 'q', 'pass1', 'pass2')):
  """Every output of dz_test_fraction_forward, NaN-filled with one spare row past the last; outputs not named are NULL."""
  from dqn_zoo_b200 import _lib
  napp, (E, _) = len(feats), feats[0].shape
  N = L.net.num_fractions
  x = [dev(f) for f in feats]
  o = {k: [nan(E + 1, N + (k == 'tau')) for _ in range(napp)] for k in ('tau', 'tau_hat', 'w', 'q') if k in outputs}
  p1 = nan(E + 1, N) if 'pass1' in outputs else None
  p2 = nan(E + 1, 2 * N) if 'pass2' in outputs else None
  arr = lambda k: (C.c_void_p * 2)(*([t.data_ptr() for t in o[k]] + [None] * (2 - napp))) if k in o else None
  _lib.call('dz_test_fraction_forward', L._h, E, napp, (C.c_void_p * 2)(*([t.data_ptr() for t in x] + [None] * (2 - napp))),
            blob.data_ptr(), arr('tau'), arr('tau_hat'), arr('w'), arr('q'), None if p1 is None else p1.data_ptr(),
            None if p2 is None else p2.data_ptr(), stream())
  torch.cuda.synchronize()
  got = {k: [t.cpu().numpy() for t in v] for k, v in o.items()}
  if p1 is not None:
    got['pass1'] = p1.cpu().numpy()
  if p2 is not None:
    got['pass2'] = p2.cpu().numpy()
  return got


def check_fractions(got, x, W, b, app, N):
  """Compares application `app` of `got` with the oracle's proposal of x W + b; returns the worst error / budget."""
  E, D = x.shape
  x64, W64, b64 = x.astype(np.float64), W.astype(np.float64), b.astype(np.float64)
  logits = x64 @ W64 + b64
  e_l = ((D / 8 + 9) * U * (np.abs(x64) @ np.abs(W64) + np.abs(b64))).max(-1, keepdims=True)
  p = fo.proposal(torch.tensor(logits))
  R = np.abs(logits - logits.max(-1, keepdims=True)).max(-1, keepdims=True)
  q = p['q'].numpy()
  T = (2 * N + 4 + 2 * R) * U + 2 * e_l + N * 2.0 ** -147
  budgets = {'q': ((N + 4 + 2 * R) * U + 2 * e_l) * q + 2.0 ** -147, 'tau': T, 'tau_hat': T + U, 'w': 2 * T + U}
  worst = 0.0
  for k, bud in budgets.items():
    g = got[k][app]
    assert np.isnan(g[E]).all(), (k, 'a row past the last was written')
    want = p[k].numpy()
    worst = max(worst, within('%s app %d' % (k, app), g[:E], want, np.broadcast_to(bud, want.shape), np.abs(want) + 1))
  assert_fraction_invariant(got['tau'][app][:E], got['tau_hat'][app][:E], got['w'][app][:E], N)
  assert (got['q'][app][:E] >= 0).all()
  return worst


@pytest.mark.parametrize('hw', [84, 44])
@pytest.mark.parametrize('N', [2, 3, 32, 33, 127, 128])
def test_fraction_forward_against_float64(N, hw):
  """One and two applications at E = 1024 over every logit pattern, then E in {1, 7, 33} on rows drawn from the same
  features at other positions: every row has the bits it has at E = 1024."""
  L = learner(hw, N)
  D = L.tensors['fraction/w'][1][0]
  rs = np.random.RandomState(N * 7 + hw)
  x0, W, b = fraction_inputs(N, D, 1024, rs)
  x1 = x0[rs.permutation(1024)]
  x1[:, len(patterns(N)):] *= 0.5
  blob = blob_with(L, W, b)
  full = run_fractions(L, [x0, x1], blob)
  worst = max(check_fractions(full, x0, W, b, 0, N), check_fractions(full, x1, W, b, 1, N))
  # the learner's pass inputs: pass1 = tau_1..tau_N of application 0, pass2 = [tau_hat of 1 | tau_hat of 0]
  np.testing.assert_array_equal(full['pass1'][:1024], full['tau'][0][:1024, 1:])
  np.testing.assert_array_equal(full['pass2'][:1024, :N], full['tau_hat'][1][:1024])
  np.testing.assert_array_equal(full['pass2'][:1024, N:], full['tau_hat'][0][:1024])
  assert np.isnan(full['pass1'][1024]).all() and np.isnan(full['pass2'][1024]).all()
  # a saturated middle fraction closes its interval: tau ties and the weight is exactly 0
  mid = np.arange(1024) % len(patterns(N)) == 1
  if N >= 3:
    assert (full['w'][0][:1024][mid, N // 2] == 0).all()
  for E in (1, 7, 33):
    rows = rs.choice(1024, E, replace=False)
    one = run_fractions(L, [x0[rows]], blob)
    for k in ('tau', 'tau_hat', 'w', 'q'):
      np.testing.assert_array_equal(one[k][0][:E], full[k][0][rows], err_msg='%s E=%d' % (k, E))
      assert np.isnan(one[k][0][E]).all()
    np.testing.assert_array_equal(one['pass1'][:E], full['pass1'][rows])
    np.testing.assert_array_equal(one['pass2'][:E, N:], full['pass2'][rows, N:])
    assert np.isnan(one['pass2'][:E + 1, :N]).all()     # one application writes only its own half
  # NULL outputs: what is given has the same bits, nothing else is needed
  part = run_fractions(L, [x0, x1], blob, outputs=('tau_hat', 'pass2'))
  np.testing.assert_array_equal(part['tau_hat'][1], full['tau_hat'][1])
  np.testing.assert_array_equal(part['pass2'], full['pass2'])
  print('fraction_forward N=%d hw=%d: worst error / budget %.3f' % (N, hw, worst))


@pytest.mark.parametrize('N', [11, 19, 27, 31])
def test_saturated_last_fraction_stays_inside_0_1_on_the_device(N):
  """Logits (0, ..., 0, -30): the device's q_0..q_{N-2} add up (serially in float32) to more than 1, and the kernel's
  fractions still end at exactly 1 with a zero last weight, the same bits as the host twin."""
  from dqn_zoo_b200 import _lib
  L = learner(44, N)
  D = L.tensors['fraction/w'][1][0]
  lg = np.zeros(N, np.float32)
  lg[-1] = -30.0
  W = np.zeros((D, N), np.float32)
  W[0] = lg
  x = np.zeros((3, D), np.float32)
  x[:, 0] = 1.0
  got = run_fractions(L, [x], blob_with(L, W, np.zeros(N, np.float32)))
  q = got['q'][0][:3]
  s = np.float32(0)
  for k in range(N - 1):
    s = np.float32(s + q[0, k])
  assert s > 1, 'the device no longer overshoots at N=%d: %r' % (N, s)
  assert_fraction_invariant(got['tau'][0][:3], got['tau_hat'][0][:3], got['w'][0][:3], N)
  assert (got['tau'][0][:3, N - 1] == 1).all() and (got['w'][0][:3, N - 1] == 0).all()
  out = np.zeros(5 * N + 1, np.float32)
  z = np.zeros(N, np.float32)
  _lib.call('dz_test_fqf_example', lg.ctypes.data, z.ctypes.data, z.ctypes.data, N, 1.0, out.ctypes.data)
  np.testing.assert_array_equal(got['tau'][0][0], out[N:2 * N + 1])
  np.testing.assert_array_equal(got['tau_hat'][0][0], out[2 * N + 1:3 * N + 1])
  print('fqf N=%d: device prefix sum of q_0..q_%d = %r, tau_%d = 1' % (N, N - 2, float(s), N - 1))


# ---- loss_fqf_kernel --------------------------------------------------------------------------------------------------

class FqfCase:
  """One fqf loss call: heads (out0 [B][N][A], ftau [B][N-1][A] at tau_1..tau_{N-1}, zsel, ztgt [B][N][A]), tau_hat,
  w_t, q_tm1 [B][N], the batch and kappa."""

  def __init__(self, out0, ftau, zsel, ztgt, a, r, d, tau_hat, w_t, q_tm1, w=None, kappa=1.0, name=''):
    self.out0, self.ftau, self.zsel, self.ztgt = f32(out0), f32(ftau), f32(zsel), f32(ztgt)
    self.B, self.N, self.A = self.out0.shape
    self.kind, self.a, self.r, self.d = 'fqf', np.asarray(a, np.int32), f32(r), f32(d)
    self.taus, self.w_t, self.q_tm1 = f32(tau_hat), f32(w_t), f32(q_tm1)
    self.w = None if w is None else f32(w)
    self.kappa, self.name = kappa, name

  def config(self):
    from dqn_zoo_b200 import _lib
    c = _lib.LearnerConfig(huber_param=self.kappa)
    c.kind = _lib.AGENT_KINDS['fqf']
    c.num_actions, c.num_atoms, c.num_quantiles, c.latent_dim = self.A, 51, 1, 64
    c.tau_samples_s_tm1 = c.tau_samples_policy = c.tau_samples_s_t = 1
    c.num_fractions, c.batch = self.N, self.B
    return c


def run_loss_device(case):
  from dqn_zoo_b200 import _lib
  B, N, A = case.B, case.N, case.A
  out1 = np.full((B, N, A), np.nan, np.float32)   # the last row, tau_N = 1, is padding no term may read
  out1[:, :N - 1] = case.ftau
  heads = [dev(case.out0), dev(out1), dev(np.concatenate([case.zsel, case.ztgt], axis=1))]
  keep = [dev(x) for x in (case.a, case.r, case.d, case.taus, case.w_t, case.q_tm1)]
  wt = None if case.w is None else dev(case.w)
  o = dict(dout=nan(B + 1, N, A), per_example=nan(B + 1), loss_terms=nan(B + 1), loss=nan(1), dlogits=nan(B + 1, N))
  _lib.call('dz_test_loss_fqf', C.byref(case.config()), B, (C.c_void_p * 3)(*[t.data_ptr() for t in heads]),
            *[t.data_ptr() for t in keep[:3]], None if wt is None else wt.data_ptr(), *[t.data_ptr() for t in keep[3:]],
            o['dout'].data_ptr(), o['dlogits'].data_ptr(), o['per_example'].data_ptr(), o['loss_terms'].data_ptr(),
            o['loss'].data_ptr(), stream())
  torch.cuda.synchronize()
  got = {k: v.cpu().numpy().astype(np.float64) for k, v in o.items()}
  for k in ('dout', 'per_example', 'loss_terms', 'dlogits'):
    assert np.isnan(got[k][B]).all(), (k, 'a row past the last was written')
    got[k] = got[k][:B]
  return got


def dlogits_budget(case, cot):
  """The module docstring's dlogits budget and the float64 dlogits, per element [B, N]."""
  rows = np.arange(case.B)
  ft = np.concatenate([np.zeros((case.B, 1)), case.ftau[rows, :, case.a].astype(np.float64)], axis=1)   # F(tau_i)
  fh = case.out0[rows, :, case.a].astype(np.float64)
  q = case.q_tm1.astype(np.float64)
  g = fo.tau_gradient(torch.tensor(ft[:, 1:]), torch.tensor(fh))
  dl = fo.dlogits_of(g, torch.tensor(q), torch.tensor(cot)).numpy()
  G = 2 * np.abs(ft[:, 1:]) + np.abs(fh[:, 1:]) + np.abs(fh[:, :-1])
  gg = np.concatenate([np.zeros((case.B, 1)), g.numpy()], axis=1)
  dq = np.cumsum(gg[:, ::-1], axis=1)[:, ::-1] - gg
  D = (q * dq).sum(1, keepdims=True)
  e_dq = (case.N + 2) * U * G.sum(1, keepdims=True)
  e_D = case.N * U * (q * np.abs(dq)).sum(1, keepdims=True) + (q * e_dq).sum(1, keepdims=True)
  bud = cot[:, None] * (q * (e_dq + e_D) + 2 * U * q * np.abs(dq - D)) + U * np.abs(dl) + 1e-45
  return dl, bud


def check_loss(case):
  got = run_loss_device(case)
  B, N, A = case.B, case.N, case.A
  rows = np.arange(B)
  t = lambda x: torch.tensor(np.asarray(x, np.float64))
  _, aux = fo.head_loss((t(case.out0), t(case.ftau), t(case.zsel), t(case.ztgt)), case.a, case.r, case.d, t(case.taus),
                        t(case.w_t), None if case.w is None else t(case.w), huber_param=case.kappa)
  w = np.ones(B) if case.w is None else case.w.astype(np.float64)
  bud = lk.budget_quantile(case, aux)
  ratios = {}
  dout = got['dout']
  mask = np.zeros(dout.shape, dtype=bool)
  mask[rows, :, case.a] = True
  assert (dout[~mask] == 0).all(), 'non-zero gradient off a_tm1'
  ratios['dout'] = within('dout', dout[rows, :, case.a], bud['g_value'], bud['g'], np.abs(bud['g_value']) + 1)
  loss = aux['losses'].numpy()
  ratios['per_example'] = within('loss', got['per_example'], loss, bud['per_example'], np.abs(loss) + 1)
  terms = w * loss
  ratios['loss_terms'] = within('loss_terms', got['loss_terms'], terms, bud['term'], np.abs(terms) + 1)
  e_mean = (bud['term'].sum() + (B + 1) * U * np.abs(terms).sum()) / B
  ratios['loss'] = within('loss', got['loss'][0], terms.mean(), e_mean, np.abs(terms).mean() + 1)
  cot = (w.astype(np.float32) / np.float32(B)).astype(np.float64)
  dl, e_dl = dlogits_budget(case, cot)
  ratios['dlogits'] = within('dlogits', got['dlogits'], dl, e_dl, np.abs(dl) + 1)
  assert (got['dlogits'][case.q_tm1 == 0] == 0).all(), 'a zero-width interval passed a gradient'
  zero_w = w == 0
  assert (got['dlogits'][zero_w] == 0).all() and (dout[zero_w] == 0).all(), 'importance weight 0 passed a gradient'
  print('fqf %-34s %s' % (case.name, ' '.join('%s %.3f' % kv for kv in sorted(ratios.items()))))
  return got, aux


def proposal_f32(logits):
  p = fo.proposal(torch.tensor(np.asarray(logits, np.float64)))
  return f32(p['tau_hat'].numpy()), f32(p['w'].numpy()), f32(p['q'].numpy())


def random_loss_case(B, A, N, rs, kappa=1.0, weights=False, name=''):
  g = lambda *shape: f32(rs.standard_normal(shape))
  hat, _, q = proposal_f32(rs.standard_normal((B, N)))
  _, w_t, _ = proposal_f32(rs.standard_normal((B, N)))
  return FqfCase(np.sort(g(B, N, A), axis=1), np.sort(g(B, N - 1, A), axis=1), g(B, N, A), g(B, N, A),
                 rs.randint(0, A, B), rs.choice([-1.0, 0.0, 1.0, 0.37], B), rs.choice([0.0, 0.99, 1.0], B), hat, w_t, q,
                 rs.uniform(0.1, 1.0, B) if weights else None, kappa=kappa, name=name)


@pytest.mark.parametrize('B,A,N', [(1, 1, 2), (5, 2, 32), (32, 18, 128), (1024, 64, 32), (256, 2, 128), (5, 64, 2)])
def test_fqf_loss_random_heads(B, A, N):
  rs = np.random.RandomState(B + A + N)
  check_loss(random_loss_case(B, A, N, rs, weights=B > 1, name='B=%d A=%d N=%d' % (B, A, N)))


def test_fqf_loss_selection_ties_and_weights_against_the_mean():
  """Rows 0-1: actions 0..2 have identical Z columns but different target columns, so only the first may win.  Row 2: the
  interval weights pick action 1 where the unweighted mean picks action 0."""
  N, A = 4, 3
  zsel = np.zeros((3, N, A), np.float32)
  zsel[0] = 2.0
  zsel[1, :, :] = np.array([1.0, -3.0, 0.5, 7.0])[:, None]
  zsel[2, :, 0] = [0.0, 0.0, 0.0, 12.0]     # mean 3, weighted 1.5
  zsel[2, :, 1] = 2.0                          # mean 2, weighted 2
  zsel[2, :, 2] = -1.0
  ztgt = np.zeros((3, N, A), np.float32)
  ztgt[:, :, 1] = 50.0
  ztgt[:, :, 2] = -50.0
  w_t = f32([[0.25] * 4, [0.25] * 4, [0.5, 0.25, 0.125, 0.125]])
  hat = f32([[0.125, 0.375, 0.625, 0.875]] * 3)
  rs = np.random.RandomState(5)
  case = FqfCase(np.sort(f32(rs.standard_normal((3, N, A))), axis=1), f32(rs.standard_normal((3, N - 1, A))), zsel, ztgt,
                 [0, 1, 2], [0.5, 0.5, 0.5], [1.0, 1.0, 1.0], hat, w_t, w_t, name='selection ties')
  _, aux = check_loss(case)
  assert aux['a_star'].tolist() == [0, 0, 1]


@pytest.mark.parametrize('kappa', [0.0, 0.5, 1.0, 3.0])
def test_fqf_loss_differences_on_zero_and_kappa_with_zero_width_intervals_and_weights(kappa):
  """r = 0, discount 1: the targets are the target quantiles exactly, and the online quantiles sit at 0 and +-kappa from
  them; tau_hat and the fractions come from the test, with q_k = 0 (zero-width intervals) in some rows and importance
  weight 0 in one; row 3 is terminal."""
  N, A, B = 8, 3, 6
  ztgt = np.zeros((B, N, A), np.float32)
  ztgt[:, :, 0] = np.arange(N) * 0.5
  offsets = np.array([0.0, kappa, -kappa, 0.0, kappa, -kappa, 0.0, 2 * kappa + 0.25], np.float32)
  out0 = np.zeros((B, N, A), np.float32)
  out0[:, :, 0] = ztgt[:, :, 0] + offsets[None, :]
  out0[:, :, 1] = 3.0
  ftau = np.broadcast_to(np.arange(1, N, dtype=np.float32)[None, :, None] * 0.25, (B, N - 1, A))
  zsel = np.zeros((B, N, A), np.float32)
  zsel[:, :, 0] = 1.0                        # action 0 is selected
  hat = np.tile(((np.arange(N) + 0.5) / N).astype(np.float32), (B, 1))
  q = np.tile(np.full(N, 1.0 / N, np.float32), (B, 1))
  q[1] = 0.0; q[1, 2] = 0.5; q[1, 5] = 0.5   # six zero-width intervals
  q[4] = 0.0; q[4, 0] = 1.0
  w = f32([1.0, 0.5, 0.0, 1.0, 0.25, 1.0])
  d = f32([1.0, 1.0, 1.0, 0.0, 1.0, 1.0])
  case = FqfCase(out0, ftau, zsel, ztgt, [0, 0, 0, 0, 1, 0], np.zeros(B), d, hat, np.full((B, N), 1.0 / N), q, w,
                 kappa=kappa, name='kink kappa=%g' % kappa)
  got, _ = check_loss(case)
  assert (got['dlogits'][2] == 0).all() and (got['dout'][2] == 0).all()
  assert (got['dlogits'][1][q[1] == 0] == 0).all()


def _hand_cases():
  with open(GOLDEN) as f:
    return json.load(f)['cases']


@pytest.mark.parametrize('case', _hand_cases(), ids=lambda c: c['name'])
def test_fqf_hand_vectors_through_the_device_kernels(case):
  """Each hand case through loss_fqf_kernel (against its hand dlogits and the oracle) and q_values_fqf_kernel / the
  acting selection (against its hand a*)."""
  N, A = len(case['logits']), len(case['zsel'][0])
  F_hat = f32(case['F_hat'])
  out0 = np.repeat(F_hat[None, :, None], A, axis=2)
  ftau = np.repeat(f32(case['F_tau'][1:])[None, :, None], A, axis=2)
  c = FqfCase(out0, ftau, f32(case['zsel'])[None], f32(case['ztgt'])[None], [0], [case['r_t']], [case['discount_t']],
              f32(case['tau_hat'])[None], f32(case['w'])[None], f32(case['q'])[None], name='hand ' + case['name'])
  got, aux = check_loss(c)
  assert int(aux['a_star'][0]) == case['a_star']
  np.testing.assert_allclose(got['dlogits'][0], case['dlogits'], rtol=0, atol=2e-6)
  q, act = q_values_fqf(f32(case['zsel'])[None], f32(case['w'])[None])
  assert act[0] == case['a_star']


# ---- q_values_fqf_kernel and act_select_kernel --------------------------------------------------------------------------

def q_values_fqf(out, w, explore=None, eps=0.0):
  from dqn_zoo_b200 import _lib
  E, N, A = out.shape
  c = FqfCase(np.zeros((1, N, A)), np.zeros((1, N - 1, A)), np.zeros((1, N, A)), np.zeros((1, N, A)), [0], [0], [0],
              np.zeros((1, N)), np.zeros((1, N)), np.zeros((1, N))).config()
  o, wd = dev(f32(out)), dev(f32(w))
  ex = None if explore is None else dev(f32(explore))
  q = nan(E + 1, A)
  act = torch.full((E + 1,), -1, dtype=torch.int32, device='cuda')
  _lib.call('dz_test_q_values_fqf', C.byref(c), E, o.data_ptr(), wd.data_ptr(), None if ex is None else ex.data_ptr(),
            float(eps), q.data_ptr(), act.data_ptr(), stream())
  torch.cuda.synchronize()
  q, act = q.cpu().numpy().astype(np.float64), act.cpu().numpy()
  assert np.isnan(q[E]).all() and act[E] == -1
  return q[:E], act[:E]


@pytest.mark.parametrize('E,N,A', [(1, 2, 1), (7, 32, 18), (1024, 128, 6), (33, 3, 64)])
def test_fqf_q_values_and_acting(E, N, A):
  """Random quantiles and proposals: q within budget, the greedy action the first maximum of the device's q; rows with
  tied weighted q-values (a duplicated column) take the first; an explore uniform exactly at epsilon is greedy and one
  next to 1 takes the last action."""
  rs = np.random.RandomState(E + N + A)
  z = f32(rs.standard_normal((E, N, A)))
  _, w, _ = proposal_f32(rs.standard_normal((E, N)))
  if A > 1:
    z[::2, :, A - 1] = z[::2, :, 0]          # tie the last action with the first
    z[1::2, :, 1] = z[1::2, :, 0] + 0.0      # tie action 1 with action 0
  q, act = q_values_fqf(z, w)
  want = (w.astype(np.float64)[:, :, None] * z.astype(np.float64)).sum(1)
  e = (N + 1) * U * (np.abs(w.astype(np.float64))[:, :, None] * np.abs(z.astype(np.float64))).sum(1)
  ratio = within('q fqf', q, want, e, np.abs(want) + 1)
  np.testing.assert_array_equal(act, np.argmax(q, axis=1))
  if A > 1:
    assert (q[::2, A - 1] == q[::2, 0]).all() and (q[1::2, 1] == q[1::2, 0]).all()
    assert (act[::2] != A - 1).all() or A == 1
  below_one = float(np.nextafter(np.float32(1), np.float32(0)))
  eps = 0.25
  u0 = np.where(np.arange(E) % 3 == 0, eps, np.where(np.arange(E) % 3 == 1, 0.0, 0.75))
  u1 = np.full(E, below_one)
  _, act_e = q_values_fqf(z, w, explore=np.stack([u0, u1]), eps=eps)
  np.testing.assert_array_equal(act_e, np.where(f32(u0) < np.float32(eps), A - 1, act))
  print('fqf q-values E=%d N=%d A=%d: error / budget %.3f' % (E, N, A, ratio))
