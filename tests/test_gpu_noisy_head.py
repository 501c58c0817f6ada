"""GPU: rainbow's noisy head kernels (DESIGN.md §7), forward and input gradient, against float64.

`dz_test_noisy_head_fwd` / `dz_test_noisy_head_bwd` run the learner's own launch functions (launch_noisy_head_fwd:
noisy_head_fwd_kernel, launch_noisy_head_bwd: noisy_head_bwd_kernel) with a rainbow learner's offsets and noise layout
on h1 streams, parameter blobs and noise applies given here.  The references restate the head in numpy float64 on the
same fp32 inputs: out_s = h1_s (mu_s + sigma_s . (eps_in eps_out^T)) + sigma_b eps_out, and dh1_s = [h1_s > 0]
dout_s (mu_s + sigma_s . (eps_in eps_out^T))^T through noise apply 0.

Budgets per element, u = 2^-24, S the sum of the magnitudes of the terms:
  forward   a formed weight rounds twice (eps_in * eps_out, the fmaf); a warp sums 64 products serially, the eight warp
            sums are added serially, then the sigma bias fmaf:  (64 + 8 + 3) u S
  backward  a lane sums ceil(N / 32) products serially, five butterfly levels add the lanes:  (ceil(N / 32) + 8) u S
Exact: the ReLU mask (h1 = +0, -0 give 0, the smallest denormal passes), the tf32 hi/lo pair of the kernel's own dh1,
a row's bits at every row count, and two launches' bits.
"""

import ctypes as C
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
ATOMS = 51
_LEARNERS = {}


def f32(x):
  return np.asarray(x, dtype=np.float32)


def dev(x):
  return torch.as_tensor(np.ascontiguousarray(x)).cuda()


def learner(obs):
  from dqn_zoo_b200 import learner as dl
  if obs not in _LEARNERS:
    _LEARNERS[obs] = dl.Learner(dl.NetworkSpec('rainbow', 6, obs_shape=(obs, obs, 4)), batch_size=32 if obs == 84 else 5)
  return _LEARNERS[obs]


@pytest.fixture(scope='module', autouse=True)
def _free_learners():
  yield
  _LEARNERS.clear()


def stream():
  return torch.cuda.current_stream().cuda_stream


def nan(*shape):
  return torch.full(shape, float('nan'), dtype=torch.float32, device='cuda')


def ptrs(ts):
  return (C.c_void_p * len(ts))(*[None if t is None else t.data_ptr() for t in ts])


def noise_offsets(L):
  """Offsets of the heads' eps_in / eps_out in one noise apply (a1i, a1o, a2i, a2o, v1i, v1o, v2i, v2o, each padded
  to 4 floats), checked against the library's stride."""
  D = L.tensors['adv1/mu/w'][1][0]
  A = L.net.num_actions
  r4 = lambda n: (n + 3) // 4 * 4
  a2i = r4(D) + 512
  a2o = a2i + 512
  v2i = a2o + r4(A * ATOMS) + r4(D) + 512
  v2o = v2i + 512
  assert v2o + r4(ATOMS) == L.noise_stride
  return a2i, a2o, v2i, v2o


class Head:
  """A parameter blob of learner L with random head weights: per stream (mu, sigma, mu_b or None, sigma_b)."""

  def __init__(self, L, rs):
    self.blob = torch.full((L.plan.param_count,), float('nan'), dtype=torch.float32, device='cuda')
    s = 1 / np.sqrt(512)
    self.p = {}
    for name, n in (('adv2', 6 * ATOMS), ('val2', ATOMS)):
      mu, sg = f32(rs.uniform(-s, s, (512, n))), f32(rs.uniform(0, 0.5 * s, (512, n)))
      sgb = f32(rs.uniform(0, 0.5 * s, n))
      mub = f32(rs.uniform(-s, s, n)) if name + '/mu/b' in L.tensors else None
      self.p[name] = (mu, sg, mub, sgb)
      for key, v in ((name + '/mu/w', mu), (name + '/sigma/w', sg), (name + '/mu/b', mub), (name + '/sigma/b', sgb)):
        if v is not None:
          L.view(self.blob, key).copy_(torch.as_tensor(v))


def h1_rows(rows, rs):
  """Post-ReLU activations with exact zeros of both signs and the smallest denormal among the positives."""
  x = f32(np.maximum(rs.standard_normal((rows, 512)), 0.0))
  x[rs.uniform(size=x.shape) < 0.1] = -0.0
  x[rs.uniform(size=x.shape) < 0.05] = np.float32(2.0 ** -149)
  return x


def noise_applies(L, n, rs):
  e = rs.standard_normal((n, L.noise_stride))
  return f32(np.sign(e) * np.sqrt(np.abs(e)))


def eps(L, noise, apply, s):
  a2i, a2o, v2i, v2o = noise_offsets(L)
  n = noise[apply].astype(np.float64)
  return (n[a2i:a2i + 512], n[a2o:a2o + 6 * ATOMS]) if s == 0 else (n[v2i:v2i + 512], n[v2o:v2o + ATOMS])


def weights(p, ei, eo):
  mu, sg = p[0].astype(np.float64), p[1].astype(np.float64)
  return mu + sg * np.outer(ei, eo), np.abs(mu) + sg * np.abs(np.outer(ei, eo))


def within(name, got, want, budget):
  got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
  assert np.isfinite(got).all(), (name, 'unwritten or non-finite element')
  ratio = float((np.abs(got - want) / (budget + 1e-30)).max())
  assert ratio <= 1.0, (name, ratio)
  return ratio


def run_fwd(L, rows, h1, blobs, noise_dev):
  from dqn_zoo_b200 import _lib
  outs = []
  for _ in blobs:
    outs += [nan(rows, 6 * ATOMS), nan(rows, ATOMS)]
  _lib.call('dz_test_noisy_head_fwd', L._h, rows, len(blobs), ptrs([t for pair in h1 for t in pair]),
            ptrs([b.blob for b in blobs]), C.c_void_p(noise_dev.data_ptr()), ptrs(outs), C.c_void_p(stream()))
  torch.cuda.synchronize()
  return [o.cpu().numpy() for o in outs]


@pytest.mark.parametrize('obs', [84, 44])
def test_noisy_head_forward(obs):
  """Three passes, online on two of them (one CTA group) and target on the third, at 1, 5 and 32 rows against float64;
  every row count gives the bits of the first rows of 32, and a second launch gives the same bits."""
  L = learner(obs)
  rs = np.random.RandomState(obs)
  online, target = Head(L, rs), Head(L, rs)
  noise = noise_applies(L, 3, rs)
  nd = dev(noise)
  xs = [[h1_rows(32, rs) for _ in range(2)] for _ in range(3)]
  blobs = [online, online, target]
  full = None
  worst = 0.0
  for rows in (32, 1, 5):
    h1 = [[dev(x[:rows]) for x in pair] for pair in xs]
    got = run_fwd(L, rows, h1, blobs, nd)
    if rows == 32:
      full = got
      again = run_fwd(L, rows, h1, blobs, nd)
      for a, b in zip(got, again):
        np.testing.assert_array_equal(a, b)
    for i, blob in enumerate(blobs):
      for s, name in enumerate(('adv2', 'val2')):
        p = blob.p[name]
        ei, eo = eps(L, noise, i, s)
        W, Wabs = weights(p, ei, eo)
        x = xs[i][s][:rows].astype(np.float64)
        want = x @ W + p[3].astype(np.float64) * eo
        S = np.abs(x) @ Wabs + np.abs(p[3].astype(np.float64) * eo)
        if p[2] is not None:
          want, S = want + p[2], S + np.abs(p[2].astype(np.float64))
        worst = max(worst, within('out pass %d %s rows %d' % (i, name, rows), got[2 * i + s], want, 75 * U * S))
        np.testing.assert_array_equal(got[2 * i + s], full[2 * i + s][:rows])
  print('noisy head fwd %dx%d: worst error / budget %.3f' % (obs, obs, worst))


def rna_tf32(x):
  """cvt.rna.tf32.f32 on finite float32: round to 10 mantissa bits, ties away from zero."""
  b = np.asarray(x, np.float32).view(np.uint32)
  return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def run_bwd(L, rows, dout, blob, noise_dev, h1, with_hilo):
  from dqn_zoo_b200 import _lib
  dh1 = [nan(rows, 512), nan(rows, 512)]
  hi = [nan(rows, 512), nan(rows, 512)] if with_hilo else None
  lo = [nan(rows, 512), nan(rows, 512)] if with_hilo else None
  _lib.call('dz_test_noisy_head_bwd', L._h, rows, ptrs(dout), C.c_void_p(blob.blob.data_ptr()),
            C.c_void_p(noise_dev.data_ptr()), ptrs(h1), ptrs(dh1), ptrs(hi) if hi else None, ptrs(lo) if lo else None,
            C.c_void_p(stream()))
  torch.cuda.synchronize()
  return [t.cpu().numpy() for t in dh1], None if hi is None else [t.cpu().numpy() for t in hi], \
      None if lo is None else [t.cpu().numpy() for t in lo]


@pytest.mark.parametrize('obs', [84, 44])
def test_noisy_head_input_gradient(obs):
  """dh1 of both streams at 1, 5 and 32 rows against float64 with the exact ReLU mask; the tf32 hi/lo pair is the
  split of dh1 bit for bit; every row count gives the bits of the first rows of 32; a second launch the same bits."""
  L = learner(obs)
  rs = np.random.RandomState(100 + obs)
  head = Head(L, rs)
  noise = noise_applies(L, 1, rs)
  nd = dev(noise)
  h1 = [h1_rows(32, rs) for _ in range(2)]
  dout = [f32(rs.standard_normal((32, 6 * ATOMS)) / 32), f32(rs.standard_normal((32, ATOMS)) / 32)]
  full = None
  worst = 0.0
  for rows in (32, 1, 5):
    args = ([dev(d[:rows]) for d in dout], head, nd, [dev(h[:rows]) for h in h1])
    dh1, hi, lo = run_bwd(L, rows, *args, True)
    if rows == 32:
      full = dh1
      again, _, _ = run_bwd(L, rows, *args, False)
      for a, b in zip(dh1, again):
        np.testing.assert_array_equal(a, b)
    for s, name in enumerate(('adv2', 'val2')):
      ei, eo = eps(L, noise, 0, s)
      W, Wabs = weights(head.p[name], ei, eo)
      g = dout[s][:rows].astype(np.float64)
      mask = h1[s][:rows] > 0
      want = np.where(mask, g @ W.T, 0.0)
      S = np.abs(g) @ Wabs.T
      n = W.shape[1]
      worst = max(worst, within('dh1 %s rows %d' % (name, rows), dh1[s], want, ((n + 31) // 32 + 8) * U * S))
      assert (dh1[s][~mask] == 0).all() and not np.signbit(dh1[s][~mask]).any()
      np.testing.assert_array_equal(hi[s], rna_tf32(dh1[s]))
      np.testing.assert_array_equal(lo[s], rna_tf32(dh1[s] - hi[s]))
      np.testing.assert_array_equal(dh1[s], full[s][:rows])
  print('noisy head bwd %dx%d: worst error / budget %.3f' % (obs, obs, worst))


# ---- the learner step ------------------------------------------------------------------------------------------------

def _rainbow_agent(graph, seed=3):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rep = dr.PrioritizedTransitionReplay(512, dr.Transition(None, None, None, None, None), 0.5, lambda t: 0.4, 1e-3, True,
                                       np.random.RandomState(seed))
  agent = ag.Rainbow(support=np.linspace(-10, 10, ATOMS), preprocessor=None, sample_network_input=None,
                     network=dl.NetworkSpec('rainbow', 6), optimizer=None,
                     transition_accumulator=dr.NStepTransitionAccumulator(3), replay=rep, batch_size=32,
                     min_replay_capacity_fraction=1.0, learn_period=4, target_network_update_period=16,
                     rng_key=[0, seed], use_cuda_graph=graph)
  dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6)
  return agent


def test_rainbow_step_graph_is_bit_identical_to_eager():
  runs = []
  for graph in (True, False, False):
    agent = _rainbow_agent(graph)
    for _ in range(6):
      agent.learn()
    torch.cuda.synchronize()
    runs.append({n: getattr(agent.learner, n).clone() for n in ('online', 'target', 'opt_state', 'loss', 'per_example',
                                                                  'priorities')})
  for other in runs[1:]:
    for name, t in runs[0].items():
      assert torch.equal(t, other[name]), name


def test_rainbow_step_runs_the_head_without_split_finishes():
  """One eager rainbow step launches the head forward and its input gradient once each, under their own geometries,
  and neither split finish."""
  from dqn_zoo_b200 import _lib
  agent = _rainbow_agent(False)
  for _ in range(2):
    agent.learn()
  torch.cuda.synchronize()
  _lib.call('dz_profile_begin')
  agent.learn()
  buf = C.create_string_buffer(1 << 16)
  _lib.call('dz_profile_end', buf, len(buf))
  prof = json.loads(buf.value.decode())
  assert 'finish_nn_kernel' not in prof and 'finish_nt_kernel' not in prof, sorted(prof)
  geo = {k: tuple(v[2:5]) for k, v in prof.items()}
  assert geo['noisy2_fwd'] == (46, 2, 256) and geo['noisy2_dgrad'] == (128, 1, 256), geo
  for k, g in geo.items():
    if k not in ('noisy2_fwd', 'noisy2_dgrad'):
      assert g not in (geo['noisy2_fwd'], geo['noisy2_dgrad']), (k, g)
