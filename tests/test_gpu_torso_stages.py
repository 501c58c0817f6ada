"""GPU: every launch of the learner's backward between the head and the optimizer, element by element, against float64
references computed from the device's own inputs to that launch (oracle/stage_oracle.py).

After one update without the optimizer step, the device's activations act1..3 (with their tf32 lo images on the
tensor-core torso), fc1's input gradients dh1, the conv input gradients dact1..3 and the frames are read back.  Each
stage's reference takes exactly those inputs, so a bar measures that launch's arithmetic alone and no ReLU can flip:
  dact3       (sum over fc1's streams of dh1_s W1_s^T) . [act3 > 0]; IQN's network: the Hadamard backward of the
              device's dhi (itself checked against dh1 W1^T) through the embedding E0, or both as one stage where
              the unpacked Hadamard backward writes the embedding's gradient over dhi
  dact2/1     conv3 / conv2 transpose of dact3 / dact2, masked by [act2 > 0] / [act1 > 0]
  dW, db      fc1 (mu and sigma of a noisy layer), conv3, conv2 and conv1 (input u8 / 255) from the activations and
              the input gradients, split-K partials and bias chunks summed by the finish kernels

Bars, u = 2^-24, S the stage's magnitude scale (sum |a| |b| over the K terms of an element):
  hard         |got - ref| <= tau_K S + 2^-126 for every element.
               fp32 FMA: each product is exact, or formed from operands rounded at most three times (u8 / 255, a
               noisy weight mu + sigma . eps_in eps_out, IQN's act3 . E0); any order of K - 1 round-to-nearest adds
               costs (K - 1) u S:  tau_K = (K + 4) u.
               3xTF32 on the tensor cores: each operand is carried as a tf32 hi / lo pair whose sum is within 2^-22 of
               it, and the lo . lo product is dropped: 3 . 2^-22 = 12 u per product, plus the operand roundings above;
               the accumulator may truncate instead of rounding, 2 u per add:  tau_K = (2 K + 16) u.
  statistical  the 99th percentile of |got - ref| / S is at most (4 sqrt(K) + e) u, e the per-product term above (4
               or 16): rounding errors of independent adds grow as sqrt(K), so a systematic error (a slice added twice
               or dropped, a scaled row) that the worst-case bound absorbs shows here.
  per example  the input gradients of each example within learner_parity.REL (the project's 1e-5) of the reference
               in norm, so that one example's row is compared on its own and not inside the norm of the whole batch.
  exact        dact* is exactly 0 where the device's mask is 0; on the tensor-core torso dact*_hi / dact*_lo are the
               tf32 split of dact* by the rule test_gpu_noisy_head.py pins for dh1; the global gradient norm is the
               float64 norm of the device's own gradients within 64 u (every square rounds once, and no path chains
               more than 60 fp32 adds from a square to the norm).

test_used_learner_equals_a_fresh_one: one update on extreme frames, then one on random frames, gives the bits of a
fresh learner's single update on the random frames, eagerly and replayed from a CUDA graph: no scratch (split-K
partials, bias-chunk tickets, norm slots) carries over between steps.
"""

import math

import numpy as np
import pytest
import torch

from learner_parity import REL, device_buffer, mma_path, tensor_core_torso
from oracle import stage_oracle as so
from test_gpu_noisy_head import rna_tf32

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
TINY = 2.0 ** -126
A = 6


def _hw(hw):
  return (hw, hw) if isinstance(hw, int) else tuple(hw)


def dims(H, W):
  h1, w1 = (H - 8) // 4 + 1, (W - 8) // 4 + 1
  h2, w2 = (h1 - 4) // 2 + 1, (w1 - 4) // 2 + 1
  return (h1, w1), (h2, w2), (h2 - 2, w2 - 2)


def make_learner(kind, hw, B, dueling=False, noisy=False, seed=11):
  """A learner with the library's initial parameters, a distinct target and host-drawn taus / noise in its buffers."""
  from dqn_zoo_b200 import learner as dl
  H, W = _hw(hw)
  full = (H, W) == (84, 84)
  taus = (64, 64, 64) if full else (8, 5, 7)
  net = dl.NetworkSpec(kind, A, num_atoms=51 if full else 21, num_quantiles=201 if full else 33, latent_dim=64,
                       tau_samples_s_tm1=taus[0], tau_samples_policy=taus[1], tau_samples_s_t=taus[2],
                       obs_shape=(H, W, 4), dueling=dueling, noisy=noisy)
  L = dl.Learner(net, batch_size=B)
  L.init_params(seed)
  rs = np.random.RandomState(seed)
  L.set_params({k: v + np.float32(0.01) * rs.standard_normal(v.shape).astype(np.float32)
                for k, v in L.get_params().items()}, blob='target')
  L.taus.copy_(torch.as_tensor(rs.uniform(size=L.taus.numel()).astype(np.float32)))
  e = rs.standard_normal(L.noise.numel())
  L.noise.copy_(torch.as_tensor((np.sign(e) * np.sqrt(np.abs(e))).astype(np.float32)))
  return L


def random_batch(L, rs, frames=None):
  B = L.batch_size
  H, W, C = L.net.obs_shape
  s_tm1 = rs.randint(0, 256, (B, H, W, C)).astype(np.uint8) if frames is None else frames[0]
  s_t = rs.randint(0, 256, (B, H, W, C)).astype(np.uint8) if frames is None else frames[1]
  a = rs.randint(0, A, B).astype(np.int32)
  r = rs.choice([-1.0, 0.0, 1.0, 0.37], size=B).astype(np.float32)
  d = rs.choice([0.0, 0.99, 0.99 ** 3], size=B).astype(np.float32)
  w = rs.uniform(0.1, 1.0, B).astype(np.float32) if L.kind in ('rainbow', 'prioritized') else None
  return s_tm1, a, r, d, s_t, w


def extreme_frames(L):
  B = L.batch_size
  H, W, C = L.net.obs_shape
  white = np.full((H, W, C), 255, np.uint8)
  black = np.zeros((H, W, C), np.uint8)
  s_tm1 = np.stack([white if b % 2 else black for b in range(B)])
  return s_tm1, s_tm1[::-1].copy()


def buf(L, name, shape):
  return device_buffer(L, name).to(torch.float64).reshape(shape)


def check(name, got, ref, S, K, tc, rows=None):
  """The hard, statistical and per-example bars of the module docstring; returns the worst error / tau_K S."""
  got = torch.as_tensor(got).to(torch.float64).reshape(ref.shape)
  assert torch.isfinite(got).all(), (name, 'non-finite element')
  e = 16 if tc else 4
  tau = ((2 * K if tc else K) + e) * U
  err = (got - ref).abs()
  ratio = err / (tau * S + TINY)
  worst = float(ratio.max())
  if worst > 1.0:
    i = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
    raise AssertionError((name, 'hard bar', worst, 'at', i, float(got[i]), float(ref[i]), float(S[i]),
                          int((ratio > 1).sum()), 'elements over'))
  live = S > 0
  if live.any():
    p99 = float(np.percentile((err[live] / S[live]).numpy(), 99))
    assert p99 <= (4 * math.sqrt(K) + e) * U, (name, 'statistical bar', p99 / U, 'u; bar',
                                               4 * math.sqrt(K) + e, 'u')
  if rows is not None:
    d = (got - ref).reshape(rows, -1).norm(dim=1)
    n = ref.reshape(rows, -1).norm(dim=1)
    bad = d > REL * n + TINY
    assert not bad.any(), (name, 'per-example bar, examples', bad.nonzero().flatten().tolist(), (d / n)[bad].tolist())
  return worst


def check_masked(name, got, mask):
  z = torch.as_tensor(got).reshape(mask.shape)[~mask]
  assert (z == 0).all(), (name, 'non-zero where the mask is 0', int((z != 0).sum()))


def check_split(L, name, dact):
  f = dact.to(torch.float32).numpy().reshape(-1)
  hi = device_buffer(L, name + '_hi').numpy()
  lo = device_buffer(L, name + '_lo').numpy()
  np.testing.assert_array_equal(hi, rna_tf32(f), err_msg=name + '_hi')
  np.testing.assert_array_equal(lo, rna_tf32(f - hi), err_msg=name + '_lo')


def noise_vectors(L, apply=0):
  from dqn_zoo_b200 import learner as dl
  out, off = {}, apply * L.noise_stride
  noise = L.noise.cpu().numpy()
  for name, n in dl.noise_vector_sizes(L.net):
    out[name] = noise[off:off + n]
    off += (n + 3) // 4 * 4
  return out


def fc1_layers(L):
  """fc1's streams as (weight name prefix, h1 buffer, dh1 buffer, noise vector prefix or None)."""
  noisy = L.kind == 'rainbow' or L.net.noisy
  if 'adv1/w' in L.tensors or 'adv1/mu/w' in L.tensors:
    return [('adv1', 'h1', 'dh1', 'adv1' if noisy else None), ('val1', 'h1_val', 'dh1_val', 'val1' if noisy else None)]
  return [('fc1', 'h1', 'dh1', 'fc1' if noisy else None)]


def check_stages(L, s_tm1):
  """Every stage of the module docstring on learner L after its last update on frames s_tm1."""
  from dqn_zoo_b200 import learner as dl
  B = L.batch_size
  H, W, _ = L.net.obs_shape
  (h1, w1), (h2, w2), (h3, w3) = dims(H, W)
  feat = h3 * w3 * 64
  tc = tensor_core_torso(L)
  P = {k: torch.as_tensor(v).to(torch.float64) for k, v in L.get_params().items()}
  G = {k: torch.as_tensor(v).to(torch.float64) for k, v in L.get_params('grads').items()}
  act1 = buf(L, 'act1', (B, h1, w1, 32))
  act2 = buf(L, 'act2', (B, h2, w2, 64))
  if tc:   # the tensor-core torso keeps act1 / act2 as tf32 hi / lo images, and its GEMMs read both
    act1 = act1 + buf(L, 'act1_lo', act1.shape)
    act2 = act2 + buf(L, 'act2_lo', act2.shape)
  act3 = buf(L, 'act3', (B, feat))
  dact = {i: buf(L, 'dact%d' % i, shape) for i, shape in ((1, (B, h1, w1, 32)), (2, (B, h2, w2, 64)), (3, (B, feat)))}
  worst = {}

  # fc1: dact3 and the fc1 weight gradients
  if dl.uses_iqn_network(L.kind):
    dh1 = device_buffer(L, 'dh1').to(torch.float64).reshape(B, -1, 512)
    N = dh1.shape[1]
    packed = mma_path(L, 'iqn_fc1_wgrad') == 1
    E0 = buf(L, 'iqn_e0', (B, N, feat))
    ref, S = so.linear_dgrad([(dh1.reshape(-1, 512), P['fc1/w'], None)])
    ref, S = ref.reshape(B, N, feat), S.reshape(B, N, feat)
    if mma_path(L, 'iqn_embed_wgrad') == 1:   # the packed Hadamard backward leaves dhi as it found it
      dhi = buf(L, 'iqn_dhi', (B, N, feat))
      worst['dhi'] = check('dhi', dhi, ref, S, 512, packed, rows=B)
      ref, S = so.hadamard_dgrad(dhi, E0, act3 > 0)
      worst['dact3'] = check('dact3', dact[3], ref, S, N, False, rows=B)
    else:   # the unpacked one writes the embedding's gradient over dhi: check fc1's input gradient and it as one stage
      S = (S * E0.abs()).sum(1) * (act3 > 0)
      ref, _ = so.hadamard_dgrad(ref, E0, act3 > 0)
      worst['dact3'] = check('dact3', dact[3], ref, S, 512 + N, packed, rows=B)
    hi = (act3[:, None, :] * E0).reshape(-1, feat)
    dW, db, SW, Sb = so.linear_wgrad(hi, dh1.reshape(-1, 512))
    worst['fc1/w'] = check('fc1/w', G['fc1/w'], dW, SW, B * N, packed)
    worst['fc1/b'] = check('fc1/b', G['fc1/b'], db, Sb, B * N, packed)
  else:
    layers = fc1_layers(L)
    nz = noise_vectors(L) if layers[0][3] else None
    terms = []
    for prefix, _, dh1_name, noise in layers:
      dh1 = buf(L, dh1_name, (B, 512))
      if noise is None:
        terms.append((dh1, P[prefix + '/w'], None))
        dW, db, SW, Sb = so.linear_wgrad(act3, dh1)
        worst[prefix + '/w'] = check(prefix + '/w', G[prefix + '/w'], dW, SW, B, False)
        worst[prefix + '/b'] = check(prefix + '/b', G[prefix + '/b'], db, Sb, B, False)
        continue
      ei = torch.as_tensor(nz[noise + '/in']).to(torch.float64)
      eo = torch.as_tensor(nz[noise + '/out']).to(torch.float64)
      Wf, Wabs = so.noisy_weight(P[prefix + '/mu/w'], P[prefix + '/sigma/w'], ei, eo)
      terms.append((dh1, Wf, Wabs))
      for part, x, g in (('mu', act3, dh1), ('sigma', act3 * ei, dh1 * eo)):
        dW, db, SW, Sb = so.linear_wgrad(x, g)
        worst['%s/%s/w' % (prefix, part)] = check('%s/%s/w' % (prefix, part), G['%s/%s/w' % (prefix, part)], dW, SW, B,
                                                  False)
        worst['%s/%s/b' % (prefix, part)] = check('%s/%s/b' % (prefix, part), G['%s/%s/b' % (prefix, part)], db, Sb, B,
                                                  False)
    ref, S = so.linear_dgrad(terms, act3 > 0)
    worst['dact3'] = check('dact3', dact[3], ref, S, 512 * len(terms), tc, rows=B)

  # the torso: each input gradient from the next one's, each weight gradient from its input and its output's gradient
  d3 = dact[3].reshape(B, h3, w3, 64)
  ref, S = so.conv_dgrad(d3, P['conv3/w'], 1, (h2, w2), act2 > 0)
  worst['dact2'] = check('dact2', dact[2], ref, S, 64 * 9, tc, rows=B)
  ref, S = so.conv_dgrad(dact[2], P['conv2/w'], 2, (h1, w1), act1 > 0)
  worst['dact1'] = check('dact1', dact[1], ref, S, 64 * 4, tc, rows=B)
  x0 = so.unit_frames(s_tm1)
  for layer, x, dy, k, s in ((3, act2, d3, 3, 1), (2, act1, dact[2], 4, 2), (1, x0, dact[1], 8, 4)):
    dW, db, SW, Sb = so.conv_wgrad(x, dy, k, s)
    K = B * dy.shape[1] * dy.shape[2]
    worst['conv%d/w' % layer] = check('conv%d/w' % layer, G['conv%d/w' % layer], dW, SW, K, tc)
    worst['conv%d/b' % layer] = check('conv%d/b' % layer, G['conv%d/b' % layer], db, Sb, K, tc)

  # exact: the masks, the tf32 split the next GEMM reads, the global norm over the device's own gradients
  for i, a in ((1, act1), (2, act2), (3, act3)):
    check_masked('dact%d' % i, dact[i], a > 0)
    if tc:
      check_split(L, 'dact%d' % i, dact[i])
  ss = sum(float((g * g).sum()) for k, g in G.items() if not k.startswith('fraction/'))   # fqf's norm excludes its
  gn = float(L.grad_norm.item())                                                            # fraction layer
  assert abs(gn - math.sqrt(ss)) <= 64 * U * math.sqrt(ss), ('global norm', gn, math.sqrt(ss))
  return worst


def run_stages(kind, hw, B, tc, dueling=False, noisy=False, packed=None):
  L = make_learner(kind, hw, B, dueling, noisy)
  assert tensor_core_torso(L) == tc, 'torso path'
  if packed is not None:
    assert (mma_path(L, 'iqn_fc1_wgrad') == 1) == packed, 'packed IQN GEMM'
  rs = np.random.RandomState(B)
  s_tm1, a, r, d, s_t, w = random_batch(L, rs)
  L.update(s_tm1, a, r, d, s_t, weights=w, apply_update=False)
  torch.cuda.synchronize()
  worst = check_stages(L, s_tm1)
  print('%s %s B=%d: worst error / tau_K S %s' % (kind, _hw(hw), B, {k: round(v, 4) for k, v in worst.items()}))


# (kind, observation, batch, tensor-core torso, packed IQN GEMM): every kind, on both torso paths, with the batches
# paired to geometries: 1 and 5 (partial M tiles), 32 / 33 / 64 (the split and 128-row bias-chunk edges), 65 (> 64:
# the fp32-FMA torso at 84x84); 84x88 has an odd conv1 width (21), which the tensor-core torso does not take
CASES = [
    ('dqn', 84, 32, True, None), ('double_q', 84, 33, True, None), ('prioritized', 84, 64, True, None),
    ('c51', 84, 5, True, None), ('qrdqn', 84, 1, True, None), ('rainbow', 84, 33, True, None),
    ('iqn', 84, 32, True, True), ('munchausen', 84, 33, True, None), ('munchausen_iqn', 84, 32, True, True),
    ('fqf', 84, 33, True, None),
    ('dqn', 44, 5, True, None), ('rainbow', 44, 1, True, None), ('c51', 44, 33, True, None),
    ('qrdqn', 44, 64, True, None), ('iqn', 44, 5, True, False), ('munchausen_iqn', 44, 33, True, None),
    ('fqf', 44, 5, True, None), ('munchausen', 44, 64, True, None),
    ('dqn', 84, 65, False, None), ('rainbow', 84, 65, False, None), ('iqn', 84, 65, False, True),
    ('dqn', (84, 88), 33, False, None), ('c51', (84, 88), 5, False, None), ('rainbow', (84, 88), 32, False, None),
    ('iqn', (84, 88), 5, False, False), ('fqf', (84, 88), 1, False, None), ('prioritized', (84, 88), 64, False, None),
]


@pytest.mark.parametrize('kind,hw,B,tc,packed', CASES)
def test_stages(kind, hw, B, tc, packed):
  run_stages(kind, hw, B, tc, packed=packed)


# dueling and noisy fc1 streams: dact3 sums two streams' input gradients; a noisy layer's weights are formed from the
# step's noise apply 0
NETWORK_CASES = [
    ('dqn', 84, 32, True, True, False), ('double_q', 84, 33, True, False, True), ('prioritized', 84, 1, True, True, True),
    ('munchausen', 84, 64, True, True, True), ('dqn', 44, 5, True, False, True), ('double_q', 44, 64, True, True, True),
    ('prioritized', 44, 33, True, True, False), ('munchausen', 44, 1, True, False, True),
    ('dqn', 84, 65, False, True, True), ('munchausen', (84, 88), 33, False, True, False),
    ('prioritized', (84, 88), 5, False, False, True),
]


@pytest.mark.parametrize('kind,hw,B,tc,dueling,noisy', NETWORK_CASES)
def test_stages_dueling_and_noisy(kind, hw, B, tc, dueling, noisy):
  run_stages(kind, hw, B, tc, dueling, noisy)


# ---- a used learner equals a fresh one -------------------------------------------------------------------------------

OUTPUTS = ('loss', 'per_example', 'priorities', 'regularizer', 'grad_norm', 'grads')


def snapshot(L):
  torch.cuda.synchronize()
  out = {n: getattr(L, n).clone() for n in OUTPUTS}
  for i in (1, 2, 3):
    out['dact%d' % i] = device_buffer(L, 'dact%d' % i)
  return out


def device_batch(L, host):
  s_tm1, a, r, d, s_t, w = host
  dev = lambda x: None if x is None else torch.as_tensor(x).cuda()
  return [dev(s_tm1), dev(a), dev(r), dev(d), dev(s_t), dev(w)]


def copy_batch(dst, src):
  for t, x in zip(dst, src):
    if t is not None:
      t.copy_(x)


def update(L, b):
  L.update(b[0], b[1], b[2], b[3], b[4], weights=b[5], apply_update=False)


@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graph'])
@pytest.mark.parametrize('kind', ['dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn', 'munchausen',
                                  'munchausen_iqn', 'fqf'])
def test_used_learner_equals_a_fresh_one(kind, graph):
  used = make_learner(kind, 84, 33)
  rs = np.random.RandomState(5)
  x1 = random_batch(used, rs, extreme_frames(used))
  x2 = random_batch(used, rs)
  b1, b2 = device_batch(used, x1), device_batch(used, x2)
  if graph:
    update(used, b1)                  # the first step runs eagerly (the warm-up of the capture), as the agents do
    torch.cuda.synchronize()
    static = [None if t is None else t.clone() for t in b1]
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
      update(used, static)
    g.replay()                        # extreme frames again, from the graph
    copy_batch(static, b2)
    g.replay()
  else:
    update(used, b1)
    update(used, b2)
  got = snapshot(used)
  fresh = make_learner(kind, 84, 33)
  update(fresh, b2)
  want = snapshot(fresh)
  for name, t in want.items():
    assert torch.equal(got[name], t), (kind, name, 'differs after a step on other frames')
