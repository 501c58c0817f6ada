"""GPU: the CUDA learner vs the float64 PyTorch-CPU oracle (oracle/learner_oracle.py).

Tolerance (BASELINE.json north_star): <= 1e-5 relative on fp32 losses and gradients.  Gradients
are compared per tensor as ||g - g_ref|| / ||g_ref|| (and the global norm), losses per example.
Parity is against the restatement of rlax/optax 0.1.2 (PARITY UNPINNED, see the oracle header).
"""

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo

pytestmark = pytest.mark.gpu

REL = 1e-5
KINDS = list(lo.AGENT_KINDS)


def make_case(kind, B, hw, seed, num_actions=6, num_atoms=None):
  from dqn_zoo_b200 import learner as dl
  rs = np.random.RandomState(seed)
  small = dict(num_atoms=51, num_quantiles=201) if hw == 84 else dict(num_atoms=21, num_quantiles=33)
  if num_atoms is not None:
    small['num_atoms'] = num_atoms
  spec = lo.NetSpec(kind, num_actions, obs_hw=hw, **small)
  net = dl.NetworkSpec(kind, num_actions, obs_shape=(hw, hw, 4), tau_samples_s_tm1=64 if hw == 84 else 8,
                       tau_samples_policy=64 if hw == 84 else 5, tau_samples_s_t=64 if hw == 84 else 7, **small)
  online = lo.init_params(spec, seed)
  target = lo.init_params(spec, seed + 1)
  L = dl.Learner(net, batch_size=B)
  L.set_params(online)
  L.set_params(target, blob='target')
  O = lo.Learner(spec, online, dtype=torch.float64)
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  return spec, net, L, O, rs


def make_batch(spec, net, B, rs):
  hw = spec.obs_hw
  s_tm1 = rs.randint(0, 256, (B, hw, hw, 4)).astype(np.uint8)
  s_t = rs.randint(0, 256, (B, hw, hw, 4)).astype(np.uint8)
  a = rs.randint(0, spec.num_actions, B)
  r = rs.choice([-1.0, 0.0, 1.0, 0.37], size=B)
  d = rs.choice([0.0, 0.99, 0.99 ** 3], size=B)
  w = rs.uniform(0.1, 1.0, B) if spec.kind in ('rainbow', 'prioritized') else None
  taus_o = taus_flat = noise_o = noise_flat = None
  if spec.kind == 'iqn':
    n = (net.tau_samples_s_tm1, net.tau_samples_policy, net.tau_samples_s_t)
    taus = [rs.uniform(size=(B, k)).astype(np.float32) for k in n]
    taus_o = [torch.tensor(t) for t in taus]
    taus_flat = np.concatenate([t.reshape(-1) for t in taus])
  if spec.kind == 'rainbow':
    from dqn_zoo_b200 import learner as dl
    noise_o, raw = [], []
    for _ in range(3):
      one = {}
      for name, k in lo.noise_shapes(spec):
        x = np.clip(rs.standard_normal(k), -2, 2)
        one[name] = (np.sign(x) * np.sqrt(np.abs(x))).astype(np.float32)
      raw.append(one)
      noise_o.append({k: torch.tensor(v) for k, v in one.items()})
    noise_flat = dl.pack_noise(net, raw)
  batch = lo.batch_from_numpy(s_tm1, a, r, d, s_t)
  return (s_tm1, a, r, d, s_t), batch, w, taus_o, taus_flat, noise_o, noise_flat


RELU_BUFFERS = {   # oracle ReLU name -> device buffer of the post-ReLU activation (pass 0 = online(s_tm1))
    'dqn': {'conv1': 'act1', 'conv2': 'act2', 'conv3': 'act3', 'fc1': 'h1'},
    'rainbow': {'conv1': 'act1', 'conv2': 'act2', 'conv3': 'act3', 'adv1': 'h1', 'val1': 'h1_val'},
    'iqn': {'conv1': 'act1', 'conv2': 'act2', 'conv3': 'act3', 'embed': 'iqn_e0', 'fc1': 'h1'},
}


def device_buffer(L, name):
  import ctypes as C
  from dqn_zoo_b200 import _lib
  ptr, n = C.c_void_p(), C.c_int64()
  _lib.call('dz_test_learner_buffer', L._h, name.encode(), C.byref(ptr), C.byref(n))
  out = torch.empty(n.value, dtype=torch.float32, device='cuda')
  _lib.call('dz_test_copy', out.data_ptr(), ptr, 4 * n.value, torch.cuda.current_stream().cuda_stream)
  return out.cpu()


def relu_kink_flips(kind, L, tap):
  """Units of online(s_tm1) whose activation pattern differs between the device (float32) and the oracle (float64).
  Returns (device masks by oracle ReLU name, {name: (flips, units, worst |pre| / rms(pre) among the flipped)})."""
  table = RELU_BUFFERS.get(kind, RELU_BUFFERS['dqn'])
  masks, report = {}, {}
  for name, buf in table.items():
    pre = tap.pre[name]
    dev = device_buffer(L, buf).reshape(pre.shape) > 0
    masks[name] = dev
    flipped = dev != (pre > 0)
    nflip = int(flipped.sum())
    if nflip:
      rms = float(pre.pow(2).mean().sqrt())
      report[name] = (nflip, pre.numel(), float(pre[flipped].abs().max()) / rms)
  return masks, report


def rel_err(got, want):
  want = np.asarray(want, dtype=np.float64)
  denom = np.linalg.norm(want.reshape(-1))
  return np.linalg.norm((np.asarray(got, dtype=np.float64) - want).reshape(-1)) / max(denom, 1e-30)


@pytest.mark.parametrize('hw,B', [(84, 32), (44, 5)])
@pytest.mark.parametrize('kind', KINDS)
def test_loss_and_gradients_match_oracle(kind, hw, B):
  check_loss_and_gradients(kind, hw, B)


def check_loss_and_gradients(kind, hw, B, fma_torso=False, **case):
  spec, net, L, O, rs = make_case(kind, B, hw, seed=3, **case)
  if fma_torso:   # the tensor-core path must not be active, or the caller would not test the fp32-FMA torso
    from dqn_zoo_b200 import _lib
    with pytest.raises(ValueError):
      _lib.call('dz_test_learner_trace', L._h, b'', 0)
  arrs, batch, w, taus_o, taus_flat, noise_o, noise_flat = make_batch(spec, net, B, rs)
  tap = lo.ReluTap()
  loss, aux, grads = O.grads(batch, None if w is None else torch.tensor(w), taus_o, noise_o, tap=tap)
  L.update(*arrs, weights=w, taus=taus_flat, noise=noise_flat, apply_update=False)
  torch.cuda.synchronize()
  assert abs(float(L.loss.item()) - float(loss)) <= REL * abs(float(loss)), (float(L.loss.item()), float(loss))
  # ReLU kinks: the loss is continuous across them, the gradient is not.  Count the units whose float64
  # pre-activation is so close to zero that the float32 device evaluation lands on the other side; every such flip
  # must be within float32 rounding of the kink (|pre| <= 2e-5 rms of its layer) and there must be only a handful.
  # With flips present the gradient bar is applied against the oracle evaluated ON THE DEVICE'S activation pattern
  # (same arithmetic, same 1e-5), so the bar measures arithmetic error and the flips are reported, not hidden.
  masks, flips = relu_kink_flips(kind, L, tap)
  for name, (nflip, units, worst) in flips.items():
    assert worst <= 2e-5, ('a flipped unit is NOT at the kink', name, nflip, worst)
    assert nflip <= 3 + 2e-5 * units, ('too many kink flips', name, nflip, units)
  if flips:
    print('relu kink flips %s %dx%d: %s' % (kind, hw, B, {k: v[:2] for k, v in flips.items()}))
    loss2, aux, grads = O.grads(batch, None if w is None else torch.tensor(w), taus_o, noise_o, tap=lo.ReluTap(masks))
    assert abs(float(loss2) - float(loss)) <= 1e-5 * abs(float(loss))
  want_pe = (aux['td_errors'] if kind in ('dqn', 'double_q', 'prioritized') else aux['losses']).numpy()
  assert rel_err(L.per_example.cpu().numpy(), want_pe) <= REL
  gn = float(torch.sqrt(sum((g * g).sum() for g in grads.values())))
  assert abs(float(L.grad_norm.item()) - gn) <= REL * gn
  worst = {}
  for name in L.tensors:
    got = L.view(L.grads, name).cpu().numpy()
    want = grads[name].numpy()
    if np.linalg.norm(want) < 1e-12 * max(gn, 1e-30):
      assert np.abs(got).max() <= 1e-9 * max(gn, 1.0), name
      continue
    worst[name] = rel_err(got, want)
  bad = {k: v for k, v in worst.items() if v > REL}
  assert not bad, bad


@pytest.mark.parametrize('kind', ['c51', 'rainbow'])
def test_largest_categorical_head_matches_oracle(kind):
  """64 actions x 128 atoms, the largest categorical head the learner accepts: the loss kernel then stages 103,696
  bytes of head outputs in shared memory, beyond the default 48 KB.  Same loss/gradient parity."""
  check_loss_and_gradients(kind, 84, 32, num_actions=64, num_atoms=128)


@pytest.mark.parametrize('kind', KINDS)
def test_three_optimizer_steps_match_oracle(kind):
  B, hw = 32, 84
  spec, net, L, O, rs = make_case(kind, B, hw, seed=5)
  lr = L.opt.learning_rate
  p0 = {k: v.numpy().copy() for k, v in O.online.items()}
  for step in range(3):
    arrs, batch, w, taus_o, taus_flat, noise_o, noise_flat = make_batch(spec, net, B, rs)
    wt = None if w is None else torch.tensor(w)
    tap = lo.ReluTap()
    O.grads(batch, wt, taus_o, noise_o, tap=tap)   # the float64 pre-activations of this step
    L.update(*arrs, weights=w, taus=taus_flat, noise=noise_flat, apply_update=True)
    torch.cuda.synchronize()
    # as in test_loss_and_gradients_match_oracle: a unit whose float64 pre-activation is within float32 rounding of
    # zero may fall on the other side of the kink on the device; such flips must be AT the kink and few, and the oracle
    # step is then taken on the device's activation pattern so that the bars below measure arithmetic error only
    masks, flips = relu_kink_flips(kind, L, tap)
    for name, (nflip, units, worst) in flips.items():
      assert worst <= 2e-5, ('a flipped unit is NOT at the kink', step, name, nflip, worst)
      assert nflip <= 3 + 2e-5 * units, ('too many kink flips', step, name, nflip, units)
    aux = O.update(batch, wt, taus_o, noise_o, tap=lo.ReluTap(masks) if flips else None)
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 2 * REL * abs(float(aux['loss'])) + 1e-7
    if kind in ('rainbow', 'prioritized'):
      np.testing.assert_allclose(L.priorities.cpu().numpy(), aux['priorities'].numpy(), rtol=5e-5, atol=1e-6)
  got = L.get_params()
  for name, want in O.online.items():
    # compare the parameter MOVEMENT over the three steps: relative error of the total displacement,
    # plus a per-element bound of half an optimizer step (a ReLU unit whose pre-activation is within
    # float32 rounding of zero may flip between the fp32 device and the fp64 oracle).
    moved_ref = want.numpy() - p0[name]
    moved_got = got[name].astype(np.float64) - p0[name]
    # (adam moves every element by ~lr whatever |g| is, so near-zero gradient elements, whose sign is
    # rounding noise, dominate this error: 1e-2 of the displacement)
    assert rel_err(moved_got, moved_ref) <= 1e-2, (name, rel_err(moved_got, moved_ref))
    assert np.abs(moved_got - moved_ref).max() <= 0.5 * lr + 1e-7, name
  st = L.get_opt_state()
  # first-moment EMA of the gradients: iqn (adam without clipping, gradient norm ~7) amplifies the
  # step-1 sign noise into ~0.5 % gradient differences at steps 2-3; the others stay at 5e-5.
  tol = 1e-2 if kind == 'iqn' else 5e-5
  for name in L.tensors:
    assert rel_err(st['mu'][name], O.state['mu'][name].numpy()) <= tol or np.abs(st['mu'][name]).max() < 1e-12, name


def test_q_values_match_oracle_forward():
  for kind in KINDS:
    spec, net, L, O, rs = make_case(kind, 32, 84, seed=7)
    obs = rs.randint(0, 256, (84, 84, 4)).astype(np.uint8)
    taus = noise = taus_o = noise_o = None
    if kind == 'iqn':
      taus = rs.uniform(size=(1, 64)).astype(np.float32)
      taus_o = torch.tensor(taus)
    if kind == 'rainbow':
      from dqn_zoo_b200 import learner as dl
      noise_o = {}
      for name, k in lo.noise_shapes(spec):
        x = np.clip(rs.standard_normal(k), -2, 2)
        noise_o[name] = torch.tensor((np.sign(x) * np.sqrt(np.abs(x))).astype(np.float32))
      noise = dl.pack_noise(net, [{k: v.numpy() for k, v in noise_o.items()}])
    want = lo.apply_net(spec, O.online, torch.tensor(obs[None]), torch.float64, taus=taus_o, noise=noise_o)['q_values'][0]
    got = L.q_values(torch.tensor(obs), taus=taus, noise=noise).cpu().numpy()
    np.testing.assert_allclose(got, want.numpy(), rtol=2e-5, atol=2e-6, err_msg=kind)


def test_update_is_run_to_run_deterministic():
  spec, net, L, O, rs = make_case('rainbow', 32, 84, seed=9)
  arrs, batch, w, taus_o, taus_flat, noise_o, noise_flat = make_batch(spec, net, 32, rs)
  L.update(*arrs, weights=w, noise=noise_flat, apply_update=False)
  g1 = L.grads.clone()
  L.update(*arrs, weights=w, noise=noise_flat, apply_update=False)
  torch.cuda.synchronize()
  assert torch.equal(g1, L.grads)


@pytest.mark.parametrize('hw,B', [(84, 65), (40, 32)])
@pytest.mark.parametrize('kind', ['dqn', 'rainbow'])
def test_fp32_fma_fallback_matches_oracle(kind, hw, B):
  """Geometries the tensor-core torso does not cover run every contraction on the fp32-FMA kernels: batch > 64, and an
  odd conv1 output (9x9 at 40x40; at batch <= 32 this also takes the split-K FMA layers).  Same loss/gradient parity."""
  check_loss_and_gradients(kind, hw, B, fma_torso=True)


def test_uint8_to_unit_conversion_is_correctly_rounded():
  """networks.py:193 `x.astype(float32) / 255.0`: the device uses multiply + one Newton step instead of an
  IEEE division; it must give the correctly rounded quotient for every possible byte."""
  from dqn_zoo_b200 import _lib
  out = torch.zeros(256, dtype=torch.float32, device='cuda')
  _lib.call('dz_test_u8_to_unit', out.data_ptr(), torch.cuda.current_stream().cuda_stream)
  want = np.arange(256, dtype=np.float32) / np.float32(255.0)
  np.testing.assert_array_equal(out.cpu().numpy(), want)
