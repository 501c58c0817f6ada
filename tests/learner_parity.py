"""Learner parity checks shared by the GPU learner tests: the CUDA learner against the float64 PyTorch-CPU oracle
(oracle/learner_oracle.py) at a given agent, observation geometry, batch and head shape.

Tolerance (BASELINE.json north_star): <= 1e-5 relative on fp32 losses and gradients.  Gradients are compared per
tensor as ||g - g_ref|| / ||g_ref|| (and the global norm), losses per example.
"""

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo

REL = 1e-5


def _hw(hw):
  return (hw, hw) if isinstance(hw, int) else tuple(hw)


def make_case(kind, B, hw, seed, num_actions=6, num_atoms=None, num_quantiles=None, latent_dim=64, taus=None, vmax=10.0,
              grad_error_bound=1.0 / 32, huber_param=1.0):
  """hw: side of a square observation, or (H, W).  taus: (s_tm1, policy, s_t) sample counts of IQN.  Unset head sizes
  and tau counts take the full-size values at 84x84 and small ones elsewhere.  vmax, grad_error_bound and huber_param
  go to both the device learner and the oracle."""
  from dqn_zoo_b200 import learner as dl
  H, W = _hw(hw)
  full = (H, W) == (84, 84)
  rs = np.random.RandomState(seed)
  heads = dict(num_atoms=51 if full else 21, num_quantiles=201 if full else 33, latent_dim=latent_dim)
  if num_atoms is not None:
    heads['num_atoms'] = num_atoms
  if num_quantiles is not None:
    heads['num_quantiles'] = num_quantiles
  if taus is None:
    taus = (64, 64, 64) if full else (8, 5, 7)
  spec = lo.NetSpec(kind, num_actions, obs_hw=H, obs_w=W, vmax=vmax, **heads)
  net = dl.NetworkSpec(kind, num_actions, obs_shape=(H, W, 4), tau_samples_s_tm1=taus[0], tau_samples_policy=taus[1],
                       tau_samples_s_t=taus[2], vmax=vmax, **heads)
  online = lo.init_params(spec, seed)
  target = lo.init_params(spec, seed + 1)
  L = dl.Learner(net, batch_size=B, grad_error_bound=grad_error_bound, huber_param=huber_param)
  L.set_params(online)
  L.set_params(target, blob='target')
  O = lo.Learner(spec, online, dtype=torch.float64, grad_error_bound=grad_error_bound, huber_param=huber_param)
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  return spec, net, L, O, rs


def obs_shape(spec):
  return spec.obs_hw, spec.obs_hw if spec.obs_w is None else spec.obs_w


def random_noise(spec, rs):
  one = {}
  for name, k in lo.noise_shapes(spec):
    x = np.clip(rs.standard_normal(k), -2, 2)
    one[name] = (np.sign(x) * np.sqrt(np.abs(x))).astype(np.float32)
  return one


def make_batch(spec, net, B, rs):
  H, W = obs_shape(spec)
  s_tm1 = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
  s_t = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
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
    raw = [random_noise(spec, rs) for _ in range(3)]
    noise_o = [{k: torch.tensor(v) for k, v in one.items()} for one in raw]
    noise_flat = dl.pack_noise(net, raw)
  batch = lo.batch_from_numpy(s_tm1, a, r, d, s_t)
  return (s_tm1, a, r, d, s_t), batch, w, taus_o, taus_flat, noise_o, noise_flat


RELU_BUFFERS = {   # oracle ReLU name -> device buffer of the post-ReLU activation (pass 0 = online(s_tm1))
    'dqn': {'conv1': 'act1', 'conv2': 'act2', 'conv3': 'act3', 'fc1': 'h1'},
    'rainbow': {'conv1': 'act1', 'conv2': 'act2', 'conv3': 'act3', 'adv1': 'h1', 'val1': 'h1_val'},
    'iqn': {'conv1': 'act1', 'conv2': 'act2', 'conv3': 'act3', 'embed': 'iqn_e0', 'fc1': 'h1'},
}


def device_buffer(L, name):
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


def assert_flips_at_the_kink(flips, *where):
  for name, (nflip, units, worst) in flips.items():
    assert worst <= 2e-5, ('a flipped unit is NOT at the kink',) + where + (name, nflip, worst)
    assert nflip <= 3 + 2e-5 * units, ('too many kink flips',) + where + (name, nflip, units)


def rel_err(got, want):
  want = np.asarray(want, dtype=np.float64)
  denom = np.linalg.norm(want.reshape(-1))
  return np.linalg.norm((np.asarray(got, dtype=np.float64) - want).reshape(-1)) / max(denom, 1e-30)


def check_loss_and_gradients(kind, hw, B, fma_torso=False, **case):
  """One update without the optimizer step: loss, per-example values, global norm and every gradient tensor within
  REL of the oracle.  Returns the case (spec, net, L, O, rs) for further checks."""
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
  assert_flips_at_the_kink(flips)
  if flips:
    print('relu kink flips %s %s B=%d: %s' % (kind, _hw(hw), B, {k: v[:2] for k, v in flips.items()}))
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
  return spec, net, L, O, rs


def check_three_optimizer_steps(kind, hw, B, seed=5, **case):
  """Three full updates (optimizer included) against three oracle updates: loss per step, priorities, the parameter
  movement and the first-moment state."""
  spec, net, L, O, rs = make_case(kind, B, hw, seed=seed, **case)
  lr = L.opt.learning_rate
  p0 = {k: v.numpy().copy() for k, v in O.online.items()}
  for step in range(3):
    arrs, batch, w, taus_o, taus_flat, noise_o, noise_flat = make_batch(spec, net, B, rs)
    wt = None if w is None else torch.tensor(w)
    tap = lo.ReluTap()
    O.grads(batch, wt, taus_o, noise_o, tap=tap)   # the float64 pre-activations of this step
    L.update(*arrs, weights=w, taus=taus_flat, noise=noise_flat, apply_update=True)
    torch.cuda.synchronize()
    # as in check_loss_and_gradients: a unit whose float64 pre-activation is within float32 rounding of zero may fall
    # on the other side of the kink on the device; such flips must be AT the kink and few, and the oracle step is then
    # taken on the device's activation pattern so that the bars below measure arithmetic error only
    masks, flips = relu_kink_flips(kind, L, tap)
    assert_flips_at_the_kink(flips, step)
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


def check_q_values(spec, net, L, O, rs):
  """Q-values of one observation (the acting forward, batch 1) against lo.apply_net."""
  from dqn_zoo_b200 import learner as dl
  H, W = obs_shape(spec)
  obs = rs.randint(0, 256, (H, W, 4)).astype(np.uint8)
  taus = noise = taus_o = noise_o = None
  if spec.kind == 'iqn':
    taus = rs.uniform(size=(1, net.tau_samples_policy)).astype(np.float32)
    taus_o = torch.tensor(taus)
  if spec.kind == 'rainbow':
    one = random_noise(spec, rs)
    noise_o = {k: torch.tensor(v) for k, v in one.items()}
    noise = dl.pack_noise(net, [one])
  want = lo.apply_net(spec, O.online, torch.tensor(obs[None]), torch.float64, taus=taus_o, noise=noise_o)['q_values'][0]
  got = L.q_values(torch.tensor(obs), taus=taus, noise=noise).cpu().numpy()
  np.testing.assert_allclose(got, want.numpy(), rtol=2e-5, atol=2e-6, err_msg=spec.kind)


def mma_path(L, tag):
  """dz_test_learner_mma_path of the launch `tag`: 1 mma.sync, 2 wgmma; None when the launch is not on a tensor-core
  kernel (or the learner has no such launch)."""
  from dqn_zoo_b200 import _lib
  p = C.c_int32(-1)
  try:
    _lib.call('dz_test_learner_mma_path', L._h, tag.encode(), C.byref(p))
  except ValueError:
    return None
  return p.value


def tensor_core_torso(L):
  from dqn_zoo_b200 import _lib
  try:
    _lib.call('dz_test_learner_trace', L._h, b'', 0)
  except ValueError:
    return False
  return True
