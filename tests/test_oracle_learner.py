"""CPU: independent checks of the learner oracle (oracle/learner_oracle.py), whose parity is otherwise UNPINNED
(jax / rlax / optax cannot be installed; the reference's tests assert no loss or gradient value, SURVEY §8(c)).

Two kinds of evidence that do not go through the oracle's own autograd or its own reading of rlax/optax:
  1. finite differences: for all 7 agents the autograd gradient of `loss_fn` equals the central difference of the loss
     in float64 on sampled coordinates of every parameter tensor (with `clip_gradient` inactive), and the clipped
     DQN-family gradient equals the finite difference of the surrogate  sum_b const(clip(w_b td_b / B)) * (-q_b);
  2. hand-computed vectors (tests/golden/learner_hand_vectors.json, every number derived in that file's `derivation`
     strings from the published rlax / optax formulas): categorical_l2_project, the categorical cross-entropy,
     quantile-Huber regression, double-Q TD error, Adam, centred RMSProp, clip_by_global_norm, the noisy linear layer
     and the dueling combine.
"""

import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'learner_hand_vectors.json')


def tiny_case(kind, seed=0, B=3, hw=(44, 44)):
  H, W = hw
  spec = lo.NetSpec(kind, 4, num_atoms=7, num_quantiles=5, latent_dim=16, obs_hw=H, obs_w=W)
  rs = np.random.RandomState(seed)
  # larger-than-default weights so that every head has O(1) outputs and the loss is well away from flat regions
  online = {k: (v * 3.0).astype(np.float64) for k, v in lo.init_params(spec, seed).items()}
  target = {k: (v * 3.0).astype(np.float64) for k, v in lo.init_params(spec, seed + 1).items()}
  s_tm1 = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
  s_t = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
  batch = lo.batch_from_numpy(s_tm1, rs.randint(0, 4, B), rs.choice([-1.0, 0.5, 1.0], B), rs.choice([0.0, 0.99], B), s_t)
  w = torch.tensor(rs.uniform(0.2, 1.0, B)) if kind in ('rainbow', 'prioritized') else None
  taus = [torch.tensor(rs.uniform(size=(B, n)).astype(np.float32)) for n in (6, 4, 5)] if kind == 'iqn' else None
  noise = None
  if kind == 'rainbow':
    noise = []
    for _ in range(3):
      one = {}
      for name, n in lo.noise_shapes(spec):
        x = np.clip(rs.standard_normal(n), -2, 2)
        one[name] = torch.tensor(np.sign(x) * np.sqrt(np.abs(x)))
      noise.append(one)
  return spec, online, target, batch, w, taus, noise


def loss_value(spec, online_np, target_np, batch, w, taus, noise, bound):
  on = {k: torch.tensor(v, dtype=torch.float64) for k, v in online_np.items()}
  tg = {k: torch.tensor(v, dtype=torch.float64) for k, v in target_np.items()}
  loss, aux = lo.loss_fn(spec, on, tg, batch, torch.float64, w, taus, noise, grad_error_bound=bound)
  return float(loss), aux


@pytest.mark.parametrize('kind', lo.AGENT_KINDS)
def test_autograd_gradients_equal_finite_differences(kind):
  check_finite_differences(kind, (44, 44))


@pytest.mark.parametrize('kind,hw', [('dqn', (36, 52)), ('rainbow', (52, 36)), ('iqn', (52, 36))])
def test_non_square_observation_gradients_equal_finite_differences(kind, hw):
  """A non-square observation (conv3 output 1x3 or 3x1): the feature size follows obs_hw x obs_w, so the fc1 / embed /
  noise shapes of the spec must match what the torso produces, and the gradients still equal finite differences."""
  assert lo.feature_dim(lo.NetSpec(kind, 4, obs_hw=hw[0], obs_w=hw[1])) == 64 * 3
  assert lo.feature_dim(lo.NetSpec(kind, 4, obs_hw=hw[0])) == 64 * (1 if hw[0] == 36 else 9)   # obs_w defaults to obs_hw
  check_finite_differences(kind, hw)


def check_finite_differences(kind, hw):
  spec, online, target, batch, w, taus, noise = tiny_case(kind, hw=hw)
  bound = 1e9   # clip_gradient inactive: the gradient is the derivative of the loss
  on = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in online.items()}
  tg = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  loss, _ = lo.loss_fn(spec, on, tg, batch, torch.float64, w, taus, noise, grad_error_bound=bound)
  loss.backward()
  rs = np.random.RandomState(1)
  checked = 0
  scale = max(float(v.grad.abs().max()) for v in on.values() if v.grad is not None)
  for name, v in online.items():
    g = on[name].grad
    g = np.zeros_like(v) if g is None else g.numpy()
    flat = v.reshape(-1)
    # the coordinates with the largest gradients (informative) plus random ones
    idx = sorted(set(list(np.argsort(-np.abs(g.reshape(-1)))[:2]) + list(rs.randint(0, flat.size, 2))))
    for i in idx:
      h = 1e-5 * max(1.0, abs(flat[i]))
      keep = flat[i]
      flat[i] = keep + h
      lp, _ = loss_value(spec, online, target, batch, w, taus, noise, bound)
      flat[i] = keep - h
      lm, _ = loss_value(spec, online, target, batch, w, taus, noise, bound)
      flat[i] = keep
      fd = (lp - lm) / (2 * h)
      assert abs(fd - g.reshape(-1)[i]) <= 2e-6 * scale + 1e-9, (name, int(i), fd, float(g.reshape(-1)[i]))
      checked += 1
  assert checked >= 2 * len(online)


@pytest.mark.parametrize('kind', ['dqn', 'double_q', 'prioritized'])
def test_clip_gradient_semantics_against_a_surrogate(kind):
  """rlax.clip_gradient (dqn/agent.py:101-104): forward identity, cotangent clipped.  With bound 1/32 and O(1) TD errors
  every example clips, so d loss / d theta must equal the finite difference of  sum_b c_b * (-q_tm1[b, a_b])  with the
  constants c_b = clip(w_b * td_b / B, -1/32, 1/32)."""
  spec, online, target, batch, w, taus, noise = tiny_case(kind, seed=2)
  bound = 1.0 / 32
  on = {k: torch.tensor(v, dtype=torch.float64, requires_grad=True) for k, v in online.items()}
  tg = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  loss, aux = lo.loss_fn(spec, on, tg, batch, torch.float64, w, taus, noise, grad_error_bound=bound)
  loss.backward()
  B = batch['s_tm1'].shape[0]
  wb = np.ones(B) if w is None else w.to(torch.float32).to(torch.float64).numpy()
  td = aux['td_errors'].numpy()
  assert (np.abs(wb * td / B) > bound).any(), 'test case must exercise the clip'
  coef = np.clip(wb * td / B, -bound, bound)
  a = batch['a_tm1'].numpy()

  def surrogate(params_np):
    p = {k: torch.tensor(v, dtype=torch.float64) for k, v in params_np.items()}
    q = lo.apply_net(spec, p, batch['s_tm1'], torch.float64)['q_values'].numpy()
    return float(-(coef * q[np.arange(B), a]).sum())

  for name in ('head/w', 'fc1/b', 'conv3/w', 'conv1/b'):
    g = on[name].grad.numpy().reshape(-1)
    flat = online[name].reshape(-1)
    for i in np.argsort(-np.abs(g))[:3]:
      h = 1e-5 * max(1.0, abs(flat[i]))
      keep = flat[i]
      flat[i] = keep + h
      sp = surrogate(online)
      flat[i] = keep - h
      sm = surrogate(online)
      flat[i] = keep
      fd = (sp - sm) / (2 * h)
      assert abs(fd - g[i]) <= 1e-6 * max(1.0, abs(g[i])), (name, int(i), fd, float(g[i]))


# ----------------------------------------------------------------------------------------------------------------
# hand-computed vectors
# ----------------------------------------------------------------------------------------------------------------


@pytest.fixture(scope='module')
def hand():
  with open(GOLDEN) as f:
    return json.load(f)


def t64(x):
  return torch.tensor(x, dtype=torch.float64)


def test_categorical_l2_project_hand_vectors(hand):
  for case in hand['categorical_l2_project']:
    got = lo.categorical_l2_project(t64([case['z_p']]), t64([case['probs']]), t64(case['z_q']))[0].numpy()
    np.testing.assert_allclose(got, case['expected'], rtol=0, atol=1e-15, err_msg=case['derivation'])


def test_categorical_cross_entropy_hand_vector(hand):
  case = hand['categorical_cross_entropy']
  logits = t64(case['logits_tm1'])
  loss = -(t64(case['target']) * torch.log_softmax(logits, dim=-1)).sum()
  assert abs(float(loss) - case['expected']) < 1e-14, case['derivation']
  # and the closed form the derivation uses
  want = -(0.35 * math.log(1.0 / 3.0) + 0.65 * math.log(0.5))
  assert abs(case['expected'] - want) < 1e-15


def test_quantile_huber_hand_vector(hand):
  for case in hand['quantile_regression_loss']:
    got = lo.quantile_regression_loss(t64([case['dist_src']]), t64(case['tau']), t64([case['target']]), case['kappa'])
    assert abs(float(got[0]) - case['expected']) < 1e-15, case['derivation']


def test_double_q_td_hand_vector(hand):
  case = hand['double_q_learning']
  q_sel, q_val = np.array(case['q_t_selector']), np.array(case['q_t_value'])
  td = case['r_t'] + case['discount_t'] * q_val[int(np.argmax(q_sel))] - case['q_tm1'][case['a_tm1']]
  assert abs(td - case['expected_td']) < 1e-15
  assert abs(0.5 * td * td - case['expected_l2']) < 1e-15


def test_optimizer_hand_vectors(hand):
  for case in hand['optimizer']:
    opt = lo.OptSpec(case['name'], case['lr'], case['eps'], decay=case.get('decay', 0.95), max_global_grad_norm=case.get('max_norm', 0.0))
    p = {'p': t64(case['p'])}
    state = lo.init_opt_state(opt, p)
    for g in case['grads']:
      p, state, gn = lo.optimizer_step(opt, p, {'p': t64(g)}, state)
    np.testing.assert_allclose(p['p'].numpy(), case['expected_p'], rtol=1e-13, atol=0, err_msg=case['derivation'])
    if 'expected_norm' in case:
      assert abs(float(gn) - case['expected_norm']) < 1e-14


def test_noisy_linear_and_dueling_hand_vectors(hand):
  case = hand['noisy_linear']
  p = {'l/mu/w': t64(case['mu_w']), 'l/mu/b': t64(case['mu_b']), 'l/sigma/w': t64(case['sigma_w']), 'l/sigma/b': t64(case['sigma_b'])}
  y = lo._noisy(p, 'l', t64([case['x']]), t64([case['eps_in']]), t64([case['eps_out']]), True)[0].numpy()
  np.testing.assert_allclose(y, case['expected'], rtol=0, atol=1e-15, err_msg=case['derivation'])
  duel = hand['dueling']
  adv, val = np.array(duel['adv']), np.array(duel['val'])
  logits = val[None, :] + adv - adv.mean(axis=0, keepdims=True)
  np.testing.assert_allclose(logits, duel['expected'], rtol=0, atol=1e-15)


def test_autograd_conventions_at_the_kinks_are_jaxs():
  """The GPU loss-kernel tests compare against head_loss's autograd exactly at the kinks, so its conventions there are
  pinned here, each against the JAX rule it restates."""
  # abs'(0) = sign(0) = 0 (jax.lax.abs_p's jvp multiplies by sign(x)).
  x = torch.zeros(1, dtype=torch.float64, requires_grad=True)
  x.abs().sum().backward()
  assert float(x.grad) == 0.0
  # rlax.huber_loss at |x| = k: jnp.minimum's tie sends half the cotangent to each operand, so
  # d/dx [0.5 q^2 + k (|x| - q)] = 0.5 (k * 1) + k (1 - 0.5) = k; torch.clamp(max=k) passes all of it through q
  # (d/dx = k * 1 + k * (1 - 1) = k): both give k, and the device's clamp(delta, -k, k) gives k too.
  for k in (0.5, 1.0, 3.0):
    for sgn in (1.0, -1.0):
      x = torch.tensor([sgn * k], dtype=torch.float64, requires_grad=True)
      lo.huber(x, k).sum().backward()
      assert float(x.grad) == sgn * k, (k, sgn)
  # quantile_regression_loss at delta = 0: the weight's 1[delta < 0] is 0 (tau, not 1 - tau) and the Huber slope is 0,
  # so a source quantile equal to its target contributes neither loss nor gradient, at k > 0 and at k = 0.
  for k in (0.0, 1.0):
    src = torch.tensor([[0.5]], dtype=torch.float64, requires_grad=True)
    loss = lo.quantile_regression_loss(src, torch.tensor([0.25], dtype=torch.float64), torch.tensor([[0.5]], dtype=torch.float64), k)
    loss.sum().backward()
    assert float(loss.detach()) == 0.0 and float(src.grad) == 0.0
  # jnp.argmax and torch.argmax both return the first maximum.
  assert int(torch.tensor([1.0, 3.0, 3.0, 2.0]).argmax()) == 1
  assert int(torch.tensor([[0.0, 0.0]]).argmax(dim=1)) == 0
  # rlax.clip_gradient at exactly the bound: the clipped cotangent is the bound itself.
  x = torch.tensor([2.0], dtype=torch.float64, requires_grad=True)
  (lo._ClipGrad.apply(x, -0.25, 0.25) * 0.25).sum().backward()
  assert float(x.grad) == 0.25


def test_head_loss_is_loss_fn_after_the_networks():
  """head_loss on the head outputs loss_fn's networks produce gives loss_fn's loss, and its pass-0 gradient is the
  autograd gradient of that loss wrt those outputs, for every reference kind (rainbow: advantages and values)."""
  for kind in lo.AGENT_KINDS:
    spec, online, target, batch, w, taus, noise = tiny_case(kind)
    on = {k: torch.tensor(v, dtype=torch.float64) for k, v in online.items()}
    tg = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
    loss, aux = lo.loss_fn(spec, on, tg, batch, torch.float64, w, taus, noise, grad_error_bound=0.05, huber_param=0.5)
    nz = noise or [None] * 3
    tau3 = taus or [None] * 3
    nets = [(on, batch['s_tm1']), (on if kind in ('double_q', 'prioritized', 'rainbow') else tg, batch['s_t']),
            (tg, batch['s_t'])]
    outs = [lo.apply_net(spec, p, s, torch.float64, taus=tau3[i], noise=nz[i]) for i, (p, s) in enumerate(nets)]
    field = {'c51': 'q_logits', 'qrdqn': 'q_dist', 'iqn': 'q_dist'}.get(kind, 'q_values')
    heads = [(o['adv'], o['val']) if kind == 'rainbow' else o[field] for o in outs]
    hl, haux = lo.head_loss(kind, heads, batch['a_tm1'], batch['r_t'], batch['discount_t'], w, tau3[0], vmax=spec.vmax,
                            grad_error_bound=0.05, huber_param=0.5)
    assert float(hl.detach()) == float(loss.detach()), kind
    np.testing.assert_array_equal(haux['losses'].numpy(), aux['losses'].numpy())
    grads = haux['grad'] if kind == 'rainbow' else (haux['grad'],)
    assert [g.shape for g in grads] == [x.shape for x in (heads[0] if kind == 'rainbow' else (heads[0],))]
    assert float(sum(g.abs().sum() for g in grads)) > 0 and haux['per_example'].shape == (3,)


def test_device_loss_formulas_are_the_hand_vectors_formulas(hand):
  """The same vectors again through `loss_fn`-level code paths of the oracle that the CUDA kernels are compared with:
  a 3-atom C51 head reduced to the projection + cross entropy above."""
  case = hand['categorical_l2_project'][0]
  z_q = t64(case['z_q'])
  r, disc = case['r_t'], case['discount_t']
  target_z = r + disc * z_q
  np.testing.assert_allclose(target_z.numpy(), case['z_p'], atol=1e-15)
