"""CPU: noisy networks (DESIGN.md §17) of dqn, double_q, prioritized and munchausen, plain and dueling.

- the float64 oracle (oracle/noisy_oracle.py): autograd against central differences of each kind's loss for every
  tensor, sigma tensors included; the factorised identity; the sigma = 0 limit against the plain and dueling oracles,
  with the sigma gradients in closed form;
- the C ABI and the Python surface: the parameter layout, the noise sizes and slots, and the rejection of noisy=True
  for every other kind.
"""

import ctypes as C

import numpy as np
import pytest
import torch

from oracle import dueling_oracle as do
from oracle import learner_oracle as lo
from oracle import noisy_oracle as no

KINDS = no.KINDS
OTHER_KINDS = ('c51', 'qrdqn', 'rainbow', 'iqn', 'munchausen_iqn', 'fqf')


def _noise(spec, dueling, rs):
  one = {}
  for name, n in no.noise_shapes(spec, dueling):
    x = np.clip(rs.standard_normal(n), -2, 2)
    one[name] = torch.tensor(np.sign(x) * np.sqrt(np.abs(x)))
  return one


def _case(kind, dueling, A=6, hw=36, B=4, seed=0, sigma0=0.1):
  spec = lo.NetSpec(kind, A, obs_hw=hw, noisy_sigma0=sigma0)
  rs = np.random.RandomState(seed)
  online = {k: torch.tensor(v, dtype=torch.float64) for k, v in no.init_params(spec, seed, dueling).items()}
  target = {k: torch.tensor(v, dtype=torch.float64) for k, v in no.init_params(spec, seed + 1, dueling).items()}
  # larger sigmas than the init's, so that the sigma terms are not small beside mu in the checks below
  for p in (online, target):
    for k in p:
      if '/sigma/' in k:
        p[k] = p[k] * 5.0 + torch.tensor(rs.uniform(-0.02, 0.02, p[k].shape))
  s = rs.randint(0, 256, (2, B, hw, hw, 4)).astype(np.uint8)
  batch = lo.batch_from_numpy(s[0], rs.randint(0, A, B), rs.choice([-1.0, 0.0, 1.0], B), rs.choice([0.0, 0.99], B), s[1])
  w = torch.tensor(rs.uniform(0.1, 1.0, B)) if kind == 'prioritized' else None
  noise = [_noise(spec, dueling, rs) for _ in range(3)]
  return spec, online, target, batch, w, noise


def _loss(spec, p, target, batch, w, noise, dueling):
  # a clip far above every td: rlax.clip_gradient clips the gradient, not the loss
  return no.loss_fn(spec, p, target, batch, torch.float64, noise, dueling, w, grad_error_bound=1e6)[0]


# ---- the oracle ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dueling', [False, True], ids=['plain', 'dueling'])
@pytest.mark.parametrize('kind', KINDS)
def test_autograd_matches_central_differences_for_every_tensor(kind, dueling):
  spec, online, target, batch, w, noise = _case(kind, dueling)
  p = {k: v.clone().requires_grad_(True) for k, v in online.items()}
  _loss(spec, p, target, batch, w, noise, dueling).backward()
  rs = np.random.RandomState(1)
  h = 1e-6
  assert any('/sigma/' in k for k in online)
  for name, value in online.items():
    d = torch.tensor(rs.standard_normal(value.shape))
    d /= d.norm()
    plus = {k: (v + h * d if k == name else v) for k, v in online.items()}
    minus = {k: (v - h * d if k == name else v) for k, v in online.items()}
    fd = float(_loss(spec, plus, target, batch, w, noise, dueling) - _loss(spec, minus, target, batch, w, noise, dueling)) / (2 * h)
    ad = float((p[name].grad * d).sum())
    scale = max(float(p[name].grad.norm()), 1e-8)
    assert abs(fd - ad) <= 1e-6 * scale, (kind, name, fd, ad)


@pytest.mark.parametrize('dueling', [False, True], ids=['plain', 'dueling'])
def test_a_noisy_layer_is_a_linear_layer_with_the_factorised_weight(dueling):
  """noisy(x) = x W + b with W = mu_w + sigma_w * (eps_in eps_out^T) and b = mu_b + sigma_b * eps_out."""
  spec, p, _, batch, _, noise = _case('dqn', dueling)
  n = noise[0]
  feat = lo.torso(p, batch['s_tm1'], torch.float64)
  for name, n_in, n_out in no.layers(spec, dueling):
    x = feat if n_in != 512 else torch.tensor(np.random.RandomState(n_out).standard_normal((feat.shape[0], 512)))
    W = p[name + '/mu/w'] + p[name + '/sigma/w'] * torch.outer(n[name + '/in'], n[name + '/out'])
    b = p[name + '/mu/b'] + p[name + '/sigma/b'] * n[name + '/out']
    got = lo._noisy(p, name, x, n[name + '/in'][None], n[name + '/out'][None], True)
    torch.testing.assert_close(got, x @ W + b, rtol=1e-12, atol=1e-12)


def _zero_sigma(p):
  return {k: (torch.zeros_like(v) if '/sigma/' in k else v) for k, v in p.items()}


def _as_plain(p):
  """The noiseless oracles' parameters: a noisy network's mu tensors under the plain names."""
  return {k.replace('/mu', ''): v for k, v in p.items() if '/sigma/' not in k}


@pytest.mark.parametrize('dueling', [False, True], ids=['plain', 'dueling'])
@pytest.mark.parametrize('kind', KINDS)
def test_zero_sigma_is_the_noiseless_network_and_sigma_gradients_are_closed_form(kind, dueling):
  spec, online, target, batch, w, noise = _case(kind, dueling)
  on0, tg0 = _zero_sigma(online), _zero_sigma(target)
  p = {k: v.clone().requires_grad_(True) for k, v in on0.items()}
  loss, _ = no.loss_fn(spec, p, tg0, batch, torch.float64, noise, dueling, w)
  loss.backward()
  # the noiseless oracle on the mu tensors: the dueling oracle, or learner_oracle's dqn network (whose head bias is
  # per action for every kind: double_q's and prioritized's shared bias gives way to the mu bias)
  mu_on, mu_tg = _as_plain(on0), _as_plain(tg0)
  q = lambda pp, s: (do.apply_net(spec, pp, s, torch.float64) if dueling else
                     lo.apply_net(spec._replace(kind='dqn'), pp, s, torch.float64))['q_values']
  s_tm1, s_t = batch['s_tm1'], batch['s_t']
  for pp, ppn, s, slot in ((mu_on, on0, s_tm1, 0), (mu_tg, tg0, s_t, 2), (mu_on, on0, s_t, 1)):
    torch.testing.assert_close(no.apply_net(spec, ppn, s, torch.float64, noise[slot], dueling)['q_values'], q(pp, s),
                               rtol=1e-12, atol=1e-12)
  # sigma gradients: dL/dsigma_w = (x * eps_in)^T (g * eps_out) = dL/dmu_w * eps_in eps_out^T summed over the batch,
  # which is (eps_in eps_out^T) * dL/dmu_w for one noise apply; dL/dsigma_b = dL/dmu_b * eps_out.  Only slot 0
  # (online(s_tm1)) carries gradient.
  n = noise[0]
  for name, _, _ in no.layers(spec, dueling):
    gw, gb = p[name + '/mu/w'].grad, p[name + '/mu/b'].grad
    if gw is None:
      continue
    torch.testing.assert_close(p[name + '/sigma/w'].grad, gw * torch.outer(n[name + '/in'], n[name + '/out']),
                               rtol=1e-10, atol=1e-14)
    torch.testing.assert_close(p[name + '/sigma/b'].grad, gb * n[name + '/out'], rtol=1e-10, atol=1e-14)


class _Recording(dict):
  read = False

  def __getitem__(self, key):
    self.read = True
    return dict.__getitem__(self, key)


def test_slots_follow_the_passes():
  """The loss reads noise slot k exactly when a pass of the kind applies it (dqn: slot 1 is unread)."""
  for kind in KINDS:
    for dueling in (False, True):
      spec, online, target, batch, w, noise = _case(kind, dueling)
      rec = [_Recording(one) for one in noise]
      _loss(spec, online, target, batch, w, rec, dueling)
      reads = [s for s in no.slot_of_pass(kind) if s is not None]
      assert [k for k in range(3) if rec[k].read] == reads, (kind, dueling)


# ---- the C ABI and the Python surface --------------------------------------------------------------------------------

def _cfg(kind, noisy, dueling=0, A=6, hw=84):
  from dqn_zoo_b200 import _lib
  cfg = _lib.LearnerConfig(kind=_lib.AGENT_KINDS[kind], num_actions=A, num_atoms=51, num_quantiles=201, latent_dim=64,
                           tau_samples_s_tm1=64, tau_samples_policy=64, tau_samples_s_t=64, batch=32, obs_h=hw, obs_w=hw,
                           obs_c=4, learning_rate=1e-4, opt_eps=1e-5, rms_decay=0.95, adam_b1=0.9, adam_b2=0.999,
                           munchausen_alpha=0.9, entropy_temperature=0.03, log_policy_clip=-1.0)
  cfg.dueling, cfg.noisy = dueling, noisy
  return cfg


def _tensors(cfg):
  from dqn_zoo_b200 import _lib
  plan = _lib.LearnerPlan()
  _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(plan))
  name, shape = C.create_string_buffer(64), (C.c_int64 * 4)()
  ndim, off = C.c_int32(), C.c_int64()
  out = []
  for i in range(plan.num_tensors):
    _lib.call('dz_learner_tensor_info', C.byref(cfg), i, name, shape, C.byref(ndim), C.byref(off))
    out.append((name.value.decode(), tuple(shape[k] for k in range(ndim.value)), off.value))
  return plan, out


@pytest.mark.parametrize('dueling', [0, 1], ids=['plain', 'dueling'])
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('A,hw', [(6, 84), (1, 84), (18, 44), (64, 84)])
def test_layout_noise_sizes_and_stride(kind, dueling, A, hw):
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  A = min(A, 18) if kind == 'munchausen' else A
  cfg = _cfg(kind, 1, dueling, A, hw)
  plan, tensors = _tensors(cfg)
  spec = lo.NetSpec(kind, A, obs_hw=hw)
  assert [(n, s) for n, s, _ in tensors] == list(no.param_shapes(spec, dueling).items())
  first = 'adv1' if dueling else 'fc1'
  assert [n for n, _, _ in tensors][6:10] == [first + '/mu/w', first + '/mu/b', first + '/sigma/w', first + '/sigma/b']
  end = 0
  for n, s, off in tensors:
    assert off % 4 == 0 and off >= end, n
    end = off + int(np.prod(s))
  net = dl.NetworkSpec(kind, A, obs_shape=(hw, hw, 4), dueling=bool(dueling), noisy=True)
  sizes = dl.noise_vector_sizes(net)
  assert sizes == no.noise_shapes(spec, dueling)
  stride = C.c_int64()
  _lib.call('dz_learner_noise_stride', C.byref(cfg), C.byref(stride))
  assert stride.value == sum((n + 3) // 4 * 4 for _, n in sizes)
  assert plan.noise_floats == 3 * stride.value and plan.tau_floats == 0
  rs = np.random.RandomState(A)
  applies = [{n: rs.standard_normal(k).astype(np.float32) for n, k in sizes} for _ in range(3)]
  packed = dl.pack_noise(net, applies)
  assert packed.size == plan.noise_floats
  at = 0
  for one in applies:   # every vector starts on a 4-float boundary
    for n, k in sizes:
      np.testing.assert_array_equal(packed[at:at + k], one[n])
      at += (k + 3) // 4 * 4
  # the network without noise is unchanged by the field's existence
  assert _tensors(_cfg(kind, 0, dueling, A, hw))[0].noise_floats == 0


def test_slot_mapping_per_kind():
  assert no.slot_of_pass('dqn') == (0, None, 2)
  for kind in ('double_q', 'prioritized', 'munchausen'):
    assert no.slot_of_pass(kind) == (0, 1, 2)


@pytest.mark.parametrize('kind', OTHER_KINDS)
def test_other_kinds_reject_noisy(kind):
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  cfg = _cfg(kind, 1)
  with pytest.raises(ValueError, match='noisy'):
    _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(_lib.LearnerPlan()))
  bufs = _lib.LearnerBuffers(0, 0, 0, 0, 0, 0)
  with pytest.raises(ValueError, match='noisy'):
    _lib.call('dz_learner_create', C.byref(cfg), C.byref(bufs), C.byref(C.c_void_p()))
  _tensors(_cfg(kind, 0))   # the same configuration without the field is valid
  with pytest.raises(ValueError, match='noisy' if kind != 'rainbow' else 'noisy already'):
    dl.Learner(dl.NetworkSpec(kind, 6, noisy=True))


def test_noisy_field_must_be_zero_or_one():
  from dqn_zoo_b200 import _lib
  with pytest.raises(ValueError, match='noisy'):
    _lib.call('dz_learner_plan_query', C.byref(_cfg('dqn', 2)), C.byref(_lib.LearnerPlan()))


def test_noise_calls_still_refuse_networks_without_noise():
  from dqn_zoo_b200 import _lib
  for kind in ('dqn', 'double_q', 'c51', 'iqn'):
    with pytest.raises(ValueError):
      _lib.call('dz_learner_noise_stride', C.byref(_cfg(kind, 0)), C.byref(C.c_int64()))


def test_haiku_names_are_stable_and_distinct():
  from dqn_zoo_b200 import learner as dl
  for dueling in (False, True):
    names = list(no.param_shapes(lo.NetSpec('dqn', 6), dueling))
    mods = [dl.haiku_name(n, 'dqn') for n in names]
    assert len(set(mods)) == len(mods)
  assert dl.haiku_name('fc1/mu/w', 'dqn') == ('sequential/sequential_1/noisy_linear/mu', 'w')
  assert dl.haiku_name('head/sigma/b', 'double_q') == ('sequential/sequential_1/noisy_linear_1/sigma', 'b')
  assert dl.haiku_name('adv2/mu/b', 'prioritized') == ('dueling/advantage/noisy_linear_1/mu', 'b')
  assert dl.haiku_name('val1/sigma/w', 'munchausen') == ('dueling/value/noisy_linear/sigma', 'w')
  assert dl.haiku_name('adv1/mu/w', 'rainbow') == ('noisy_linear/mu', 'w')   # rainbow's names are unchanged
  assert dl.haiku_name('fc1/w', 'dqn') == ('sequential/sequential_1/linear', 'w')
