"""CPU oracle for the learner half of the hot path (TEST INFRASTRUCTURE ONLY).

PyTorch-CPU restatement (float64 by default, float32 on request) of
  * the networks in the reference's `dqn_zoo/networks.py`,
  * each agent's `loss_fn` (`dqn_zoo/<agent>/agent.py`),
  * the third-party arithmetic those call: rlax 0.1.2 (`q_learning`,
    `double_q_learning`, `clip_gradient`, `l2_loss`, `categorical_l2_project`,
    `categorical_[double_]q_learning`, `quantile_q_learning`), optax 0.1.2
    (`adam`, `rmsprop(centered=True)`, `clip_by_global_norm`) and dm-haiku 0.0.6
    layer conventions (Conv2D NHWC/HWIO VALID, Linear y = xW + b, Flatten in
    H,W,C order) — all pinned in `/root/reference/docker_requirements.txt:6-16`.

PARITY UNPINNED: none of jax/haiku/rlax/optax is installable in the build
container or on the GPU box, and the reference's own tests assert no numeric
value of any loss, gradient or optimizer step (SURVEY §4, §8(c)).  This file is
therefore the de-facto specification of the learner arithmetic ("vs restatement
of rlax/optax 0.1.2 semantics").  What IS independent: gradients come from
torch autograd over torch's own conv/matmul kernels, so the hand-written CUDA
forward/backward is checked against a second implementation, not against itself.

Randomness (IQN taus, noisy-net noise) is an INPUT here; the JAX PRNG stream is
not reproduced (SURVEY §7.2 item 4).

Only tests/, __graft_entry__.smoke() and bench.py's CPU-baseline legs import this.
"""

from __future__ import annotations

import math
from typing import Dict, NamedTuple, Optional

import numpy as np
import torch
import torch.nn.functional as F

# agent kind -> (network family, number of forward passes that use online params on s_t)
AGENT_KINDS = ('dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn')


class NetSpec(NamedTuple):
  kind: str                    # one of AGENT_KINDS
  num_actions: int
  num_atoms: int = 51          # c51 / rainbow (`c51/run_atari.py:84`, `rainbow/run_atari.py:97`)
  vmax: float = 10.0
  num_quantiles: int = 201     # qrdqn (`qrdqn/run_atari.py:83`)
  latent_dim: int = 64         # iqn (`iqn/run_atari.py:56`)
  noisy_sigma0: float = 0.1    # rainbow (`rainbow/run_atari.py:99`)
  obs_hw: int = 84             # observation height (and width, unless obs_w is given)
  obs_c: int = 4
  obs_w: Optional[int] = None  # observation width of a non-square observation; None: obs_hw


def conv_out(n, k, s):
  return (n - k) // s + 1


def feature_dim(spec):
  h = conv_out(conv_out(conv_out(spec.obs_hw, 8, 4), 4, 2), 3, 1)
  w = conv_out(conv_out(conv_out(spec.obs_hw if spec.obs_w is None else spec.obs_w, 8, 4), 4, 2), 3, 1)
  return h * w * 64


def head_out(spec):
  if spec.kind in ('dqn', 'double_q', 'prioritized', 'iqn'):
    return spec.num_actions
  if spec.kind == 'c51':
    return spec.num_actions * spec.num_atoms
  if spec.kind == 'qrdqn':
    return spec.num_quantiles * spec.num_actions
  raise ValueError(spec.kind)


def param_shapes(spec):
  """Ordered {name: shape}.  Layouts: conv w = HWIO, linear w = (in, out)
  (`networks_test.py:44,53`), shared bias shape (1,) (`networks_test.py:78`),
  noisy sigma layer always has a bias (`networks.py:160-166`)."""
  c = spec.obs_c
  d = feature_dim(spec)
  out = {
      'conv1/w': (8, 8, c, 32), 'conv1/b': (32,),
      'conv2/w': (4, 4, 32, 64), 'conv2/b': (64,),
      'conv3/w': (3, 3, 64, 64), 'conv3/b': (64,),
  }
  if spec.kind == 'rainbow':
    a, k = spec.num_actions, spec.num_atoms
    for stream, n_out in (('adv', a * k), ('val', k)):
      out[stream + '1/mu/w'] = (d, 512)
      out[stream + '1/mu/b'] = (512,)
      out[stream + '1/sigma/w'] = (d, 512)
      out[stream + '1/sigma/b'] = (512,)
      out[stream + '2/mu/w'] = (512, n_out)
      out[stream + '2/sigma/w'] = (512, n_out)
      out[stream + '2/sigma/b'] = (n_out,)
    return out
  if spec.kind == 'iqn':
    out['embed/w'] = (spec.latent_dim, d)
    out['embed/b'] = (d,)
  out['fc1/w'] = (d, 512)
  out['fc1/b'] = (512,)
  out['head/w'] = (512, head_out(spec))
  out['head/b'] = (1,) if spec.kind in ('double_q', 'prioritized') else (head_out(spec),)
  return out


def fan_in(name, shape):
  return int(np.prod(shape[:-1])) if name.endswith('/w') else None


def init_params(spec, seed):
  """Legacy U(+-1/sqrt(fan_in)) init for w AND b (`networks.py:58-79,82-134`);
  sigma = const sigma0/sqrt(in) (`networks.py:156-166`).  numpy RandomState, NOT
  JAX-identical (documented in DESIGN.md)."""
  rs = np.random.RandomState(seed)
  shapes = param_shapes(spec)
  params = {}
  for name, shape in shapes.items():
    layer = name.rsplit('/', 1)[0]
    w_shape = shapes[layer + '/w']
    n_in = int(np.prod(w_shape[:-1]))
    if '/sigma/' in name:
      params[name] = np.full(shape, spec.noisy_sigma0 / math.sqrt(n_in), dtype=np.float32)
    else:
      bound = math.sqrt(1.0 / n_in)
      params[name] = rs.uniform(-bound, bound, size=shape).astype(np.float32)
  return params


def support_atoms(spec, dtype):
  """The support is a float32 array in the reference (`rainbow/run_atari.py:146`); both the
  oracle and the CUDA path take linspace evaluated in float64 and rounded once to float32."""
  return torch.tensor(np.linspace(-spec.vmax, spec.vmax, spec.num_atoms).astype(np.float32)).to(dtype)


def noise_shapes(spec):
  """Per `network.apply`: 8 noise vectors, in `hk.next_rng_key()` call order
  (`networks.py:169-170`, `:235-248`): adv1 in/out, adv2 in/out, val1 in/out, val2 in/out."""
  d = feature_dim(spec)
  a, k = spec.num_actions, spec.num_atoms
  return [('adv1/in', d), ('adv1/out', 512), ('adv2/in', 512), ('adv2/out', a * k),
          ('val1/in', d), ('val1/out', 512), ('val2/in', 512), ('val2/out', k)]


# ----------------------------------------------------------------------------
# networks (`networks.py`)
# ----------------------------------------------------------------------------


def dueling(adv, val):
  """`networks.py:251`: logits [B,A,K] of advantages [B,A,K] and values [B,K]."""
  return val[:, None, :] + adv - adv.mean(dim=1, keepdim=True)


def _conv(x, w, b, stride):
  """hk.Conv2D VALID, NHWC activations, HWIO weights (`networks.py:82-103`)."""
  y = F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), b, stride=stride)
  return y.permute(0, 2, 3, 1)


class ReluTap:
  """Test instrumentation for the ReLU kinks of ONE network apply.  `pre[name]` records every pre-activation; if
  `masks[name]` (bool, same shape) is given, relu(x) is replaced by x * mask, i.e. the gradient is evaluated on the
  given activation pattern.  The GPU tests use it to separate two things the 1e-5 gradient bar mixes up: arithmetic
  error, and units whose float64 pre-activation is within float32 rounding of zero and therefore legitimately fall
  on the other side of the kink in ANY float32 evaluation (each flips one 0/1 factor of the gradient)."""

  def __init__(self, masks=None):
    self.pre = {}
    self.masks = masks or {}

  def relu(self, x, name):
    self.pre[name] = x.detach()
    if name in self.masks:
      return x * self.masks[name].to(x.dtype).reshape(x.shape)
    return F.relu(x)


def _relu(x, tap, name):
  return F.relu(x) if tap is None else tap.relu(x, name)


def torso(p, obs_u8, dtype, tap=None):
  """`networks.py:181-204`: /255, three conv+relu, flatten in (H,W,C) order."""
  x = obs_u8.to(dtype) / 255.0
  x = _relu(_conv(x, p['conv1/w'], p['conv1/b'], 4), tap, 'conv1')
  x = _relu(_conv(x, p['conv2/w'], p['conv2/b'], 2), tap, 'conv2')
  x = _relu(_conv(x, p['conv3/w'], p['conv3/b'], 1), tap, 'conv3')
  return x.reshape(x.shape[0], -1)


def _noisy(p, prefix, x, eps_in, eps_out, with_bias):
  """`networks.py:137-178`: mu(x) + sigma(eps_in * x) * eps_out; sigma always biased."""
  mu = x @ p[prefix + '/mu/w']
  if with_bias:
    mu = mu + p[prefix + '/mu/b']
  sig = (eps_in * x) @ p[prefix + '/sigma/w'] + p[prefix + '/sigma/b']
  return mu + sig * eps_out


def apply_net(spec, p, obs_u8, dtype, taus=None, noise=None, tap=None):
  """One `network.apply`.  Returns dict with the NamedTuple fields of
  `networks.py:34-55` for the family.  `tap`: optional ReluTap (tests)."""
  feat = torso(p, obs_u8, dtype, tap)
  kind = spec.kind
  a = spec.num_actions
  if kind == 'rainbow':
    k = spec.num_atoms
    n = {name: noise[name].to(dtype)[None, :] for name, _ in noise_shapes(spec)}
    adv = _relu(_noisy(p, 'adv1', feat, n['adv1/in'], n['adv1/out'], True), tap, 'adv1')
    adv = _noisy(p, 'adv2', adv, n['adv2/in'], n['adv2/out'], False).reshape(-1, a, k)
    val = _relu(_noisy(p, 'val1', feat, n['val1/in'], n['val1/out'], True), tap, 'val1')
    val = _noisy(p, 'val2', val, n['val2/in'], n['val2/out'], False).reshape(-1, 1, k)
    logits = dueling(adv, val[:, 0, :])
    support = support_atoms(spec, dtype)
    q = (F.softmax(logits, dim=-1) * support).sum(-1).detach()
    return {'q_logits': logits, 'q_values': q, 'adv': adv, 'val': val[:, 0, :]}
  if kind == 'iqn':
    # `networks.py:264-292`
    latent = spec.latent_dim
    # The product pi*i*tau is formed in float32 in the reference (argument up to ~201, so its
    # float32 rounding is worth ~1e-5 in cos); the oracle keeps that rounding, then widens.
    pi_mult = torch.arange(1, latent + 1, dtype=torch.float32) * float(np.float32(np.pi))
    arg = (pi_mult[None, None, :] * taus.to(torch.float32)[:, :, None]).to(dtype)
    emb = torch.cos(arg)                                                     # [B,N,latent]
    emb = _relu(emb @ p['embed/w'] + p['embed/b'], tap, 'embed')              # [B,N,D]
    h = emb * feat[:, None, :]
    h = _relu(h @ p['fc1/w'] + p['fc1/b'], tap, 'fc1')
    q_dist = h @ p['head/w'] + p['head/b']                                   # [B,N,A]
    return {'q_dist': q_dist, 'q_values': q_dist.mean(dim=1).detach()}
  h = _relu(feat @ p['fc1/w'] + p['fc1/b'], tap, 'fc1')
  out = h @ p['head/w'] + p['head/b']          # shared bias (1,) broadcasts (`networks.py:130-132`)
  if kind in ('dqn', 'double_q', 'prioritized'):
    return {'q_values': out}
  if kind == 'c51':
    k = spec.num_atoms
    logits = out.reshape(-1, a, k)
    support = support_atoms(spec, dtype)
    q = (F.softmax(logits, dim=-1) * support).sum(-1).detach()
    return {'q_logits': logits, 'q_values': q}
  if kind == 'qrdqn':
    q_dist = out.reshape(-1, spec.num_quantiles, a)   # quantile-major (`networks.py:308`)
    return {'q_dist': q_dist, 'q_values': q_dist.mean(dim=1).detach()}
  raise ValueError(kind)


# ----------------------------------------------------------------------------
# rlax 0.1.2 restatements
# ----------------------------------------------------------------------------


class _ClipGrad(torch.autograd.Function):
  """rlax.clip_gradient: identity forward, cotangent clipped to [lo, hi]."""

  @staticmethod
  def forward(ctx, x, lo, hi):
    ctx.lo, ctx.hi = lo, hi
    return x.clone()

  @staticmethod
  def backward(ctx, g):
    return g.clamp(ctx.lo, ctx.hi), None, None


def categorical_l2_project(z_p, probs, z_q):
  """rlax.categorical_l2_project, batched over the leading dim.
  z_p [B,Kp] target atoms, probs [B,Kp], z_q [Kq] support -> [B,Kq]."""
  d_pos = torch.roll(z_q, -1) - z_q
  d_neg = z_q - torch.roll(z_q, 1)
  d_pos = torch.where(d_pos > 0, 1.0 / d_pos, torch.zeros_like(d_pos))[None, :, None]
  d_neg = torch.where(d_neg > 0, 1.0 / d_neg, torch.zeros_like(d_neg))[None, :, None]
  z_p = z_p.clamp(z_q[0], z_q[-1])[:, None, :]
  delta = z_p - z_q[None, :, None]                      # [B,Kq,Kp]
  sign = (delta >= 0).to(delta.dtype)
  delta_hat = sign * delta * d_pos - (1.0 - sign) * delta * d_neg
  return ((1.0 - delta_hat).clamp(0.0, 1.0) * probs[:, None, :]).sum(-1)


def huber(x, kappa):
  """rlax.huber_loss: 0.5*min(|x|,k)^2 + k*(|x| - min(|x|,k)); no division by k."""
  ax = x.abs()
  quad = torch.clamp(ax, max=kappa)
  return 0.5 * quad * quad + kappa * (ax - quad)


def quantile_regression_loss(dist_src, tau_src, dist_target, kappa):
  """rlax.quantile_regression_loss batched: src [B,N], tau [B,N] or [N], target [B,M] -> [B]."""
  delta = dist_target[:, None, :] - dist_src[:, :, None]       # [B,N,M]
  neg = (delta < 0).to(delta.dtype).detach()
  if tau_src.dim() == 1:
    tau_src = tau_src[None, :]
  weight = (tau_src[:, :, None] - neg).abs()
  loss = huber(delta, kappa) if kappa > 0 else delta.abs()
  return (loss * weight).mean(-1).sum(-1)


# ----------------------------------------------------------------------------
# loss functions (one per agent)
# ----------------------------------------------------------------------------


def loss_fn(spec, online, target, batch, dtype, weights=None, taus=None, noise=None,
            grad_error_bound=1.0 / 32, huber_param=1.0, tap=None):
  """Returns (scalar loss, aux dict).  `batch` = dict(s_tm1,a_tm1,r_t,discount_t,s_t) of
  torch tensors; r_t/discount_t are cast to `dtype` AFTER a float32 rounding, as the
  reference feeds float32 into jit.  Cites: dqn `dqn/agent.py:85-107`, double_q
  `double_q/agent.py:85-111`, prioritized `prioritized/agent.py:86-113`, c51
  `c51/agent.py:87-107`, qrdqn `qrdqn/agent.py:88-110`, rainbow `rainbow/agent.py:85-109`,
  iqn `iqn/agent.py:178-214`."""
  kind = spec.kind
  s_tm1, s_t = batch['s_tm1'], batch['s_t']
  if kind in ('dqn', 'double_q', 'prioritized', 'c51', 'qrdqn'):
    heads = [apply_net(spec, online, s_tm1, dtype, tap=tap), None, apply_net(spec, target, s_t, dtype)]
    if kind in ('double_q', 'prioritized'):
      heads[1] = apply_net(spec, online, s_t, dtype)
  elif kind == 'rainbow':
    nz = noise or [None, None, None]
    heads = [apply_net(spec, online, s_tm1, dtype, noise=nz[0], tap=tap), apply_net(spec, online, s_t, dtype, noise=nz[1]),
             apply_net(spec, target, s_t, dtype, noise=nz[2])]
  elif kind == 'iqn':
    heads = [apply_net(spec, online, s_tm1, dtype, taus=taus[0], tap=tap), apply_net(spec, target, s_t, dtype, taus=taus[1]),
             apply_net(spec, target, s_t, dtype, taus=taus[2])]
  else:
    raise ValueError(kind)
  field = {'c51': 'q_logits', 'qrdqn': 'q_dist', 'iqn': 'q_dist'}.get(kind, 'q_values')
  if kind == 'rainbow':
    heads = [(h['adv'], h['val']) for h in heads]
  else:
    heads = [None if h is None else h[field] for h in heads]
  loss, aux = head_loss(kind, heads, batch['a_tm1'], batch['r_t'], batch['discount_t'], weights,
                        None if taus is None else taus[0], vmax=spec.vmax, grad_error_bound=grad_error_bound,
                        huber_param=huber_param, grad=False)
  return loss, aux


def head_loss(kind, heads, a_tm1, r_t, discount_t, weights=None, taus=None, *, vmax=10.0, grad_error_bound=1.0 / 32,
              huber_param=1.0, grad=True):
  """The loss of each agent from its head outputs: everything `loss_fn` does after the network applies.

  heads: the three passes (online(s_tm1), selector, target(s_t)) in `dtype`, as the device lays them out:
    dqn [B,A] with heads[1] unused (None); double_q / prioritized [B,A], heads[1] online(s_t);
    c51 [B,A,K] logits, heads[1] unused (the target pass selects); rainbow (adv [B,A,K], val [B,K]) per pass,
    heads[1] online(s_t); qrdqn [B,N,A], heads[1] unused; iqn [B,N,A] at (tau_tm1, tau_policy, tau_t).
  taus: iqn's s_tm1 taus [B,N].  r_t / discount_t / weights are rounded to float32 first, as the reference feeds float32.
  Returns (scalar loss, aux): aux 'losses' [B], 'per_example' (td for the dqn family, the loss otherwise),
  'priorities' (prioritized |td|, rainbow clip(|loss|, 0, 100)), 'a_star' (the selected action; dqn: argmax of the
  target pass) and, with grad=True, 'grad': the gradient of the loss wrt the pass-0 head outputs (rainbow: a tuple
  (d adv, d val)), by autograd.  grad=False leaves the pass-0 tensors in the caller's graph (loss_fn)."""
  dtype = (heads[0][0] if kind == 'rainbow' else heads[0]).dtype
  a_tm1 = torch.as_tensor(a_tm1).long()
  r = torch.as_tensor(r_t).to(torch.float32).to(dtype)
  disc = torch.as_tensor(discount_t).to(torch.float32).to(dtype)
  pass0 = list(heads[0]) if kind == 'rainbow' else [heads[0]]
  if grad:
    pass0 = [x.detach().clone().requires_grad_(True) for x in pass0]
  rows = torch.arange(a_tm1.shape[0])
  aux = {}
  if kind in ('dqn', 'double_q', 'prioritized'):
    q_tm1 = pass0[0]
    q_target = heads[2].detach()
    sel = q_target if kind == 'dqn' else heads[1].detach()
    a_star = sel.argmax(dim=1)                 # first maximum, as jnp.argmax
    boot = q_target.max(dim=1).values if kind == 'dqn' else q_target[rows, a_star]
    td = (r + disc * boot).detach() - q_tm1[rows, a_tm1]
    aux['td_errors'] = td.detach()
    td_c = _ClipGrad.apply(td, -grad_error_bound, grad_error_bound)
    losses = 0.5 * td_c * td_c
    aux['q_tm1'] = q_tm1.detach()
  elif kind in ('c51', 'rainbow'):
    if kind == 'rainbow':
      logits_tm1 = dueling(*pass0)
      sel_logits = dueling(*[x.detach() for x in heads[1]])
      tgt_logits = dueling(*[x.detach() for x in heads[2]])
    else:
      logits_tm1, tgt_logits = pass0[0], heads[2].detach()
      sel_logits = tgt_logits
    support = torch.tensor(np.linspace(-vmax, vmax, logits_tm1.shape[-1]).astype(np.float32)).to(dtype)
    sel_q = (F.softmax(sel_logits, dim=-1) * support).sum(-1)
    a_star = sel_q.argmax(dim=1)
    p_target = F.softmax(tgt_logits[rows, a_star], dim=-1)
    target_z = r[:, None] + disc[:, None] * support[None, :]
    proj = categorical_l2_project(target_z, p_target, support).detach()
    logit_qa = logits_tm1[rows, a_tm1]
    losses = -(proj * F.log_softmax(logit_qa, dim=-1)).sum(-1)
    aux['logits_tm1'] = logits_tm1.detach()
    aux['target_probs'] = proj
    aux['p_target'] = p_target
  elif kind in ('qrdqn', 'iqn'):
    dist_tm1, dist_t = pass0[0], heads[2].detach()
    if kind == 'qrdqn':
      n = dist_tm1.shape[1]
      tau_src = ((torch.arange(0, n, dtype=torch.float32) + 0.5) / float(n)).to(dtype)   # `qrdqn/run_atari.py:136-137`
      sel = dist_t
    else:
      tau_src = torch.as_tensor(taus).to(dtype)
      sel = heads[1].detach()
    a_star = sel.mean(dim=1).argmax(dim=1)
    tgt = (r[:, None] + disc[:, None] * dist_t[rows, :, a_star]).detach()
    losses = quantile_regression_loss(dist_tm1[rows, :, a_tm1], tau_src, tgt, huber_param)
    aux['dist_tm1'] = dist_tm1.detach()
    aux['targets'] = tgt
  else:
    raise ValueError(kind)
  return _finish(kind, losses, weights, pass0, grad, dict(aux, a_star=a_star))


def _finish(kind, losses, weights, pass0, grad, aux):
  """The weighted mean, the per-example values and priorities of `head_loss` and, with grad, its pass-0 gradient."""
  dtype = losses.dtype
  aux['losses'] = losses.detach()
  w = None if weights is None else torch.as_tensor(weights).to(torch.float32).to(dtype)
  loss = losses.mean() if w is None else (losses * w).mean()
  aux['per_example'] = aux['td_errors'] if kind in ('dqn', 'double_q', 'prioritized') else aux['losses']
  if kind == 'rainbow':
    aux['priorities'] = aux['losses'].abs().clamp(0.0, 100.0)       # `rainbow/agent.py:194`
  elif kind == 'prioritized':
    aux['priorities'] = aux['td_errors'].abs()                       # `prioritized/agent.py:201`
  if grad:
    g = torch.autograd.grad(loss, pass0, allow_unused=True)
    g = [torch.zeros_like(x) if gi is None else gi for x, gi in zip(pass0, g)]
    aux['grad'] = tuple(g) if kind == 'rainbow' else g[0]
  return loss, aux


# ----------------------------------------------------------------------------
# optax 0.1.2 restatements
# ----------------------------------------------------------------------------


class OptSpec(NamedTuple):
  name: str                  # 'adam' | 'rmsprop'
  learning_rate: float
  eps: float
  decay: float = 0.95        # rmsprop
  b1: float = 0.9
  b2: float = 0.999
  max_global_grad_norm: float = 0.0   # 0 = no clip


def default_opt(kind):
  """Hyper-parameters per agent (SURVEY §5.1 with run_atari cites)."""
  if kind in ('dqn', 'double_q'):
    return OptSpec('rmsprop', 0.00025, 0.01 / 32 ** 2)
  if kind == 'prioritized':
    return OptSpec('rmsprop', 0.00025 / 4, 0.01 / 32 ** 2 / 16)   # `prioritized/run_atari.py:92-99`
  if kind == 'c51':
    return OptSpec('adam', 0.00025, 0.01 / 32, max_global_grad_norm=10.0)
  if kind == 'qrdqn':
    return OptSpec('adam', 0.00005, 0.01 / 32, max_global_grad_norm=10.0)
  if kind == 'rainbow':
    return OptSpec('adam', 0.0000625, 0.005 / 32, max_global_grad_norm=10.0)
  if kind == 'iqn':
    return OptSpec('adam', 0.00005, 0.01 / 32)
  raise ValueError(kind)


def init_opt_state(opt, params):
  z = {k: torch.zeros_like(v) for k, v in params.items()}
  if opt.name == 'adam':
    return {'count': 0, 'mu': z, 'nu': {k: torch.zeros_like(v) for k, v in params.items()}}
  return {'mu': z, 'nu': {k: torch.zeros_like(v) for k, v in params.items()}}


def optimizer_step(opt, params, grads, state):
  """optax.chain(clip_by_global_norm?, adam | rmsprop(centered)) then apply_updates.
  Returns (new_params, new_state, global_norm)."""
  gn = torch.sqrt(sum((g * g).sum() for g in grads.values()))
  if opt.max_global_grad_norm > 0 and not bool(gn < opt.max_global_grad_norm):
    grads = {k: (g / gn) * opt.max_global_grad_norm for k, g in grads.items()}
  new_p, mu_n, nu_n = {}, {}, {}
  if opt.name == 'adam':
    count = state['count'] + 1
    c1 = 1.0 - opt.b1 ** count
    c2 = 1.0 - opt.b2 ** count
    for k, g in grads.items():
      mu = opt.b1 * state['mu'][k] + (1.0 - opt.b1) * g
      nu = opt.b2 * state['nu'][k] + (1.0 - opt.b2) * g * g
      upd = (mu / c1) / (torch.sqrt(nu / c2) + opt.eps)
      new_p[k] = params[k] - opt.learning_rate * upd
      mu_n[k], nu_n[k] = mu, nu
    return new_p, {'count': count, 'mu': mu_n, 'nu': nu_n}, gn
  for k, g in grads.items():
    mu = opt.decay * state['mu'][k] + (1.0 - opt.decay) * g
    nu = opt.decay * state['nu'][k] + (1.0 - opt.decay) * g * g
    upd = g * torch.rsqrt(nu - mu * mu + opt.eps)
    new_p[k] = params[k] - opt.learning_rate * upd
    mu_n[k], nu_n[k] = mu, nu
  return new_p, {'mu': mu_n, 'nu': nu_n}, gn


# ----------------------------------------------------------------------------
# one learner update (`<agent>/agent.py` `update` + `_learn` priority rule)
# ----------------------------------------------------------------------------


class Learner:
  """Holds params/opt-state as torch tensors in `dtype`; `update()` is one jit(update)."""

  def __init__(self, spec, params_np, opt=None, dtype=torch.float64, grad_error_bound=1.0 / 32, huber_param=1.0):
    self.spec, self.dtype = spec, dtype
    self.opt = opt or default_opt(spec.kind)
    self.grad_error_bound, self.huber_param = grad_error_bound, huber_param
    self.online = {k: torch.tensor(v, dtype=dtype) for k, v in params_np.items()}
    self.target = {k: v.clone() for k, v in self.online.items()}
    self.state = init_opt_state(self.opt, self.online)

  def grads(self, batch, weights=None, taus=None, noise=None, tap=None):
    p = {k: v.clone().requires_grad_(True) for k, v in self.online.items()}
    loss, aux = loss_fn(self.spec, p, self.target, batch, self.dtype, weights, taus, noise,
                        grad_error_bound=self.grad_error_bound, huber_param=self.huber_param, tap=tap)
    loss.backward()
    g = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return loss.detach(), aux, g

  def update(self, batch, weights=None, taus=None, noise=None, tap=None):
    loss, aux, g = self.grads(batch, weights, taus, noise, tap=tap)
    self.online, self.state, gn = optimizer_step(self.opt, self.online, g, self.state)
    aux = dict(aux, loss=loss, grads=g, global_norm=gn)
    # priority rule: rainbow clip(|losses|,0,100) (`rainbow/agent.py:194`), prioritized |td| (`prioritized/agent.py:201`)
    if self.spec.kind == 'rainbow':
      aux['priorities'] = aux['losses'].abs().clamp(0.0, 100.0).to(torch.float32)
    elif self.spec.kind == 'prioritized':
      aux['priorities'] = aux['td_errors'].abs().to(torch.float32)
    return aux

  def sync_target(self):
    self.target = {k: v.clone() for k, v in self.online.items()}


def batch_from_numpy(s_tm1, a_tm1, r_t, discount_t, s_t):
  return {'s_tm1': torch.as_tensor(np.ascontiguousarray(s_tm1)), 'a_tm1': torch.as_tensor(np.asarray(a_tm1)),
          'r_t': torch.as_tensor(np.asarray(r_t, dtype=np.float64)),
          'discount_t': torch.as_tensor(np.asarray(discount_t, dtype=np.float64)),
          's_t': torch.as_tensor(np.ascontiguousarray(s_t))}
