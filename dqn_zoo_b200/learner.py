"""Host wrapper of the CUDA learner (`dz_learner_*` in include/dqn_zoo_b200.h).

Replaces the `jax.jit(update)` closure + `_learn()` glue of every dqn_zoo agent
(`dqn/agent.py:109-119,179-189`, `rainbow/agent.py:111-123,181-198`, ...).  The network and
optimizer are declarative (`kind`, hyper-parameters) instead of `hk.Transformed` /
`optax.GradientTransformation` objects, which cannot cross into CUDA; that is the one place the
agent constructor surface differs from the reference (SURVEY §8(b)).

PyTorch tensors are used purely as device memory; all math runs in csrc/*.cu.
"""

from __future__ import annotations

import ctypes as C
import math
from typing import Dict, Mapping, NamedTuple, Optional

import numpy as np
import torch

from dqn_zoo_b200 import _lib


class OptimizerSpec(NamedTuple):
  """optax stand-in: 'adam' (+ optional clip_by_global_norm) or centred 'rmsprop'."""
  name: str
  learning_rate: float
  eps: float
  decay: float = 0.95
  b1: float = 0.9
  b2: float = 0.999
  max_global_grad_norm: float = 0.0


def default_optimizer(kind: str) -> OptimizerSpec:
  """Per-agent optimizers from the reference's run_atari flags (SURVEY §5.1)."""
  if kind in ('dqn', 'double_q'):
    return OptimizerSpec('rmsprop', 0.00025, 0.01 / 32 ** 2)             # dqn/run_atari.py:205-210
  if kind == 'prioritized':
    return OptimizerSpec('rmsprop', 0.00025 / 4, 0.01 / 32 ** 2 / 16)    # prioritized/run_atari.py:92-99
  if kind == 'c51':
    return OptimizerSpec('adam', 0.00025, 0.01 / 32, max_global_grad_norm=10.0)
  if kind == 'qrdqn':
    return OptimizerSpec('adam', 0.00005, 0.01 / 32, max_global_grad_norm=10.0)
  if kind == 'rainbow':
    return OptimizerSpec('adam', 0.0000625, 0.005 / 32, max_global_grad_norm=10.0)  # rainbow/run_atari.py:229-235
  if uses_iqn_network(kind):
    # munchausen_iqn: iqn's, as the M-IQN paper's Atari values; fqf: the same Adam over every tensor but the fraction
    # layer, which has its own RMSProp (Learner's fraction_* keywords, DESIGN.md §15)
    return OptimizerSpec('adam', 0.00005, 0.01 / 32)
  if kind == 'munchausen':
    return OptimizerSpec('adam', 0.00005, 0.01 / 32)   # the M-DQN paper's Atari values; no run_atari pins them
  raise ValueError(kind)


def uses_iqn_network(kind: str) -> bool:
  """Whether the agent kind applies IQN's network (cosine tau embedding, quantile samples): iqn, munchausen_iqn
  (DESIGN.md §14), which shares its parameters, taus and acting, and fqf (DESIGN.md §15), which adds a fraction layer."""
  return kind in ('iqn', 'munchausen_iqn', 'fqf')


def draws_taus(kind: str) -> bool:
  """Whether the agent kind's steps and acting take taus drawn by the caller: IQN's network except fqf, whose fraction
  layer proposes them from the torso features.  Every place that allocates, draws or passes taus asks this."""
  return uses_iqn_network(kind) and kind != 'fqf'


class NetworkSpec(NamedTuple):
  """Declarative stand-in for `networks.<kind>_atari_network(...)` (networks.py:224-363)."""
  kind: str
  num_actions: int
  num_atoms: int = 51
  vmax: float = 10.0
  num_quantiles: int = 201
  latent_dim: int = 64
  noisy_weight_init: float = 0.1
  tau_samples_s_tm1: int = 64
  tau_samples_policy: int = 64
  tau_samples_s_t: int = 64
  obs_shape: tuple = (84, 84, 4)
  num_fractions: int = 32              # fqf: N, the number of proposed quantile fractions
  dueling: bool = False                # the dueling network (DESIGN.md §16): dqn, double_q, prioritized, munchausen
  noisy: bool = False                  # noisy networks (DESIGN.md §17): the same kinds, plain or dueling


# The kinds that take NetworkSpec(dueling=True) and NetworkSpec(noisy=True); rainbow's network is dueling and noisy already.
DUELING_KINDS = ('dqn', 'double_q', 'prioritized', 'munchausen')
NOISY_KINDS = DUELING_KINDS


def noisy_layers(net: NetworkSpec) -> bool:
  """Whether the network has factorised-noise layers (rainbow, and NetworkSpec(noisy=True)): every place that allocates,
  draws or passes noise asks this."""
  return net.kind == 'rainbow' or bool(net.noisy)

# The dueling network's linear modules.  The reference has no plain dueling network, so these module paths are the
# project's own, kept stable for hk.Params-shaped dicts.
_DUELING_MODULES = {'adv1': 'dueling/advantage/linear', 'adv2': 'dueling/advantage/linear_1',
                    'val1': 'dueling/value/linear', 'val2': 'dueling/value/linear_1'}


# canonical name -> haiku-style module path (the nested "sequential/..." prefixes are
# [UNVERIFIED-3P]; leaf names conv2_d / linear / mu / sigma / w / b are pinned by networks_test.py:41-53,153-163)
def haiku_name(canonical: str, kind: str):
  parts = canonical.split('/')
  leaf = parts[-1]
  conv = {'conv1': 'conv2_d', 'conv2': 'conv2_d_1', 'conv3': 'conv2_d_2'}
  if parts[0] in conv:
    return 'sequential/sequential/' + conv[parts[0]], leaf
  if kind != 'rainbow' and len(parts) == 3:   # noisy networks (DESIGN.md §17): '<layer>/{mu,sigma}/{w,b}'
    module = _DUELING_MODULES.get(parts[0]) or {'fc1': 'sequential/sequential_1/linear',
                                               'head': 'sequential/sequential_1/linear_1'}[parts[0]]
    return module.replace('linear', 'noisy_linear') + '/' + parts[1], leaf
  if kind != 'rainbow' and parts[0] in _DUELING_MODULES:   # the tensor names identify the dueling network
    return _DUELING_MODULES[parts[0]], leaf
  if kind == 'rainbow':
    idx = {'adv1': '', 'adv2': '_1', 'val1': '_2', 'val2': '_3'}[parts[0]]
    return 'noisy_linear%s/%s' % (idx, parts[1]), leaf
  if uses_iqn_network(kind):   # fqf's fraction layer: a linear module of its own beside the quantile network
    return {'embed': 'batch_apply/linear', 'fc1': 'batch_apply_1/sequential/linear',
            'head': 'batch_apply_1/sequential/linear_1', 'fraction': 'fraction_proposal/linear'}[parts[0]], leaf
  return {'fc1': 'sequential/sequential_1/linear', 'head': 'sequential/sequential_1/linear_1'}[parts[0]], leaf


def check_network(net: NetworkSpec) -> None:
  """ValueError for a NetworkSpec no learner can build: dueling=True on a kind outside DUELING_KINDS, noisy=True on a
  kind outside NOISY_KINDS."""
  if net.dueling and net.kind not in DUELING_KINDS:
    raise ValueError('dueling=True needs one of %s, got %r%s' % (', '.join(DUELING_KINDS), net.kind,
                                                                 ' (its network is dueling already)' if net.kind == 'rainbow' else ''))
  if net.noisy and net.kind not in NOISY_KINDS:
    raise ValueError('noisy=True needs one of %s, got %r%s' % (', '.join(NOISY_KINDS), net.kind,
                                                               ' (its network is noisy already)' if net.kind == 'rainbow' else ''))


MAX_RANDOM_SHIFT_PAD = 16


def check_cql_alpha(alpha) -> float:
  """The CQL weight (DESIGN.md §20) as a float; ValueError unless it is a finite real number >= 0."""
  if isinstance(alpha, (bool, np.bool_)) or not isinstance(alpha, (int, float, np.integer, np.floating)):
    raise ValueError('cql_alpha must be a real number, got %r' % (alpha,))
  alpha = float(alpha)
  if not math.isfinite(alpha) or alpha < 0.0:
    raise ValueError('cql_alpha must be finite and >= 0, got %r' % (alpha,))
  return alpha


def check_random_shift_pad(pad, obs_shape) -> int:
  """The random-shift pad (DESIGN.md §18) as an int; ValueError unless it is an integer in [0, 16] and less than
  min(H, W)."""
  if isinstance(pad, (bool, np.bool_)) or not isinstance(pad, (int, np.integer)):
    raise ValueError('random_shift_pad must be an integer, got %r' % (pad,))
  pad = int(pad)
  if not 0 <= pad <= MAX_RANDOM_SHIFT_PAD:
    raise ValueError('random_shift_pad must be in [0, %d], got %d' % (MAX_RANDOM_SHIFT_PAD, pad))
  if pad >= min(obs_shape[0], obs_shape[1]):
    raise ValueError('random_shift_pad must be less than min(H, W) = %d, got %d' % (min(obs_shape[0], obs_shape[1]), pad))
  return pad


def noise_vector_sizes(net: NetworkSpec):
  """(name, length) of the factorised-noise vectors of ONE `network.apply`: rainbow's 8 in `hk.next_rng_key()` order
  (networks.py:169-170, :235-248); a noisy network's (DESIGN.md §17) fc1 in / out and head in / out, or dueling,
  rainbow's 8 with one atom."""
  h = net.obs_shape[0]
  for k, s in ((8, 4), (4, 2), (3, 1)):
    h = (h - k) // s + 1
  w = net.obs_shape[1]
  for k, s in ((8, 4), (4, 2), (3, 1)):
    w = (w - k) // s + 1
  d = h * w * 64
  a, k = net.num_actions, net.num_atoms
  if net.kind != 'rainbow':
    if not net.dueling:
      return [('fc1/in', d), ('fc1/out', 512), ('head/in', 512), ('head/out', a)]
    k = 1
  return [('adv1/in', d), ('adv1/out', 512), ('adv2/in', 512), ('adv2/out', a * k),
          ('val1/in', d), ('val1/out', 512), ('val2/in', 512), ('val2/out', k)]


def pack_noise(net: NetworkSpec, applies) -> np.ndarray:
  """Flattens a list of per-apply {name: vector} dicts into the device layout (each vector padded
  to a multiple of 4 floats so the kernels can use 16-byte loads)."""
  out = []
  for one in applies:
    for name, n in noise_vector_sizes(net):
      v = np.asarray(one[name], dtype=np.float32).reshape(-1)
      assert v.size == n, (name, v.size, n)
      out.append(np.concatenate([v, np.zeros((-n) % 4, dtype=np.float32)]))
  return np.concatenate(out)


def _cstream():
  return torch.cuda.current_stream().cuda_stream


def _f32(x, device):
  """`x` as a contiguous float32 tensor on `device`; None stays None."""
  return None if x is None else torch.as_tensor(x, device=device).to(torch.float32).contiguous()


def _ptr(t):
  return 0 if t is None else t.data_ptr()


def _act_inputs(owner, E, explore, taus, noise, stream_noise):
  """The exploration and randomness inputs of one act of E streams on `owner` (a `Learner` or an `Actor`) as device
  tensors: (explore, taus, noise, noise_ld).  `stream_noise` is a noisy network's [E, noise_stride] block whose row e is stream
  e's own apply; it replaces noise / taus and sets noise_ld to the stride (0: one apply shared by the streams)."""
  x = _f32(explore, owner.device)
  if stream_noise is None:
    return x, _f32(taus, owner.device), _f32(noise, owner.device), 0
  if noise is not None or taus is not None:
    raise ValueError('stream_noise replaces noise / taus')
  if not noisy_layers(owner.net):
    raise ValueError('stream_noise needs a learner with noisy layers')
  n = _f32(stream_noise, owner.device)
  if n.dim() != 2 or n.shape[0] != E or n.shape[1] != owner.noise_stride:
    raise ValueError('stream_noise must be [E, noise_stride] = [%d, %d], got %s' % (E, owner.noise_stride, tuple(n.shape)))
  return x, None, n, owner.noise_stride


class Learner:
  """Device-resident parameters, optimizer state and workspace + the fused update."""

  def __init__(self, net: NetworkSpec, batch_size: int = 32, optimizer: Optional[OptimizerSpec] = None,
               grad_error_bound: float = 1.0 / 32, huber_param: float = 1.0, munchausen_alpha: float = 0.9,
               entropy_temperature: float = 0.03, log_policy_clip: float = -1.0, fraction_learning_rate: float = 2.5e-9,
               fraction_opt_eps: float = 1e-5, fraction_rms_decay: float = 0.95, device=None, random_shift_pad: int = 0,
               prioritized: bool = False, cql_alpha: float = 0.0):
    """`munchausen_alpha`, `entropy_temperature` (tau) and `log_policy_clip` (l0) are Munchausen DQN's and
    Munchausen-IQN's (DESIGN.md §13, §14, defaults the paper's Atari values); the library rejects tau <= 0, alpha < 0,
    l0 > 0 and non-finite values for those kinds, and the other kinds ignore them.  `fraction_learning_rate`,
    `fraction_opt_eps` and `fraction_rms_decay` are fqf's centred RMSProp over its fraction layer (DESIGN.md §15); the
    library rejects a negative or non-finite rate, eps <= 0 and a decay outside [0, 1) for fqf.  `random_shift_pad` p > 0
    turns on random-shift augmentation of the update (DrQ; DESIGN.md §18): every update reads s_tm1 and s_t shifted by
    the [B, 4] int32 `shifts`, which `generate_randomness` draws; acting never sees a shift.  ValueError unless p is an
    integer in [0, 16] and less than min(H, W).  `prioritized=True` makes every update fill `.priorities` by the kind's
    rule and lets `learn` sample by priority and write them back (DESIGN.md §19); prioritized and rainbow do so
    whatever it says.  `cql_alpha` > 0 adds conservative Q-learning's alpha (logsumexp_a Q(s_tm1, a) - Q(s_tm1, a_tm1))
    to each example's loss (CQL(H), DESIGN.md §20) and fills `.regularizer` [B] with that difference; 0 is off.
    ValueError unless it is finite and >= 0."""
    check_network(net)
    random_shift_pad = check_random_shift_pad(random_shift_pad, net.obs_shape)
    cql_alpha = check_cql_alpha(cql_alpha)
    if not torch.cuda.is_available():
      raise RuntimeError('dqn_zoo_b200.learner needs a CUDA device (there is no CPU fallback)')
    self.net = net
    self.kind = net.kind
    self.batch_size = batch_size
    self.opt = optimizer or default_optimizer(net.kind)
    self.device = torch.device(device or ('cuda:%d' % torch.cuda.current_device()))
    cfg = _lib.LearnerConfig()
    cfg.kind = _lib.AGENT_KINDS[net.kind]
    cfg.num_actions, cfg.num_atoms, cfg.num_quantiles, cfg.latent_dim = net.num_actions, net.num_atoms, net.num_quantiles, net.latent_dim
    cfg.tau_samples_s_tm1, cfg.tau_samples_policy, cfg.tau_samples_s_t = net.tau_samples_s_tm1, net.tau_samples_policy, net.tau_samples_s_t
    cfg.batch = batch_size
    cfg.obs_h, cfg.obs_w, cfg.obs_c = net.obs_shape
    cfg.vmax, cfg.grad_error_bound, cfg.huber_param = net.vmax, grad_error_bound, huber_param
    cfg.optimizer = _lib.OPTIMIZERS[self.opt.name]
    cfg.learning_rate, cfg.opt_eps, cfg.rms_decay = self.opt.learning_rate, self.opt.eps, self.opt.decay
    cfg.adam_b1, cfg.adam_b2, cfg.max_global_grad_norm = self.opt.b1, self.opt.b2, self.opt.max_global_grad_norm
    cfg.munchausen_alpha, cfg.entropy_temperature, cfg.log_policy_clip = munchausen_alpha, entropy_temperature, log_policy_clip
    cfg.num_fractions = net.num_fractions
    cfg.fraction_learning_rate, cfg.fraction_opt_eps, cfg.fraction_rms_decay = (fraction_learning_rate, fraction_opt_eps,
                                                                                fraction_rms_decay)
    cfg.dueling = 1 if net.dueling else 0
    cfg.noisy = 1 if net.noisy else 0
    cfg.random_shift_pad = random_shift_pad
    cfg.prioritized = 1 if prioritized else 0
    cfg.cql_alpha = cql_alpha
    self.random_shift_pad = random_shift_pad
    self.cql_alpha = cql_alpha
    self.cfg = cfg
    plan = _lib.LearnerPlan()
    _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(plan))
    self.plan = plan
    self.obs_bytes = int(np.prod(net.obs_shape))
    dev = self.device
    P = plan.param_count
    self.online = torch.zeros(P, dtype=torch.float32, device=dev)
    self.target = torch.zeros(P, dtype=torch.float32, device=dev)
    self.grads = torch.zeros(P, dtype=torch.float32, device=dev)
    self.opt_state = torch.zeros(plan.opt_state_floats, dtype=torch.float32, device=dev)
    self.workspace = torch.zeros(plan.workspace_bytes, dtype=torch.uint8, device=dev)
    self.counters = torch.zeros(4, dtype=torch.int64, device=dev)
    self.taus = torch.zeros(max(plan.tau_floats, 1), dtype=torch.float32, device=dev)
    self.noise = torch.zeros(max(plan.noise_floats, 1), dtype=torch.float32, device=dev)
    self.noise_stride = 0          # floats of one noise apply (noisy layers)
    if noisy_layers(net):
      stride = C.c_int64()
      _lib.call('dz_learner_noise_stride', C.byref(cfg), C.byref(stride))
      self.noise_stride = stride.value
    self._stream_noise = None      # [batch_size, noise_stride], allocated by the first generate_stream_noise
    # random_shift_pad > 0: (dy0, dx0, dy1, dx1) of each example of the next update
    self.shifts = torch.zeros((batch_size, 4), dtype=torch.int32, device=dev)
    self.loss = torch.zeros(1, dtype=torch.float32, device=dev)
    self.per_example = torch.zeros(batch_size, dtype=torch.float32, device=dev)
    self.priorities = torch.zeros(batch_size, dtype=torch.float32, device=dev)
    self.regularizer = torch.zeros(batch_size, dtype=torch.float32, device=dev)   # cql_alpha > 0: R_b of the last update
    self.grad_norm = torch.zeros(1, dtype=torch.float32, device=dev)
    self.max_seen_priority = torch.ones(1, dtype=torch.float32, device=dev)   # rainbow/agent.py:79
    self.q_out = torch.zeros(64, dtype=torch.float32, device=dev)
    # tensor table
    self.tensors = {}
    name = C.create_string_buffer(64)
    shape = (C.c_int64 * 4)()
    ndim, off = C.c_int32(), C.c_int64()
    for i in range(plan.num_tensors):
      _lib.call('dz_learner_tensor_info', C.byref(cfg), i, name, shape, C.byref(ndim), C.byref(off))
      self.tensors[name.value.decode()] = (off.value, tuple(shape[k] for k in range(ndim.value)))
    bufs = _lib.LearnerBuffers(self.online.data_ptr(), self.target.data_ptr(), self.grads.data_ptr(),
                               self.opt_state.data_ptr(), self.workspace.data_ptr(), self.counters.data_ptr())
    handle = C.c_void_p()
    _lib.call('dz_learner_create', C.byref(cfg), C.byref(bufs), C.byref(handle))
    self._h = handle
    self._graph = None
    self._learn_io = None

  def __del__(self):
    h, self._h = getattr(self, '_h', None), None
    if h:
      _lib.lib.dz_learner_destroy(h)

  # -- parameters ----------------------------------------------------------------------------------
  def view(self, blob: torch.Tensor, name: str) -> torch.Tensor:
    off, shape = self.tensors[name]
    return blob[off:off + int(np.prod(shape))].view(shape)

  def init_params(self, seed: int) -> None:
    """Legacy U(+-1/sqrt(fan_in)) init for weights AND biases (networks.py:58-79); noisy sigma =
    sigma0/sqrt(in) (networks.py:156-166); fqf's fraction layer U(+-0.01/sqrt(fan_in)) weights and zero biases, so the
    first fractions are uniform to within about 1e-2.  numpy RandomState stream — not the JAX PRNG."""
    rs = np.random.RandomState(seed)
    params = {}
    for name, (_, shape) in self.tensors.items():
      layer = name.rsplit('/', 1)[0]
      n_in = int(np.prod(self.tensors[layer + '/w'][1][:-1]))
      if name == 'fraction/w':
        params[name] = rs.uniform(-0.01 / math.sqrt(n_in), 0.01 / math.sqrt(n_in), size=shape).astype(np.float32)
      elif name == 'fraction/b':
        params[name] = np.zeros(shape, np.float32)
      elif '/sigma/' in name:
        params[name] = np.full(shape, self.net.noisy_weight_init / math.sqrt(n_in), dtype=np.float32)
      else:
        bound = math.sqrt(1.0 / n_in)
        params[name] = rs.uniform(-bound, bound, size=shape).astype(np.float32)
    self.set_params(params, also_target=True)

  def set_params(self, params: Mapping[str, np.ndarray], also_target: bool = False, blob: str = 'online') -> None:
    dst = getattr(self, blob)
    for name, value in params.items():
      self.view(dst, name).copy_(torch.as_tensor(np.asarray(value, dtype=np.float32)))
    if also_target:
      self.sync_target()

  def get_params(self, blob: str = 'online') -> Dict[str, np.ndarray]:
    src = getattr(self, blob)
    return {name: self.view(src, name).cpu().numpy() for name in self.tensors}

  def haiku_params(self, blob: str = 'online'):
    """Nested {module: {leaf: array}} like `hk.Params` (the reference's `online_params`)."""
    out = {}
    for name, value in self.get_params(blob).items():
      mod, leaf = haiku_name(name, self.kind)
      out.setdefault(mod, {})[leaf] = value
    return out

  def get_opt_state(self):
    """optax-shaped: adam -> {'count','mu','nu'}; rmsprop -> {'mu','nu'} (dicts by canonical name)."""
    P = self.plan.param_count
    mu, nu = self.opt_state[:P], self.opt_state[P:]
    st = {'mu': {n: self.view(mu, n).cpu().numpy() for n in self.tensors},
          'nu': {n: self.view(nu, n).cpu().numpy() for n in self.tensors}}
    st['count'] = int(self.counters[0].item())
    return st

  def set_opt_state(self, st) -> None:
    P = self.plan.param_count
    mu, nu = self.opt_state[:P], self.opt_state[P:]
    for n in self.tensors:
      self.view(mu, n).copy_(torch.as_tensor(np.asarray(st['mu'][n], dtype=np.float32)))
      self.view(nu, n).copy_(torch.as_tensor(np.asarray(st['nu'][n], dtype=np.float32)))
    self.counters[0] = int(st.get('count', 0))

  def sync_target(self) -> None:
    """`self._target_params = self._online_params` (dqn/agent.py:155-156)."""
    _lib.call('dz_learner_sync_target', self._h, _cstream())

  # -- updates -------------------------------------------------------------------------------------
  def _row_table(self, dense: torch.Tensor) -> torch.Tensor:
    n = dense.shape[0]
    stride = dense.stride(0) * dense.element_size()
    return dense.data_ptr() + torch.arange(n, dtype=torch.int64, device=self.device) * stride

  def update(self, s_tm1, a_tm1, r_t, discount_t, s_t, weights=None, taus=None, noise=None, apply_update=True,
             shifts=None):
    """`jit(update)` on an explicit batch of device tensors (uint8 [B,H,W,C], int, float, float,
    uint8).  r/discount/weights are rounded to float32 as at the jit boundary.  `shifts` ([B, 4] int, random_shift_pad
    > 0) replaces `.shifts`, as `taus` / `noise` replace theirs.  Returns nothing; results are in `.loss`,
    `.per_example`, `.priorities`, `.grad_norm`, `.grads`."""
    dev = self.device
    B = self.batch_size
    s_tm1 = torch.as_tensor(s_tm1, device=dev).contiguous().view(B, -1)
    s_t = torch.as_tensor(s_t, device=dev).contiguous().view(B, -1)
    assert s_tm1.dtype == torch.uint8 and s_tm1.shape[1] == self.obs_bytes
    keep = [s_tm1, s_t, self._row_table(s_tm1), self._row_table(s_t),
            torch.as_tensor(a_tm1, device=dev).to(torch.int32).contiguous(),
            torch.as_tensor(r_t, device=dev).to(torch.float32).contiguous(),
            torch.as_tensor(discount_t, device=dev).to(torch.float32).contiguous()]
    w = None if weights is None else torch.as_tensor(weights, device=dev).to(torch.float32).contiguous()
    if taus is not None:
      flat_t = torch.as_tensor(taus, device=dev).to(torch.float32).reshape(-1)
      self.taus[:flat_t.numel()].copy_(flat_t)
    if noise is not None:
      flat = torch.as_tensor(noise, device=dev).to(torch.float32).reshape(-1)
      self.noise[:flat.numel()].copy_(flat)
    if shifts is not None:
      if not self.random_shift_pad:
        raise ValueError('shifts need a learner with random_shift_pad > 0')
      self.shifts.copy_(torch.as_tensor(shifts, device=dev).to(torch.int32).reshape(B, 4))
    batch = _lib.Batch(keep[2].data_ptr(), keep[3].data_ptr(), keep[4].data_ptr(), keep[5].data_ptr(),
                       keep[6].data_ptr(), 0 if w is None else w.data_ptr(),
                       self.taus.data_ptr() if draws_taus(self.kind) else 0,
                       self.noise.data_ptr() if noisy_layers(self.net) else 0, self._shifts_ptr())
    out = _lib.UpdateOutputs(self.loss.data_ptr(), self.per_example.data_ptr(), self.priorities.data_ptr(),
                             self.grad_norm.data_ptr(), self.regularizer.data_ptr())
    _lib.call('dz_learner_update', self._h, C.byref(batch), C.byref(out), 1 if apply_update else 0, _cstream())
    self._keep = (keep, w)

  def _shifts_ptr(self):
    return self.shifts.data_ptr() if self.random_shift_pad else 0

  def generate_randomness(self, seed: int, beside_sampler: bool = False) -> None:
    """Fills `.taus` / `.noise` for the next update from the device generator (Philox).  `beside_sampler`: enqueue on
    the learner's side stream (ordered before the next learn()/update()/q_values() only).  With random_shift_pad > 0 it
    first fills `.shifts` on the current stream, at the same counter; the counter still advances once."""
    if self.random_shift_pad:
      _lib.call('dz_learner_generate_shifts', self._h, seed, self.shifts.data_ptr(), _cstream())
    _lib.call('dz_learner_generate_randomness_async' if beside_sampler else 'dz_learner_generate_randomness', self._h, seed,
              self.taus.data_ptr(), self.noise.data_ptr(), _cstream())

  def generate_stream_noise(self, seed: int, num_streams: int) -> torch.Tensor:
    """Noisy layers: one noise apply per actor stream, `[num_streams, noise_stride]` float32 on the device, for
    `act_batch(..., stream_noise=...)`.  Same generator and counter as `generate_randomness` (which it advances); the
    returned view is overwritten by the next call."""
    if self._stream_noise is None and noisy_layers(self.net):
      self._stream_noise = torch.zeros((self.batch_size, self.noise_stride), dtype=torch.float32, device=self.device)
    buf = self._stream_noise
    _lib.call('dz_learner_generate_stream_noise', self._h, seed, int(num_streams), 0 if buf is None else buf.data_ptr(),
              _cstream())
    return buf[:num_streams]

  def q_values(self, obs_u8: torch.Tensor, taus=None, noise=None) -> torch.Tensor:
    """Online-network Q-values for one observation (the network half of select_action)."""
    obs = torch.as_tensor(obs_u8, device=self.device).contiguous().view(-1)
    t, n = _f32(taus, self.device), _f32(noise, self.device)
    _lib.call('dz_learner_act_batch', self._h, obs.data_ptr(), 1, _ptr(t), _ptr(n), 0, 0, 0.0, self.q_out.data_ptr(), 0,
              _cstream())
    self._keep_q = (obs, t, n)
    return self.q_out[:self.net.num_actions]

  def act_batch(self, obs_u8: torch.Tensor, epsilon: float = 0.0, explore=None, taus=None, noise=None, stream_noise=None):
    """Batched select_action for E <= batch_size environment streams in ONE enqueue: `obs_u8` is [E, H, W, C] uint8 (device
    or host), `explore` a float32 [2, E] tensor of uniforms in [0, 1) (None: greedy).  Rainbow takes either `noise` (one
    apply shared by the E streams) or `stream_noise`, a [E, noise_stride] tensor whose row e is stream e's own apply
    (`generate_stream_noise`).  Returns (actions int32 [E], q_values float32 [E, num_actions]) as device tensors — the
    caller does one D2H of the actions per tick."""
    obs = torch.as_tensor(obs_u8, device=self.device).contiguous()
    E = int(obs.shape[0])
    if not hasattr(self, '_act_q') or self._act_q.shape[0] < E:
      self._act_q = torch.zeros((self.batch_size, self.net.num_actions), dtype=torch.float32, device=self.device)
      self._act_a = torch.zeros(self.batch_size, dtype=torch.int32, device=self.device)
    x, t, n, noise_ld = _act_inputs(self, E, explore, taus, noise, stream_noise)
    _lib.call('dz_learner_act_batch', self._h, obs.data_ptr(), E, _ptr(t), _ptr(n), noise_ld, _ptr(x), float(epsilon),
              self._act_q.data_ptr(), self._act_a.data_ptr(), _cstream())
    self._keep_act = (obs, t, n, x)
    return self._act_a[:E], self._act_q[:E]

  def actor(self, num_streams: int, frozen: bool = False) -> 'Actor':
    """An acting context for `num_streams` streams (not capped by batch_size) over this learner's online parameters.
    `frozen=True`: over a parameter snapshot of its own (`Actor.load_params`) with a generator counter of its own; it
    touches no device state of this learner."""
    return Actor(self, num_streams, frozen=frozen)

  # -- fused sample -> update -> priority write-back -------------------------------------------------
  def make_learn_io(self, stage: torch.Tensor, prioritized: bool, priority_exponent: float):
    """Binds the per-step staging buffer (float64 view: [pos(int64) B | u_tree B | u_mix B | scalars 4])
    and persistent sample outputs into a dz_learn_io."""
    B = self.batch_size
    dev = self.device
    self.s_ids = torch.zeros(3 * B, dtype=torch.int64, device=dev)
    self.s_f64 = torch.zeros(2 * B, dtype=torch.float64, device=dev)
    io = _lib.LearnIO()
    base = stage.data_ptr()
    io.sample_in = _lib.SampleInputs(base, base + 8 * B, base + 16 * B, base + 24 * B)
    sp, fp = self.s_ids.data_ptr(), self.s_f64.data_ptr()
    io.sample_out = _lib.SampleOutputs(sp, sp + 8 * B, sp + 16 * B, fp, fp + 8 * B)
    io.d_taus = self.taus.data_ptr() if draws_taus(self.kind) else 0
    io.d_noise = self.noise.data_ptr() if noisy_layers(self.net) else 0
    io.update_out = _lib.UpdateOutputs(self.loss.data_ptr(), self.per_example.data_ptr(), self.priorities.data_ptr(),
                                       self.grad_norm.data_ptr(), self.regularizer.data_ptr())
    io.d_max_seen_priority = self.max_seen_priority.data_ptr()
    io.priority_exponent = float(priority_exponent)
    io.d_shifts = self._shifts_ptr()
    return io

  def learn(self, replay_view, prioritized: bool, io) -> None:
    """One `_learn()` enqueue (rainbow/agent.py:181-198)."""
    _lib.call('dz_learner_learn', self._h, C.byref(replay_view), 1 if prioritized else 0, C.byref(io), _cstream())

  @property
  def sampled_ids(self):
    return self.s_ids[:self.batch_size]

  @property
  def sampled_indices(self):
    return self.s_ids[self.batch_size:2 * self.batch_size]

  @property
  def sampled_weights(self):
    return self.s_f64[self.batch_size:]


class Actor:
  """Batched acting for a fixed number of streams (1 to 1024; IQN: num_streams * tau_samples_policy <= 16384) in one
  call, over the learner's online parameters read in place: an act enqueued after `learn()` / `update()` on the stream
  sees their parameters, with no copy.  Its buffers are sized for its streams, so one learner of any batch size can act
  for many environments.  On the tensor-core geometries (84x84x4 among them) the torso and the 3136 -> 512 layer run
  on the learner's sm_90a tensor-core kernels.  Row e's result does not depend on num_streams.

  A frozen actor (`Learner.actor(E, frozen=True)`) acts on a snapshot of its own instead, taken by `load_params` (which
  also packs the tensor-core weight images once), and draws its randomness from a counter of its own (`counter`).  It
  keeps no reference to the learner and touches none of its device state, so it can act on another CUDA stream while
  the learner trains, and the learner's next draws do not depend on it.  For the same parameters and randomness inputs
  its outputs equal a live actor's bit for bit."""

  def __init__(self, learner: Learner, num_streams: int, frozen: bool = False):
    E = int(num_streams)
    self.frozen = bool(frozen)
    nbytes = C.c_int64()
    _lib.call('dz_actor_frozen_plan_query' if self.frozen else 'dz_actor_plan_query', C.byref(learner.cfg), E,
              C.byref(nbytes))
    # a live actor reads the learner's parameters: keep it alive for the actor's lifetime
    self.learner = None if self.frozen else learner
    self.num_streams = E
    self.net, self.kind, self.device = learner.net, learner.kind, learner.device
    self.obs_bytes, self.noise_stride = learner.obs_bytes, learner.noise_stride
    self.tensors = dict(learner.tensors)
    self.param_count = int(learner.plan.param_count)
    dev = learner.device
    net = learner.net
    # zero-filled: the tensor-core plan reads padding rows of its operand images that no launch writes
    self.workspace = torch.zeros(nbytes.value, dtype=torch.uint8, device=dev)
    if self.frozen:
      torch.cuda.current_stream().synchronize()   # create zeroes the counter on the legacy stream: after the fill
    self.q = torch.zeros((E, net.num_actions), dtype=torch.float32, device=dev)
    self.actions = torch.zeros(E, dtype=torch.int32, device=dev)
    self.taus = torch.zeros((E, net.tau_samples_policy), dtype=torch.float32, device=dev) if draws_taus(net.kind) else None
    rb = noisy_layers(net)
    self.noise = torch.zeros(learner.noise_stride, dtype=torch.float32, device=dev) if rb else None
    self.stream_noise = torch.zeros((E, learner.noise_stride), dtype=torch.float32, device=dev) if rb else None
    self.loaded = False
    handle = C.c_void_p()
    _lib.call('dz_actor_create_frozen' if self.frozen else 'dz_actor_create', learner._h, E, self.workspace.data_ptr(),
              C.byref(handle))
    self._h = handle

  def __del__(self):
    h, self._h = getattr(self, '_h', None), None
    if h:
      _lib.lib.dz_actor_destroy(h)

  # -- frozen actors: the parameter snapshot and the generator counter ------------------------------------------------
  def _need_frozen(self, what):
    if not self.frozen:
      raise ValueError('%s needs a frozen actor (Learner.actor(E, frozen=True)); a live actor reads the learner in place'
                       % what)

  def flat_params(self, params) -> Dict[str, np.ndarray]:
    """An `hk.Params`-shaped {module: {leaf: array}} or flat {canonical_name: array} dict as a flat dict."""
    flat = {}
    for key, value in params.items():
      if isinstance(value, Mapping):
        for leaf, arr in value.items():
          names = [n for n in self.tensors if haiku_name(n, self.kind) == (key, leaf)]
          if not names:
            raise KeyError('unknown parameter %s/%s' % (key, leaf))
          flat[names[0]] = arr
      else:
        flat[key] = value
    return flat

  def load_params(self, source) -> None:
    """Takes a snapshot: `source` is a `Learner` with this network (one device-to-device copy of its online blob, ordered
    after the work already enqueued on the current stream), an `hk.Params`-shaped dict or a flat {canonical_name: array}
    dict naming every tensor.  Enqueued on the current stream, with the packing of the tensor-core weight images."""
    self._need_frozen('load_params')
    if isinstance(source, Learner):
      if source.kind != self.kind or source.tensors != self.tensors or source.net.obs_shape != self.net.obs_shape:
        raise ValueError('the learner\'s network does not match this actor\'s')
      src = source.online
    else:
      flat = self.flat_params(source)
      missing = sorted(set(self.tensors) - set(flat))
      if missing:
        raise KeyError('parameters missing: %s' % ', '.join(missing))
      blob = np.zeros(self.param_count, np.float32)
      for name, (off, shape) in self.tensors.items():
        value = np.asarray(flat[name], dtype=np.float32)
        if value.shape != tuple(shape):
          raise ValueError('%s has shape %s, expected %s' % (name, value.shape, tuple(shape)))
        blob[off:off + value.size] = value.reshape(-1)
      src = torch.from_numpy(blob).to(self.device)
    _lib.call('dz_actor_load_params', self._h, src.data_ptr(), _cstream())
    self._keep_load = src
    self.loaded = True

  def params(self) -> torch.Tensor:
    """A device copy of the snapshot ([P] float32 in the learner's layout), made on the current stream."""
    self._need_frozen('params')
    out = torch.empty(self.param_count, dtype=torch.float32, device=self.device)
    _lib.call('dz_actor_get_params', self._h, out.data_ptr(), _cstream())
    return out

  def get_params(self) -> Dict[str, np.ndarray]:
    """The snapshot as a flat {canonical_name: array} dict of host arrays."""
    blob = self.params().cpu().numpy()
    return {name: blob[off:off + int(np.prod(shape))].reshape(shape).copy() for name, (off, shape) in self.tensors.items()}

  @property
  def counter(self) -> int:
    """A frozen actor's generator counter (0 at creation; each `generate_randomness` advances it by one), read after
    the work enqueued on the current stream."""
    self._need_frozen('counter')
    v = C.c_int64()
    _lib.call('dz_actor_get_counter', self._h, C.byref(v), _cstream())
    return int(v.value)

  @counter.setter
  def counter(self, value: int) -> None:
    self._need_frozen('counter')
    _lib.call('dz_actor_set_counter', self._h, int(value), _cstream())

  def generate_randomness(self, seed: int, per_stream: bool = False) -> torch.Tensor:
    """Fills and returns `.taus` (IQN, [E, tau_samples_policy]), `.noise` (rainbow, one apply) or, with `per_stream`,
    `.stream_noise` (rainbow, [E, noise_stride]) from the learner's generator, advancing its counter once (a frozen
    actor: its own counter).  For E <= batch_size the draws equal `Learner.generate_randomness` /
    `generate_stream_noise` at the same seed and counter."""
    kind = self.kind
    if per_stream and not noisy_layers(self.net):
      raise ValueError('per_stream randomness needs a learner with noisy layers')
    if not draws_taus(kind) and not noisy_layers(self.net):
      raise ValueError('%s acting draws no randomness' % kind)
    buf = self.taus if draws_taus(kind) else (self.stream_noise if per_stream else self.noise)
    _lib.call('dz_actor_generate_randomness', self._h, seed, 1 if per_stream else 0, buf.data_ptr(), _cstream())
    return buf

  def act(self, obs_u8, epsilon: float = 0.0, explore=None, taus=None, noise=None, stream_noise=None):
    """`Learner.act_batch` for exactly num_streams observations: `obs_u8` [E, H, W, C] uint8, `explore` float32 [2, E]
    uniforms (None: greedy), IQN `taus` [E, tau_samples_policy], rainbow `noise` (one apply shared by the streams) or
    `stream_noise` [E, noise_stride].  Returns (actions int32 [E], q_values float32 [E, num_actions]) device tensors,
    overwritten by the next call."""
    L = self                        # network shape and device, as the learner's
    E = self.num_streams
    obs = torch.as_tensor(obs_u8, device=L.device).contiguous()
    if obs.dtype != torch.uint8 or obs.dim() < 1 or obs.shape[0] != E or obs[0].numel() != L.obs_bytes:
      raise ValueError('obs must be uint8 [%d, %s], got %s %s' % (E, ', '.join(map(str, L.net.obs_shape)), obs.dtype,
                                                                  tuple(obs.shape)))
    if self.frozen and not self.loaded:
      raise RuntimeError('the frozen actor has no parameters: call load_params first')
    x, t, n, noise_ld = _act_inputs(self, E, explore, taus, noise, stream_noise)
    if x is not None and x.numel() != 2 * E:
      raise ValueError('explore must be [2, %d], got %s' % (E, tuple(x.shape)))
    if t is not None and draws_taus(L.kind) and t.numel() != E * L.net.tau_samples_policy:
      raise ValueError('taus must be [%d, %d], got %s' % (E, L.net.tau_samples_policy, tuple(t.shape)))
    if noise_ld == 0 and n is not None and noisy_layers(L.net) and n.numel() < L.noise_stride:
      raise ValueError('noise must hold one apply (%d floats), got %d' % (L.noise_stride, n.numel()))
    _lib.call('dz_actor_act', self._h, obs.data_ptr(), _ptr(t), _ptr(n), noise_ld, _ptr(x), float(epsilon), self.q.data_ptr(),
              self.actions.data_ptr(), _cstream())
    self._keep = (obs, t, n, x)
    return self.actions, self.q
