"""The seven dqn_zoo agents, and Munchausen DQN and Munchausen-IQN beside them, behind the reference's
`parts.Agent` surface, running on the CUDA replay + learner.

Each class keeps the reference constructor's argument names and the `step / reset /
get_state / set_state / statistics` behaviour (dqn/agent.py:133-229, rainbow/agent.py:135-245,
iqn/agent.py:245-340 ...).  Two arguments necessarily change type (SURVEY §8(b)):
  * `network`   is a `learner.NetworkSpec`   instead of an `hk.Transformed`,
  * `optimizer` is a `learner.OptimizerSpec` instead of an `optax.GradientTransformation`,
and `rng_key` seeds a host `np.random.RandomState` (epsilon-greedy) and the device Philox
stream (IQN taus, noisy-net noise) instead of the JAX threefry stream.

`_learn()` is ONE enqueue: host RandomState draws (reference order) -> pinned staging -> H2D ->
[sample -> gather-in-place -> forward x2/3 -> loss -> backward -> optimizer -> priority
write-back], optionally replayed as a CUDA graph.  Nothing is read back per learner step
(the reference's `jax.device_get(priorities)` sync, rainbow/agent.py:195, is gone):
`max_seen_priority` lives on the device and new transitions take their priority from there.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import os
import pickle
from typing import Any, Callable, Mapping, Optional

import numpy as np
import torch

from dqn_zoo_b200 import _lib
from dqn_zoo_b200 import jax_prng
from dqn_zoo_b200 import learner as learner_lib
from dqn_zoo_b200 import parts
from dqn_zoo_b200 import processors
from dqn_zoo_b200 import replay as replay_lib

NetworkSpec = learner_lib.NetworkSpec
OptimizerSpec = learner_lib.OptimizerSpec
_iqn_net = learner_lib.uses_iqn_network
_draws_taus = learner_lib.draws_taus


def _acting_rows_error(net, E):
  """The acting context's row limit of IQN's network (E x its rows per observation <= ACTOR_MAX_IQN_ROWS) as a
  message, or None within it: iqn / munchausen_iqn act on tau_samples_policy rows, fqf on its num_fractions."""
  if not _iqn_net(net.kind):
    return None
  if _draws_taus(net.kind):
    if E * net.tau_samples_policy > ACTOR_MAX_IQN_ROWS:
      return 'iqn acting needs num_streams * tau_samples_policy <= %d, got %d * %d' % (ACTOR_MAX_IQN_ROWS, E,
                                                                                       net.tau_samples_policy)
  elif E * net.num_fractions > ACTOR_MAX_IQN_ROWS:
    return 'fqf acting needs num_streams * num_fractions <= %d, got %d * %d' % (ACTOR_MAX_IQN_ROWS, E, net.num_fractions)
  return None


def _acting_randomness(source, seed, per_stream=False, num_streams=1):
  """The randomness of one act on `source` (a `Learner` or a `learner_lib.Actor`), drawn from its generator with one
  counter step, as the keyword argument of `Learner.q_values` / `Learner.act_batch` / `Actor.act`: a noisy network's
  own apply per stream (`per_stream`, num_streams of them), IQN's taus or a noisy network's one shared apply (rainbow,
  and NetworkSpec(noisy=True)).  The other networks act without randomness (fqf proposes its fractions) and draw
  nothing: {}."""
  if per_stream:
    what = 'stream_noise'
  elif _draws_taus(source.kind):
    what = 'taus'
  elif learner_lib.noisy_layers(source.net):
    what = 'noise'
  else:
    return {}
  if isinstance(source, learner_lib.Actor):
    return {what: source.generate_randomness(seed, per_stream=per_stream)}
  if per_stream:
    return {what: source.generate_stream_noise(seed, num_streams)}
  source.generate_randomness(seed)
  return {what: getattr(source, what)}


def _seed_of(rng_key) -> int:
  arr = np.asarray(rng_key).astype(np.uint64).reshape(-1)
  seed = 0
  for v in arr:
    seed = (seed * 0x9E3779B97F4A7C15 + int(v)) % (1 << 63)
  return seed


class _DeviceAgent(parts.Agent):
  """Shared machinery; subclasses set KIND and mirror the reference constructors.  PRIORITIZED is True for
  PrioritizedDqn and Rainbow; any other agent takes it from its replay's `prioritized` (DESIGN.md §19)."""

  KIND = 'dqn'
  PRIORITIZED = False
  GREEDY = False

  def _setup(self, preprocessor, sample_network_input, network: NetworkSpec, optimizer: Optional[OptimizerSpec],
             transition_accumulator, replay, batch_size, exploration_epsilon, min_replay_capacity_fraction,
             learn_period, target_network_update_period, rng_key, grad_error_bound=1.0 / 32, huber_param=1.0,
             use_cuda_graph=True, random_shift_pad=0, cql_alpha=0.0, **munchausen):
    if network.kind != self.KIND:
      raise ValueError('network spec kind %r does not match agent %r' % (network.kind, self.KIND))
    if sample_network_input is not None and tuple(np.asarray(sample_network_input).shape) != tuple(network.obs_shape):
      raise ValueError('sample_network_input shape %s != network obs_shape %s'
                       % (np.asarray(sample_network_input).shape, network.obs_shape))
    self._preprocessor = preprocessor
    self._replay = replay
    # on a prioritized replay every agent adds at max_seen_priority and learns by priority (DESIGN.md §19)
    self.PRIORITIZED = type(self).PRIORITIZED or bool(replay.prioritized)
    self._transition_accumulator = transition_accumulator
    self._batch_size = batch_size
    self._exploration_epsilon = exploration_epsilon
    self._min_replay_capacity = min_replay_capacity_fraction * replay.capacity
    self._learn_period = learn_period
    self._target_network_update_period = target_network_update_period
    self._seed = _seed_of(rng_key)
    self._host_rng = np.random.RandomState(self._seed % (1 << 32))
    self._learner = learner_lib.Learner(network, batch_size=batch_size, optimizer=optimizer,
                                        grad_error_bound=grad_error_bound, huber_param=huber_param,
                                        random_shift_pad=random_shift_pad, prioritized=self.PRIORITIZED,
                                        cql_alpha=cql_alpha, **munchausen)
    self._learner.init_params(seed=self._seed % (1 << 31))      # network.init + target = online
    self._action = None
    self._frame_t = -1
    self._statistics = {'state_value': np.nan}
    self._use_graph = use_cuda_graph
    self._graph = None
    self._graph_key = None
    self._io = None
    self._obs_dev = torch.zeros(int(np.prod(network.obs_shape)), dtype=torch.uint8, device=self._learner.device)
    B = batch_size
    self._stage_words = 3 * B + 4
    self._stage_dev = torch.zeros(self._stage_words, dtype=torch.float64, device=self._learner.device)
    self._ring = [torch.zeros(self._stage_words, dtype=torch.float64).pin_memory() for _ in range(8)]
    self._ring_events = [None] * len(self._ring)
    self._ring_pos = 0
    self._learn_steps = 0

  # -- parts.Agent -----------------------------------------------------------------------------------
  def step(self, timestep) -> parts.Action:
    """dqn/agent.py:133-158 (identical control flow for every agent)."""
    self._frame_t += 1
    timestep = self._preprocessor(timestep)
    if timestep is None:  # repeat action
      if self._action is None:
        raise RuntimeError('Cannot repeat if action has never been selected.')
      action = self._action
    else:
      action = self._action = self._act(timestep)
      for transition in self._transition_accumulator.step(timestep, action):
        self._add(transition)
    if self._replay.size < self._min_replay_capacity:
      return action
    if self._frame_t % self._learn_period == 0:
      self._learn()
    if self._frame_t % self._target_network_update_period == 0:
      self._learner.sync_target()
      # The fused step only RECORDS bad priorities / non-finite weights as sticky device flags (no per-step D2H sync);
      # read them on the target-update cadence so a diverged run stops with the reference's exceptions
      # (replay.py:281-282 'value must be finite and positive', :240-241 'Weights are not finite') instead of
      # training on with stale priorities.
      self.check_device_flags()
    return action

  def reset(self) -> None:
    """dqn/agent.py:160-167."""
    self._transition_accumulator.reset()
    if hasattr(self._preprocessor, 'reset'):
      self._preprocessor.reset()
    self._action = None

  @property
  def statistics(self) -> Mapping[str, float]:
    return self._statistics

  @property
  def online_params(self):
    """hk.Params-shaped nested dict of host arrays."""
    return self._learner.haiku_params('online')

  @property
  def exploration_epsilon(self) -> float:
    return 0.0 if self._exploration_epsilon is None else self._exploration_epsilon(self._frame_t)

  @property
  def learner(self) -> learner_lib.Learner:
    return self._learner

  @property
  def importance_sampling_exponent(self) -> float:
    """The prioritized replay's importance-sampling exponent at its current step; AttributeError on a uniform one."""
    self._need_prioritized('importance_sampling_exponent')
    return self._replay.importance_sampling_exponent

  @property
  def max_seen_priority(self) -> float:
    """The largest priority the learner has written (new transitions take it; a synchronising read); AttributeError on
    a uniform replay."""
    self._need_prioritized('max_seen_priority')
    return float(self._learner.max_seen_priority.item())

  def _need_prioritized(self, what):
    if not self.PRIORITIZED:
      raise AttributeError('%s needs an agent on a prioritized replay' % what)

  def get_state(self) -> Mapping[str, Any]:
    """dqn/agent.py:210-220 / rainbow/agent.py:224-235: same keys."""
    state = {
        'rng_key': {'host': self._host_rng.get_state(), 'seed': self._seed,
                    'device_counter': int(self._learner.counters[1].item())},
        'frame_t': self._frame_t,
        'opt_state': self._learner.get_opt_state(),
        'online_params': self._learner.get_params('online'),
        'target_params': self._learner.get_params('target'),
        'replay': self._replay.get_state(),
    }
    if self.PRIORITIZED:
      state['max_seen_priority'] = self.max_seen_priority
    if getattr(self, '_jax_key', None) is not None:
      state['rng_key']['jax'] = self._jax_key.copy()
    return state

  def set_state(self, state: Mapping[str, Any]) -> None:
    """dqn/agent.py:222-229 / rainbow/agent.py:237-245."""
    self._host_rng.set_state(state['rng_key']['host'])
    self._seed = state['rng_key']['seed']
    self._learner.counters[1] = int(state['rng_key']['device_counter'])
    if getattr(self, '_jax_key', None) is not None:
      self._jax_key = np.asarray(state['rng_key']['jax'], dtype=np.uint32).copy()
    self._frame_t = state['frame_t']
    self._learner.set_opt_state(state['opt_state'])
    self._learner.set_params(state['online_params'], blob='online')
    self._learner.set_params(state['target_params'], blob='target')
    self._replay.set_state(state['replay'])
    if self.PRIORITIZED:
      self._learner.max_seen_priority.fill_(float(state['max_seen_priority']))
    self._graph = None  # device pointers of the replay may have changed

  _CHECKPOINT_BLOBS = ('online', 'target', 'opt_state', 'counters', 'max_seen_priority')

  def save_checkpoint(self, directory: str) -> None:
    """Writes the agent into `directory` (DESIGN.md §9): the raw online, target and optimizer-state blobs, the learner
    counters and max_seen_priority as .npy files, the host RandomState, seed, IQN jax key and frame_t in a small
    pickle, and the replay (`save_checkpoint`) in `replay/`.  The replay's RandomState belongs to the run, as for
    `get_state`."""
    from dqn_zoo_b200 import checkpoint as ck
    write = self._checkpoint_writer(snapshot=False)
    write(directory, ck.Transfer(self._learner.device))

  def snapshot_checkpoint(self):
    """A `checkpoint.Snapshot` of the agent at the current point of the CUDA stream, after the learn steps already
    enqueued: device copies of the blobs `save_checkpoint` writes, copies of the host RandomState, seed, IQN jax key
    and frame_t, and the replay's `snapshot_checkpoint`.  Its `write(directory)` gives the files `save_checkpoint`
    would give now, byte for byte, while training goes on."""
    from dqn_zoo_b200 import checkpoint as ck
    held = []
    return ck.Snapshot(self._checkpoint_writer(snapshot=True, held=held), held, self._learner.device)

  def snapshot_checkpoint_bytes(self) -> int:
    """An upper bound of the device memory `snapshot_checkpoint()` takes now."""
    L = self._learner
    return (sum(getattr(L, name).numel() * getattr(L, name).element_size() for name in self._CHECKPOINT_BLOBS) +
            self._replay.snapshot_checkpoint_bytes())

  def _checkpoint_writer(self, snapshot, held=None):
    """(directory, xfer) -> None writing the agent's checkpoint directory: the one definition of its files, fed by
    the live blobs (snapshot=False) or by copies taken now on the current stream (appended to `held`)."""
    from dqn_zoo_b200 import checkpoint as ck
    from dqn_zoo_b200 import replay as replay_lib
    L = self._learner
    blobs = {}
    for name in self._CHECKPOINT_BLOBS:
      t = getattr(L, name)
      if snapshot:
        t = t.clone()
        held.append(t)
      blobs[name] = t
    state = {'format': 'dqn_zoo_b200.agent', 'version': 1, 'kind': self.KIND, 'dueling': bool(L.net.dueling),
             'noisy': bool(L.net.noisy), 'random_shift_pad': L.random_shift_pad, 'prioritized': self.PRIORITIZED,
             'cql_alpha': L.cql_alpha, 'param_count': L.plan.param_count, 'opt_state_floats': L.plan.opt_state_floats,
             'host_rng': self._host_rng.get_state(), 'seed': self._seed,
             'jax_key': None if getattr(self, '_jax_key', None) is None else self._jax_key.copy(),
             'frame_t': self._frame_t}
    replay_files = replay_lib._replay_files(self._replay, snapshot, held)

    def write(directory, xfer):
      os.makedirs(directory, exist_ok=True)
      digests = {}
      for name, t in blobs.items():
        a = t.cpu().numpy()
        np.save(os.path.join(directory, name + '.npy'), a)
        digests[name] = ck.digest_host(a)
      ck.write_bytes(os.path.join(directory, 'agent.pkl'),
                     pickle.dumps(dict(state, digests=digests), protocol=pickle.HIGHEST_PROTOCOL))
      replay_files.write(os.path.join(directory, 'replay'), xfer)
    return write

  def load_checkpoint(self, directory: str) -> None:
    """Restores `save_checkpoint` of an agent of the same kind and network.  ValueError (agent and replay untouched)
    for a checkpoint of another kind, network size or replay geometry; RuntimeError for a file that fails its
    digest.  Drops the CUDA graph, as `set_state` does."""
    from dqn_zoo_b200 import checkpoint as ck
    try:
      with open(os.path.join(directory, 'agent.pkl'), 'rb') as f:
        state = pickle.load(f)
    except (OSError, pickle.UnpicklingError, EOFError) as e:
      raise ValueError('%s is not a readable agent checkpoint: %s' % (directory, e)) from e
    L = self._learner
    # checkpoints written before the dueling network, noisy networks, random-shift augmentation or prioritized replay
    # for every kind existed have no 'dueling' / 'noisy' / 'random_shift_pad' / 'prioritized' key: they hold the plain
    # network, trained without augmentation, on the replay of the kind (prioritized for prioritized and rainbow only);
    # those written before the CQL term (DESIGN.md §20) have no 'cql_alpha' key: they were trained without it
    ck.validate(dict({'dueling': False, 'noisy': False, 'random_shift_pad': 0,
                      'prioritized': type(self).PRIORITIZED, 'cql_alpha': 0.0}, **state),
                {'format': 'dqn_zoo_b200.agent', 'version': 1, 'kind': self.KIND, 'dueling': bool(L.net.dueling),
                 'noisy': bool(L.net.noisy), 'random_shift_pad': L.random_shift_pad, 'prioritized': self.PRIORITIZED,
                 'cql_alpha': L.cql_alpha, 'param_count': L.plan.param_count, 'opt_state_floats': L.plan.opt_state_floats}, directory)
    blobs = {}
    for name in self._CHECKPOINT_BLOBS:
      path = os.path.join(directory, name + '.npy')
      try:
        a = np.load(path)
      except (OSError, ValueError) as e:
        raise RuntimeError('%s: %s' % (path, e)) from e
      if a.shape != tuple(getattr(L, name).shape) or ck.digest_host(a) != state['digests'][name]:
        raise RuntimeError('%s: shape or digest differs from the checkpoint\'s record' % path)
      blobs[name] = a
    self._replay.load_checkpoint(os.path.join(directory, 'replay'))
    for name, a in blobs.items():
      getattr(L, name).copy_(torch.from_numpy(a))
    self._host_rng.set_state(state['host_rng'])
    self._seed = state['seed']
    if state['jax_key'] is not None:
      self._jax_key = np.asarray(state['jax_key'], dtype=np.uint32).copy()
    self._frame_t = state['frame_t']
    self._graph = None

  # -- acting (dqn/agent.py:121-131,169-177) --------------------------------------------------------------
  def _act(self, timestep) -> parts.Action:
    obs = timestep.observation
    if isinstance(obs, torch.Tensor):        # device-resident frame stack (processors.atari(device_observations=True))
      self._obs_dev.copy_(obs.reshape(-1))
    else:
      self._obs_dev.copy_(torch.from_numpy(np.ascontiguousarray(obs).reshape(-1)))
    L = self._learner
    if getattr(self, '_jax_key', None) is not None:
      # iqn/agent.py:220-222: rng_key, sample_key, apply_key, policy_key = split(rng_key, 4); tau_t = uniform(sample_key)
      self._jax_key, sample = jax_prng.iqn_act_keys(self._jax_key)
      self._jax_act.set_keys(sample)
      self._jax_act.launch(L.taus)
      randomness = {'taus': L.taus}
    else:
      randomness = _acting_randomness(L, self._seed)
    q = L.q_values(self._obs_dev, **randomness).cpu().numpy()   # D2H sync, as jax.device_get
    eps = 0.0 if self.GREEDY else self.exploration_epsilon
    if eps > 0.0 and self._host_rng.uniform() < eps:
      a_t = int(self._host_rng.randint(len(q)))
    else:
      a_t = int(np.argmax(q))
    self._statistics['state_value'] = float(q.max())
    return parts.Action(a_t)

  # -- insert --------------------------------------------------------------------------------------
  def _add(self, transition) -> None:
    if self.PRIORITIZED:
      # rainbow/agent.py:148-149: priority = max_seen_priority (kept on the device)
      self._replay.add(transition, priority=self._learner.max_seen_priority)
    else:
      self._replay.add(transition)

  # -- learn -----------------------------------------------------------------------------------------
  def _draws(self):
    """Host RandomState draws in the reference's order (replay.py:551-567 / :78)."""
    rs = self._replay._random_state
    B = self._batch_size
    slot = self._ring[self._ring_pos]
    ev = self._ring_events[self._ring_pos]
    if ev is not None:
      ev.synchronize()
    host = slot.numpy()
    host[:B].view(np.int64)[:] = rs.randint(self._replay.size, size=B)
    if self.PRIORITIZED:
      # Scaled by the root on the device.  KNOWN DIVERGENCE: the reference skips this draw when the root is 0
      # (replay.py:556-560); the root lives on the device here and is not read back per step, so the draw is always
      # consumed and the kernel raises DZ_FLAG_ROOT_ZERO instead (surfaced by check_device_flags on the target-update
      # cadence).  A zero root needs every stored priority to be 0, which the agents' priority rule never produces.
      host[B:2 * B] = rs.uniform(size=B)
      host[2 * B:3 * B] = rs.uniform(size=B)
    host[3 * B:] = self._replay._sample_constants()
    return slot

  def _learn(self) -> None:
    """rainbow/agent.py:181-198 as one enqueue."""
    slot = self._draws()
    if getattr(self, '_jax_key', None) is not None:
      # iqn/agent.py:207 + 182: the agent key advances once per update; three sample keys feed the tau draws
      self._jax_key, sample = jax_prng.iqn_update_keys(self._jax_key)
      self._jax_learn.set_keys(sample)
    self._stage_dev.copy_(slot, non_blocking=True)
    ev = torch.cuda.Event()
    ev.record()
    self._ring_events[self._ring_pos] = ev
    self._ring_pos = (self._ring_pos + 1) % len(self._ring)
    self._launch()

  def learn(self) -> None:
    """Public alias of one learner step (`_learn`): host RNG draws -> H2D -> fused device step."""
    self._learn()

  def learn_from_device_draws(self, draws: torch.Tensor) -> None:
    """One learner step whose sampling draws are already in device memory (`draws` = float64
    [3B+4] in the staging layout).  Used by bench.py for the inputs-resident-in-HBM number."""
    self._stage_dev.copy_(draws, non_blocking=True)
    self._launch()

  def host_draws(self) -> np.ndarray:
    """The staging record for the next learner step (consumes the replay's RandomState)."""
    return self._draws().numpy().copy()

  def _launch(self) -> None:
    L = self._learner
    self._replay._flush()
    self._view = self._replay.device_view()
    key = bytes(self._view)
    if self._graph is not None and key != self._graph_key:
      self._graph = None                     # a device array moved (growth / set_state): recapture
    self._graph_key = key
    if self._io is None:
      self._io = L.make_learn_io(self._stage_dev, self.PRIORITIZED, self._replay._alpha())
    if self._use_graph:
      if self._graph is None:
        self._enqueue()                      # first step runs eagerly (also the warm-up for capture)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
          self._enqueue()
        self._graph = g                      # capture does not execute: nothing was applied twice
      else:
        self._graph.replay()
    else:
      self._enqueue()
    self._learn_steps += 1

  def _enqueue(self):
    L = self._learner
    if getattr(self, '_jax_key', None) is not None:
      if L.random_shift_pad:
        L.generate_randomness(self._seed)       # the shifts and one counter step; the jax taus below replace its taus
      self._jax_learn.launch(L.taus)            # jax.random.uniform draws from the keys staged by _learn()
    elif _draws_taus(self.KIND) or learner_lib.noisy_layers(L.net) or L.random_shift_pad:
      L.generate_randomness(self._seed, beside_sampler=True)
    L.learn(self._view, self.PRIORITIZED, self._io)

  def check_device_flags(self):
    """Raises if a kernel set a sticky error flag (bad priority, root == 0 in the fused path...)."""
    flags = self._replay._flags()
    f = int(flags.item())
    if f & _lib.DZ_FLAG_FRAME_POOL_FULL:       # sticky: the frame pool stored zeros for planes it had no room for
      self._replay._raise_if_pool_full()
    if f:
      flags.zero_()
      if f & (_lib.DZ_FLAG_BAD_VALUE | _lib.DZ_FLAG_BAD_INDEX):
        raise ValueError('value must be finite and positive, index in range (device flags %d).' % f)
      if f & _lib.DZ_FLAG_NONFINITE_WEIGHT:
        raise ValueError('Weights are not finite (device flags %d).' % f)
      raise RuntimeError('device error flags: %d (bad sum-tree target / empty tree in the fused sampler)' % f)


class Dqn(_DeviceAgent):
  """dqn/agent.py:40-229.  It takes the network it is given: with NetworkSpec(noisy=True) (DESIGN.md §17) it draws
  the noise of its noisy layers every step and every act, and still acts epsilon-greedily on the
  `exploration_epsilon` schedule, so NoisyNet-DQN (Fortunato et al., ICLR 2018) is this agent on the noisy network
  with a schedule that is zero throughout.  DoubleQ, PrioritizedDqn and Munchausen take noisy networks the same way."""
  KIND = 'dqn'

  def __init__(self, preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay,
               batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, grad_error_bound, rng_key, use_cuda_graph=True, random_shift_pad=0,
               cql_alpha=0.0):
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                grad_error_bound=grad_error_bound, use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad,
                cql_alpha=cql_alpha)


class DoubleQ(Dqn):
  """double_q/agent.py:40-233."""
  KIND = 'double_q'


class Munchausen(_DeviceAgent):
  """Munchausen DQN (Vieillard, Pietquin & Geist, NeurIPS 2020; DESIGN.md §13): dqn's constructor, network, replay
  and epsilon-greedy acting, with the soft target r + alpha clip(tau log pi(a_tm1|s_tm1), l0, 0) +
  discount sum_a pi(a|s_t) (q(s_t, a) - tau log pi(a|s_t)) of the target network's softmax policy pi.  The defaults
  of `munchausen_alpha`, `entropy_temperature` (tau) and `log_policy_clip` (l0) are the paper's Atari values."""
  KIND = 'munchausen'

  def __init__(self, preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay,
               batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, grad_error_bound, rng_key, use_cuda_graph=True, munchausen_alpha=0.9,
               entropy_temperature=0.03, log_policy_clip=-1.0, random_shift_pad=0, cql_alpha=0.0):
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                grad_error_bound=grad_error_bound, use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad,
                cql_alpha=cql_alpha,
                munchausen_alpha=munchausen_alpha, entropy_temperature=entropy_temperature, log_policy_clip=log_policy_clip)


class PrioritizedDqn(_DeviceAgent):
  """prioritized/agent.py:40-258."""
  KIND = 'prioritized'
  PRIORITIZED = True

  def __init__(self, preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay,
               batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, grad_error_bound, rng_key, use_cuda_graph=True, random_shift_pad=0,
               cql_alpha=0.0):
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                grad_error_bound=grad_error_bound, use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad,
                cql_alpha=cql_alpha)


class C51(_DeviceAgent):
  """c51/agent.py:42-229.  `support` must be linspace(-vmax, vmax, atoms) (c51/run_atari.py:135)."""
  KIND = 'c51'

  def __init__(self, preprocessor, sample_network_input, network, support, optimizer, transition_accumulator,
               replay, batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, rng_key, use_cuda_graph=True, random_shift_pad=0, cql_alpha=0.0):
    _check_support(support, network)
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad, cql_alpha=cql_alpha)


class QrDqn(_DeviceAgent):
  """qrdqn/agent.py:42-232.  `quantiles` must be (arange(n)+0.5)/n (qrdqn/run_atari.py:137)."""
  KIND = 'qrdqn'

  def __init__(self, preprocessor, sample_network_input, network, quantiles, optimizer, transition_accumulator,
               replay, batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, huber_param, rng_key, use_cuda_graph=True, random_shift_pad=0,
               cql_alpha=0.0):
    q = np.asarray(quantiles, dtype=np.float64)
    n = network.num_quantiles
    if len(q) != n or not np.allclose(q, (np.arange(n) + 0.5) / n, rtol=0, atol=1e-6):
      raise ValueError('quantiles must be the %d midpoints (i + 0.5) / n' % n)
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                huber_param=huber_param, use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad,
                cql_alpha=cql_alpha)


class Rainbow(_DeviceAgent):
  """rainbow/agent.py:41-245: greedy acting on the noisy network, PER, n-step, C51 double-Q."""
  KIND = 'rainbow'
  PRIORITIZED = True
  GREEDY = True

  def __init__(self, preprocessor, sample_network_input, network, support, optimizer, transition_accumulator,
               replay, batch_size, min_replay_capacity_fraction, learn_period, target_network_update_period,
               rng_key, use_cuda_graph=True, random_shift_pad=0, cql_alpha=0.0):
    _check_support(support, network)
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                None, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad, cql_alpha=cql_alpha)


class Iqn(_DeviceAgent):
  """iqn/agent.py:133-340."""
  KIND = 'iqn'

  def __init__(self, preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay,
               batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, huber_param, tau_samples_policy, tau_samples_s_tm1, tau_samples_s_t,
               rng_key, use_cuda_graph=True, jax_prng_taus=False, random_shift_pad=0, cql_alpha=0.0):
    """`jax_prng_taus=True`: `rng_key` is treated as a jax PRNG key (`jax.random.PRNGKey(seed)` = [0, seed]) and the tau
    samples of every update and every action selection follow the reference's key chain bit for bit
    (iqn/agent.py:182-190, 207, 220-222; threefry2x32 + jax.random.split/uniform, csrc/dz_jaxprng.cu).  The default keeps
    the device Philox stream.  Epsilon-greedy exploration uses a host RandomState either way."""
    if (network.tau_samples_policy, network.tau_samples_s_tm1, network.tau_samples_s_t) != (
        tau_samples_policy, tau_samples_s_tm1, tau_samples_s_t):
      raise ValueError('tau sample counts must match the NetworkSpec')
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                huber_param=huber_param, use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad,
                cql_alpha=cql_alpha)
    if jax_prng_taus:
      key = np.asarray(rng_key, dtype=np.uint32).reshape(-1)
      if key.size != 2:
        raise ValueError('jax_prng_taus needs a jax-style rng_key of two uint32 words')
      self._jax_key = key.copy()
      dev = self._learner.device
      self._jax_learn = jax_prng.DeviceUniform([batch_size * tau_samples_s_tm1, batch_size * tau_samples_policy,
                                                batch_size * tau_samples_s_t], dev)
      self._jax_act = jax_prng.DeviceUniform([tau_samples_policy], dev)


class MunchausenIqn(_DeviceAgent):
  """Munchausen-IQN (Vieillard, Pietquin & Geist, NeurIPS 2020; DESIGN.md §14): Iqn's constructor (without
  `jax_prng_taus`: no reference key chain pins this agent's taus), network, taus, replay and epsilon-greedy
  acting, with the soft quantile targets y_j = r + alpha clip(tau log pi(a_tm1|s_tm1), l0, 0) +
  discount sum_a pi(a|s_t) (zbar_j(s_t, a) - tau log pi(a|s_t)) of the target network's softmax policy pi over its
  mean quantiles.  The defaults of `munchausen_alpha`, `entropy_temperature` (tau) and `log_policy_clip` (l0) are the
  paper's Atari values."""
  KIND = 'munchausen_iqn'

  def __init__(self, preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay,
               batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, huber_param, tau_samples_policy, tau_samples_s_tm1, tau_samples_s_t,
               rng_key, use_cuda_graph=True, munchausen_alpha=0.9, entropy_temperature=0.03, log_policy_clip=-1.0,
               random_shift_pad=0, cql_alpha=0.0):
    if (network.tau_samples_policy, network.tau_samples_s_tm1, network.tau_samples_s_t) != (
        tau_samples_policy, tau_samples_s_tm1, tau_samples_s_t):
      raise ValueError('tau sample counts must match the NetworkSpec')
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                huber_param=huber_param, use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad,
                cql_alpha=cql_alpha,
                munchausen_alpha=munchausen_alpha, entropy_temperature=entropy_temperature, log_policy_clip=log_policy_clip)


class Fqf(_DeviceAgent):
  """FQF, the Fully parameterized Quantile Function (Yang et al., NeurIPS 2019; DESIGN.md §15): Iqn's constructor without
  the tau sample counts and `jax_prng_taus` (its taus are not drawn: a fraction proposal layer computes N fractions from
  the torso features inside every step and every action selection), plus `num_fractions` (which must match the
  NetworkSpec's) and the fraction layer's centred RMSProp (`fraction_learning_rate`, `fraction_opt_eps`,
  `fraction_rms_decay`).  `optimizer` covers every other tensor (default: Adam at lr 5e-5, eps 0.01 / 32).
  Epsilon-greedy acting on Q(s, a) = sum_i w_i Z(s, a, tau_hat_i)."""
  KIND = 'fqf'

  def __init__(self, preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay,
               batch_size, exploration_epsilon, min_replay_capacity_fraction, learn_period,
               target_network_update_period, huber_param, rng_key, use_cuda_graph=True, num_fractions=32,
               fraction_learning_rate=2.5e-9, fraction_opt_eps=1e-5, fraction_rms_decay=0.95, random_shift_pad=0,
               cql_alpha=0.0):
    if network.num_fractions != num_fractions:
      raise ValueError('num_fractions must match the NetworkSpec')
    self._setup(preprocessor, sample_network_input, network, optimizer, transition_accumulator, replay, batch_size,
                exploration_epsilon, min_replay_capacity_fraction, learn_period, target_network_update_period, rng_key,
                huber_param=huber_param, use_cuda_graph=use_cuda_graph, random_shift_pad=random_shift_pad,
                cql_alpha=cql_alpha,
                fraction_learning_rate=fraction_learning_rate, fraction_opt_eps=fraction_opt_eps,
                fraction_rms_decay=fraction_rms_decay)


def _check_support(support, network):
  s = np.asarray(support, dtype=np.float64)
  want = np.linspace(-network.vmax, network.vmax, network.num_atoms)
  if s.shape != want.shape or not np.allclose(s, want, rtol=0, atol=1e-5):
    raise ValueError('support must be linspace(-vmax, vmax, num_atoms) of the NetworkSpec')


class EpsilonGreedyActor(parts.Agent):
  """Acts epsilon-greedily with externally supplied network parameters (parts.py:336-411): the evaluation agent of
  the run drivers (`eval_agent.network_params = train_agent.online_params`, dqn/run_atari.py:260).

  `network_params` accepts what `agent.online_params` returns (haiku-shaped nested dict of host arrays), a flat
  `{canonical_name: array}` dict, or — the device-resident shortcut — the training learner itself
  (`eval_agent.network_params = train_agent.learner`: one D2D copy of the parameter blob).  The epsilon draw uses a
  host RandomState seeded from `rng_key` (the reference uses the JAX PRNG; action-sequence parity with it is SURVEY
  §8(f) #2)."""

  def __init__(self, preprocessor, network: NetworkSpec, exploration_epsilon: float, rng_key, device=None):
    self._preprocessor = preprocessor
    self._net = network
    self._epsilon = float(exploration_epsilon)
    self._learner = learner_lib.Learner(network, batch_size=1, device=device)
    self._rng = np.random.RandomState(int(np.asarray(rng_key).reshape(-1)[-1]) & 0x7FFFFFFF)
    self._seed = int(np.asarray(rng_key).reshape(-1)[-1]) & 0x7FFFFFFF
    self._obs_dev = torch.zeros(int(np.prod(network.obs_shape)), dtype=torch.uint8, device=self._learner.device)
    self._action = None
    self._has_params = False

  @property
  def network_params(self):
    return self._learner.haiku_params('online') if self._has_params else None

  @network_params.setter
  def network_params(self, params) -> None:
    if params is None:
      self._has_params = False
      return
    if isinstance(params, learner_lib.Learner):
      self._learner.online.copy_(params.online)
    else:
      flat = {}
      for key, value in params.items():
        if isinstance(value, Mapping):            # haiku-shaped {module: {leaf: array}}
          for leaf, arr in value.items():
            flat[self._canonical(key, leaf)] = arr
        else:
          flat[key] = value
      self._learner.set_params(flat)
    self._has_params = True

  def _canonical(self, module, leaf):
    for name in self._learner.tensors:
      if learner_lib.haiku_name(name, self._learner.kind) == (module, leaf):
        return name
    raise KeyError('unknown parameter %s/%s' % (module, leaf))

  def step(self, timestep) -> parts.Action:
    timestep = self._preprocessor(timestep)
    if timestep is None:
      if self._action is None:
        raise RuntimeError('Cannot repeat if action has never been selected.')
      return self._action
    if not self._has_params:
      raise RuntimeError('network_params have not been set.')
    obs = timestep.observation
    if isinstance(obs, torch.Tensor):
      self._obs_dev.copy_(obs.reshape(-1))
    else:
      self._obs_dev.copy_(torch.from_numpy(np.ascontiguousarray(obs).reshape(-1)))
    L = self._learner
    randomness = _acting_randomness(L, self._seed + 1)
    if randomness:
      self._seed += 1                       # a new seed for every act that draws
    q = L.q_values(self._obs_dev, **randomness).cpu().numpy()
    if self._epsilon > 0.0 and self._rng.uniform() < self._epsilon:
      self._action = parts.Action(int(self._rng.randint(len(q))))
    else:
      self._action = parts.Action(int(np.argmax(q)))
    return self._action

  def reset(self) -> None:
    if hasattr(self._preprocessor, 'reset'):
      self._preprocessor.reset()
    self._action = None

  def get_state(self) -> Mapping[str, Any]:
    return {'rng_key': (self._rng.get_state(), self._seed),
            'network_params': self._learner.get_params('online') if self._has_params else None}

  def set_state(self, state: Mapping[str, Any]) -> None:
    rng_state, self._seed = state['rng_key']
    self._rng.set_state(rng_state)
    self.network_params = state['network_params']

  @property
  def statistics(self) -> Mapping[str, float]:
    return {}


AGENTS = {'dqn': Dqn, 'double_q': DoubleQ, 'prioritized': PrioritizedDqn, 'c51': C51, 'qrdqn': QrDqn,
          'rainbow': Rainbow, 'iqn': Iqn, 'munchausen': Munchausen, 'munchausen_iqn': MunchausenIqn, 'fqf': Fqf}


class BatchedEpsilonGreedyActor:
  """E independent actor streams served by ONE network evaluation per tick (the many-actors shape of
  parts.py:342-411 with dqn/agent.py:121-131 acting): observations of all streams -> `Learner.act_batch` (online forward,
  q-values and the epsilon-greedy choice on the device) -> one device-to-host copy of E actions.

  `learner` is the training agent's `Learner` (shared parameters, as the reference's actors read the learner's online
  params).  Up to its batch size the tick runs on `Learner.act_batch`; beyond it, on a `learner_lib.Actor` sized for the
  E streams (up to 1024), over the same live parameters.  Exploration uniforms come from a host RandomState seeded from
  `rng_key` (2E floats per tick; the reference draws with the JAX PRNG per actor).  IQN: every stream gets its own tau
  samples.  Rainbow explores only through its noisy layers: by default one noise sample per tick is shared by the E
  streams, so they explore in lockstep; `per_stream_noise=True` draws E samples per tick and gives stream e its own, as
  the reference's actors each draw theirs (rainbow/agent.py:125-133)."""

  def __init__(self, learner: learner_lib.Learner, num_streams: int, exploration_epsilon, rng_key,
               per_stream_noise: bool = False):
    if num_streams < 1:
      raise ValueError('num_streams must be >= 1')
    if per_stream_noise and not learner_lib.noisy_layers(learner.net):
      raise ValueError('per_stream_noise needs a learner with noisy layers')
    # beyond the learner's batch the tick needs buffers of its own size
    self._actor = learner.actor(num_streams) if num_streams > learner.batch_size else None
    self._learner = learner
    self._per_stream_noise = bool(per_stream_noise)
    self._E = int(num_streams)
    self._epsilon = exploration_epsilon
    seed = int(np.asarray(rng_key).reshape(-1)[-1]) & 0x7FFFFFFF
    self._rng = np.random.RandomState(seed)
    self._seed = seed
    self._t = 0
    self._explore_host = torch.zeros((2, self._E), dtype=torch.float32).pin_memory()
    self._explore_dev = torch.zeros((2, self._E), dtype=torch.float32, device=learner.device)
    self._actions_host = torch.zeros(self._E, dtype=torch.int32).pin_memory()
    self.q_values = None

  def step(self, observations, epsilon: Optional[float] = None) -> np.ndarray:
    """observations: [E, H, W, C] uint8 (device tensor, e.g. the stacks of processors.BatchedAtariPreprocessor, or host
    array).  `epsilon` overrides the actor's own schedule for this tick (`VectorTrainer` evaluates the training agent's
    schedule at its frame count).  Returns the E actions as a host int32 array."""
    L = self._learner
    if epsilon is not None:
      eps = float(epsilon)
    else:
      eps = self._epsilon(self._t) if callable(self._epsilon) else float(self._epsilon)
    actions, self.q_values = self._tick(L if self._actor is None else self._actor, observations, eps)
    self._t += 1
    return actions

  def _tick(self, source, observations, eps):
    """One acting tick of the E streams on `source` (a `Learner`, or a `learner_lib.Actor` for E streams): 2E host
    uniforms when eps > 0, the kind's acting randomness, the act, one pinned device-to-host copy of the actions and a
    synchronise.  Returns (host actions, device q-values)."""
    explore = None
    if eps > 0.0:
      self._explore_host.copy_(torch.from_numpy(self._rng.uniform(size=(2, self._E)).astype(np.float32)))
      self._explore_dev.copy_(self._explore_host, non_blocking=True)
      explore = self._explore_dev
    randomness = _acting_randomness(source, self._seed, self._per_stream_noise, self._E)
    act = source.act if isinstance(source, learner_lib.Actor) else source.act_batch
    actions, q = act(observations, epsilon=eps, explore=explore, **randomness)
    self._actions_host.copy_(actions, non_blocking=True)
    torch.cuda.current_stream().synchronize()   # also frees the pinned uniforms for the next tick
    return self._actions_host.numpy().copy(), q



# The acting context's limits (`learner_lib.Actor`), checked when a trainer acts beyond its learner's batch.
ACTOR_MAX_STREAMS = 1024
ACTOR_MAX_IQN_ROWS = 16384


def _due(lo: int, hi: int, period: int) -> range:
  """The frames f in [lo, hi] with f % period == 0."""
  return range(lo + (-lo) % period, hi + 1, period)


class VectorTrainer:
  """Trains one agent from E environment streams: dqn/agent.py:133-158 generalised to a tick of E timesteps, over the
  batched device paths (`VectorizedAtariPreprocessor.step_arrays`, `BatchedEpsilonGreedyActor`,
  `replay.VectorNStepAccumulator` + `add_batch`, the agent's CUDA-graph learner step).

  The trainer wraps a training agent (any of `AGENTS`) and uses its state in place: learner and replay, the host
  RandomState draws of `_learn`, the CUDA graph, `min_replay_capacity`, `learn_period`, `target_network_update_period`
  and the exploration schedule.  It owns a `VectorizedAtariPreprocessor(E, device_observations=True)`, a
  `VectorNStepAccumulator(E, n)` (n read from the agent's transition accumulator) and a `BatchedEpsilonGreedyActor` over
  the agent's learner, whose exploration uniforms (and acting randomness seed) come from `rng_key`.

  Tick contract.  `frame_t` is the agent's frame counter (-1 before the first step, as for `step`).  With t0 = frame_t
  before the tick, stream e's timestep is frame f = t0 + 1 + e, and the tick leaves frame_t = t0 + E.  In order:
    1. preprocess: `step_arrays` on the E raw timesteps;
    2. act: if any stream emits a timestep, ONE act call for all E streams at epsilon = schedule(t0 + 1); emitting
       streams take the new action, the others repeat their last one (RuntimeError if a stream has none yet); the
       actions reach the host in one copy;
    3. insert: `acc.step`, then `replay.add_batch` (prioritized agents at the learner's max_seen_priority);
    4. gate: if replay.size < min_replay_capacity, return the actions (no learn step, no target sync);
    5. learn and sync: for the frames f of the tick in increasing order, one `_learn()` where f % learn_period == 0,
       then `sync_target()` + `check_device_flags()` where f % target_network_update_period == 0;
    6. return the actions without waiting for the learn steps: the next tick's act is ordered after them on the stream.
  With E = 1 this is `step`'s control flow.  The tick synchronises with the device once, for the actions, plus the flag
  reads at target syncs."""

  def __init__(self, train_agent: _DeviceAgent, num_streams: int, rng_key, per_stream_noise: bool = False,
               preprocessor_kwargs: Optional[Mapping[str, Any]] = None):
    if not isinstance(train_agent, _DeviceAgent):
      raise TypeError('train_agent must be one of the training agents (%s)' % ', '.join(sorted(AGENTS)))
    E = int(num_streams)
    L = train_agent.learner
    if E < 1:
      raise ValueError('num_streams must be >= 1')
    if E > L.batch_size:                       # acted through an acting context: its limits apply
      if E > ACTOR_MAX_STREAMS:
        raise ValueError('num_streams %d exceeds the acting limit of %d streams' % (E, ACTOR_MAX_STREAMS))
      err = _acting_rows_error(L.net, E)
      if err:
        raise ValueError(err)
    acc = train_agent._transition_accumulator
    if not isinstance(acc, replay_lib.NStepTransitionAccumulator):
      raise ValueError('the agent needs a TransitionAccumulator or NStepTransitionAccumulator')
    kwargs = dict(preprocessor_kwargs or {})
    if not kwargs.pop('device_observations', True):
      raise ValueError('the trainer keeps its frame stacks on the device: device_observations must be True')
    kwargs.setdefault('device', L.device)
    self._agent = train_agent
    self._E = E
    self._pre = processors.VectorizedAtariPreprocessor(E, device_observations=True, **kwargs)
    self._acc = replay_lib.VectorNStepAccumulator(E, acc._transitions.maxlen, device=L.device)
    self._actor = BatchedEpsilonGreedyActor(L, E, exploration_epsilon=0.0, rng_key=rng_key,
                                            per_stream_noise=per_stream_noise)
    self._actions = np.zeros(E, np.int32)
    self._has_action = np.zeros(E, bool)
    self._learn_steps = 0
    self._q_host = torch.zeros((E, L.net.num_actions), dtype=torch.float32).pin_memory()
    self._q_pending = None                     # (event, acting streams) of the last act's q-value copy
    self._statistics = {'state_value': np.nan}
    self._episode_return = np.zeros(E)
    self._episode_length = np.zeros(E, np.int64)
    self._num_episodes = np.zeros(E, np.int64)

  # -- one tick ------------------------------------------------------------------------------------
  def step(self, frames, step_type, reward, discount, lives) -> np.ndarray:
    """frames: uint8 [E, H, W, 3] raw RGB (device tensor, or host array: one H2D copy); step_type int [E]; reward /
    discount float [E] with NaN for None (FIRST timesteps); lives int [E].  Returns the E actions, int32 [E]."""
    step_type, reward, discount, lives = self._check(frames, step_type, reward, discount, lives)
    ag = self._agent
    E = self._E
    t0 = ag._frame_t
    ag._frame_t = t0 + E
    out = self._pre.step_arrays(frames, step_type, reward, discount, lives)
    self._track_episodes(step_type, reward)
    emit = out['emit']
    if np.any(~emit & ~self._has_action):
      raise RuntimeError('Cannot repeat if action has never been selected.')
    if emit.any():
      new = self._actor.step(self._pre.stacks, epsilon=self._epsilon_at(t0 + 1))
      self._actions = np.where(emit, new, self._actions).astype(np.int32)
      self._has_action |= emit
      self._q_host.copy_(self._actor.q_values, non_blocking=True)
      ev = torch.cuda.Event()
      ev.record()
      self._q_pending = (ev, emit.copy())
      batch = self._acc.step(emit, out['step_type'], out['reward'], out['discount'], self._pre.stacks, self._actions)
      if batch is not None:
        if ag.PRIORITIZED:
          ag._replay.add_batch(batch, ag._learner.max_seen_priority)
        else:
          ag._replay.add_batch(batch)
    actions = self._actions.copy()
    if ag._replay.size < ag._min_replay_capacity:
      return actions
    lo, hi = t0 + 1, t0 + E
    due = sorted([(f, 0) for f in _due(lo, hi, ag._learn_period)] +
                 [(f, 1) for f in _due(lo, hi, ag._target_network_update_period)])
    for _, sync in due:                        # at a frame due for both, the learn step comes first
      if sync:
        ag._learner.sync_target()
        ag.check_device_flags()
      else:
        ag._learn()
        self._learn_steps += 1
    return actions

  def _check(self, frames, step_type, reward, discount, lives):
    E = self._E
    shape = tuple(frames.shape)
    dtype_ok = frames.dtype == torch.uint8 if isinstance(frames, torch.Tensor) else np.asarray(frames).dtype == np.uint8
    if len(shape) != 4 or shape[0] != E or shape[3] != 3 or not dtype_ok:
      raise ValueError('frames must be uint8 [%d, H, W, 3], got %s %s' % (E, frames.dtype, shape))
    if self._pre._in_shape is not None and shape[1:] != self._pre._in_shape:
      raise ValueError('frame shape changed: %s vs %s' % (shape[1:], self._pre._in_shape))
    arrays = (np.asarray(step_type, np.int64), np.asarray(reward, np.float64), np.asarray(discount, np.float64),
              np.asarray(lives, np.int64))
    for name, a in zip(('step_type', 'reward', 'discount', 'lives'), arrays):
      if a.shape != (E,):
        raise ValueError('%s must have shape (%d,), got %s' % (name, E, a.shape))
    return arrays

  def _epsilon_at(self, t: int) -> float:
    ag = self._agent
    return 0.0 if ag.GREEDY or ag._exploration_epsilon is None else float(ag._exploration_epsilon(t))

  def _track_episodes(self, step_type, reward):
    first = step_type == int(parts.StepType.FIRST)
    self._episode_return[first] = 0.0
    self._episode_length[first] = 0
    self._episode_return += np.where(first | np.isnan(reward), 0.0, reward)
    self._episode_length += 1
    self._num_episodes += step_type == int(parts.StepType.LAST)

  def reset(self, stream=None) -> None:
    """`Agent.reset` (which `run_loop` calls before every episode) for every stream, or for one stream or a sequence of
    streams, e.g. those whose last timestep was LAST: their preprocessor and accumulator state and their last action."""
    if stream is None:
      self._pre.reset()
      self._acc.reset()
      self._has_action[:] = False
      return
    for e in np.atleast_1d(np.asarray(stream, np.int64)):    # the streams ending an episode, not every stream
      self._pre.reset(int(e))
      self._acc.reset(int(e))
      self._has_action[e] = False

  # -- surface ------------------------------------------------------------------------------------------------------
  @property
  def num_streams(self) -> int:
    return self._E

  @property
  def agent(self) -> _DeviceAgent:
    return self._agent

  @property
  def frame_t(self) -> int:
    return self._agent._frame_t

  @property
  def learn_steps(self) -> int:
    """Learner steps this trainer has run."""
    return self._learn_steps

  @property
  def exploration_epsilon(self) -> float:
    return self._agent.exploration_epsilon

  @property
  def statistics(self) -> Mapping[str, float]:
    """`state_value`: the mean over the streams that acted in the last acting tick of their max q-value."""
    if self._q_pending is not None:
      ev, acted = self._q_pending
      ev.synchronize()
      self._statistics['state_value'] = float(self._q_host.numpy()[acted].max(axis=1).mean())
      self._q_pending = None
    return self._statistics

  @property
  def episode_return(self) -> np.ndarray:
    """Per stream: the summed raw rewards of its current episode (after a LAST timestep: of the episode it ended)."""
    return self._episode_return.copy()

  @property
  def episode_length(self) -> np.ndarray:
    """Per stream: the timesteps of its current episode, FIRST included (after LAST: of the episode it ended)."""
    return self._episode_length.copy()

  @property
  def num_episodes(self) -> np.ndarray:
    """Per stream: the episodes it has completed (LAST timesteps seen)."""
    return self._num_episodes.copy()

  def get_state(self) -> Mapping[str, Any]:
    return dict(self._stream_state(), agent=self._agent.get_state())

  def set_state(self, state: Mapping[str, Any]) -> None:
    self._check_streams(state)
    self._agent.set_state(state['agent'])
    self._set_stream_state(state)

  def save_checkpoint(self, directory: str) -> None:
    """The agent's checkpoint directory (`_DeviceAgent.save_checkpoint`) in `agent/`, plus the per-stream state of
    `get_state` (actions, RandomStates, preprocessor, accumulator, episode statistics) pickled in `trainer.pkl`."""
    from dqn_zoo_b200 import checkpoint as ck
    self._checkpoint_writer(snapshot=False)(directory, ck.Transfer(self._agent.learner.device))

  def snapshot_checkpoint(self):
    """A `checkpoint.Snapshot` of the trainer after the learn steps of the ticks so far (`_DeviceAgent.
    snapshot_checkpoint`), with the per-stream state pickled now.  Its `write(directory)` gives the files
    `save_checkpoint` would give now, byte for byte, while later ticks run."""
    from dqn_zoo_b200 import checkpoint as ck
    held = []
    return ck.Snapshot(self._checkpoint_writer(snapshot=True, held=held), held, self._agent.learner.device)

  def snapshot_checkpoint_bytes(self) -> int:
    """An upper bound of the device memory `snapshot_checkpoint()` takes now."""
    return self._agent.snapshot_checkpoint_bytes()

  def _checkpoint_writer(self, snapshot, held=None):
    from dqn_zoo_b200 import checkpoint as ck
    streams = pickle.dumps(self._stream_state(), protocol=pickle.HIGHEST_PROTOCOL)
    agent = self._agent._checkpoint_writer(snapshot, held)

    def write(directory, xfer):
      os.makedirs(directory, exist_ok=True)
      agent(os.path.join(directory, 'agent'), xfer)
      ck.write_bytes(os.path.join(directory, 'trainer.pkl'), streams)
    return write

  def load_checkpoint(self, directory: str) -> None:
    """Restores `save_checkpoint` of a trainer with the same stream count over the same kind of agent."""
    try:
      with open(os.path.join(directory, 'trainer.pkl'), 'rb') as f:
        state = pickle.load(f)
    except (OSError, pickle.UnpicklingError, EOFError) as e:
      raise ValueError('%s is not a readable trainer checkpoint: %s' % (directory, e)) from e
    self._check_streams(state)
    self._agent.load_checkpoint(os.path.join(directory, 'agent'))
    self._set_stream_state(state)

  def _check_streams(self, state):
    if np.shape(state['actions']) != (self._E,):
      raise ValueError('state is for %d streams, this trainer has %d' % (len(state['actions']), self._E))

  def _stream_state(self) -> Mapping[str, Any]:
    return {
        'frame_t': self._agent._frame_t,
        'actions': self._actions.copy(),
        'has_action': self._has_action.copy(),
        'learn_steps': self._learn_steps,
        # the replay draws its samples from a RandomState the agent's state leaves to the run (as the reference does)
        'replay_rng': self._agent._replay._rng_state(),
        'actor_rng': self._actor._rng.get_state(),
        'actor_t': self._actor._t,
        'preprocessor': self._pre.get_state(),
        'accumulator': self._acc.get_state(),
        'statistics': dict(self.statistics),
        'episodes': (self._episode_return.copy(), self._episode_length.copy(), self._num_episodes.copy()),
    }

  def _set_stream_state(self, state: Mapping[str, Any]) -> None:
    self._agent._frame_t = state['frame_t']
    self._actions = np.array(state['actions'], np.int32)
    self._has_action = np.array(state['has_action'], bool)
    self._learn_steps = int(state['learn_steps'])
    self._agent._replay._set_rng_state(state['replay_rng'])
    self._actor._rng.set_state(state['actor_rng'])
    self._actor._t = int(state['actor_t'])
    self._pre.set_state(state['preprocessor'])
    self._acc.set_state(state['accumulator'])
    self._statistics = dict(state['statistics'])
    self._q_pending = None
    ret, length, count = state['episodes']
    self._episode_return, self._episode_length, self._num_episodes = (np.array(ret), np.array(length),
                                                                      np.array(count))


class OfflineTrainer:
  """Trains an agent offline from the fixed replay it holds (DESIGN.md §20): learner steps only, no acting and no
  inserts, as in offline RL on a recorded dataset (Agarwal, Schuurmans & Norouzi, ICML 2020).  Combine it with the
  agent's `cql_alpha` for conservative Q-learning (Kumar et al., NeurIPS 2020).

  It uses `train_agent`'s learner, replay and CUDA graph in place: `step(n)` runs n of the agent's own learner steps
  (`_learn()`, host draws in the reference's order; a prioritized replay keeps writing priorities back).  After update
  u (counted from 1 across calls) with u % target_update_period == 0 it syncs the target network and reads the
  device's error flags, as `step` does on the agent's target-update cadence.  The default period is the agent's own
  cadence counted in updates, max(1, target_network_update_period // learn_period).  Nothing else of the agent moves:
  not `frame_t`, the exploration schedule, the acting RandomState or the replay's contents, and no
  `min_replay_capacity` gate applies.  A dataset is a replay filled by any other means, e.g. by a `VectorTrainer`
  whose agent never reaches its learning gate, saved with `replay.save_checkpoint` and restored with
  `load_checkpoint`."""

  def __init__(self, train_agent: _DeviceAgent, target_update_period: Optional[int] = None):
    if not isinstance(train_agent, _DeviceAgent):
      raise TypeError('OfflineTrainer needs one of the device agents, got %s' % type(train_agent).__name__)
    if target_update_period is None:
      target_update_period = max(1, train_agent._target_network_update_period // train_agent._learn_period)
    if int(target_update_period) != target_update_period or target_update_period < 1:
      raise ValueError('target_update_period must be an integer >= 1, got %r' % (target_update_period,))
    self._agent = train_agent
    self._period = int(target_update_period)
    self._updates = 0

  @property
  def agent(self) -> _DeviceAgent:
    return self._agent

  @property
  def target_update_period(self) -> int:
    return self._period

  @property
  def updates(self) -> int:
    """Learner steps taken so far (restored by `set_state` / `load_checkpoint`)."""
    return self._updates

  def step(self, num_updates: int = 1) -> None:
    """`num_updates` learner steps on the replay; ValueError on an empty replay."""
    if self._agent._replay.size == 0:
      raise ValueError('offline training needs a non-empty replay')
    for _ in range(int(num_updates)):
      self._agent._learn()
      self._updates += 1
      if self._updates % self._period == 0:
        self._agent.learner.sync_target()
        self._agent.check_device_flags()

  def get_state(self) -> Mapping[str, Any]:
    """The agent's state plus `updates` and the replay's RandomState, which the agent's state leaves to the run."""
    return dict(self._own_state(), agent=self._agent.get_state())

  def set_state(self, state: Mapping[str, Any]) -> None:
    self._agent.set_state(state['agent'])
    self._set_own_state(state)

  def save_checkpoint(self, directory: str) -> None:
    """The agent's checkpoint directory (`_DeviceAgent.save_checkpoint`, its replay included) in `agent/`, plus
    `updates`, the period and the replay's RandomState pickled in `offline.pkl`."""
    from dqn_zoo_b200 import checkpoint as ck
    os.makedirs(directory, exist_ok=True)
    self._agent.save_checkpoint(os.path.join(directory, 'agent'))
    ck.write_bytes(os.path.join(directory, 'offline.pkl'), pickle.dumps(self._own_state(), protocol=pickle.HIGHEST_PROTOCOL))

  def load_checkpoint(self, directory: str) -> None:
    """Restores `save_checkpoint` of a trainer with the same target-update period over the same kind of agent."""
    try:
      with open(os.path.join(directory, 'offline.pkl'), 'rb') as f:
        state = pickle.load(f)
    except (OSError, pickle.UnpicklingError, EOFError) as e:
      raise ValueError('%s is not a readable offline trainer checkpoint: %s' % (directory, e)) from e
    if state.get('target_update_period') != self._period:
      raise ValueError('checkpoint target_update_period %r != %d' % (state.get('target_update_period'), self._period))
    self._agent.load_checkpoint(os.path.join(directory, 'agent'))
    self._set_own_state(state)

  def _own_state(self) -> Mapping[str, Any]:
    return {'format': 'dqn_zoo_b200.offline', 'version': 1, 'updates': self._updates,
            'target_update_period': self._period, 'replay_rng': self._agent._replay._rng_state()}

  def _set_own_state(self, state: Mapping[str, Any]) -> None:
    self._updates = int(state['updates'])
    self._agent._replay._set_rng_state(state['replay_rng'])


class VectorEvaluator:
  """Evaluates an agent on E environment streams: the evaluation phase of the run drivers (`eval_agent.network_params =
  train_agent.online_params` + an epsilon-greedy actor, dqn/run_atari.py:250-290) as one tick of E timesteps, over a
  frozen parameter snapshot.

  `network_or_learner` is a `NetworkSpec` or a `Learner` with the network to evaluate; either only shapes the evaluator
  (a learner's parameters are not read until `network_params` is set).  The evaluator owns a
  `VectorizedAtariPreprocessor(E, device_observations=True)` and a frozen acting context (`Learner.actor(E,
  frozen=True)`): its own parameter snapshot, weight images and generator counter, so evaluating neither reads the
  training learner's live parameters nor shifts its noise or tau draws, and it may run beside training.  It always acts
  through that context, at any E in [1, 1024] (IQN: E * tau_samples_policy <= 16384).

  Tick contract (`step`): preprocess the E raw timesteps; if any stream emits a timestep, ONE act call for all E streams
  at `exploration_epsilon`, with 2E host uniforms from a RandomState seeded by `rng_key` (as `BatchedEpsilonGreedyActor`)
  when epsilon > 0; emitting streams take the new action, the others repeat their last one (RuntimeError if a stream
  has none yet).  IQN draws E x tau_samples_policy taus and rainbow one noise apply (or, with `per_stream_noise`, one
  per stream) per acting tick from the actor's counter.  The tick waits for its actions only.

  `stream`: a `torch.cuda.Stream` on which all of the evaluator's device work is enqueued (e.g. to evaluate one
  iteration while the next one trains on the default stream).  Setting `network_params` then enqueues the snapshot copy
  on the caller's current stream, ordered after both the caller's earlier work and the evaluator's earlier acts, and
  makes the evaluator's stream wait for it through an event."""

  # the trainer's input checks and episode bookkeeping (they read only _E, _pre and the episode arrays)
  _check = VectorTrainer._check
  _track_episodes = VectorTrainer._track_episodes
  # the batched actor's acting tick (it reads only _E, _rng, _seed, _per_stream_noise and the staging buffers)
  _tick = BatchedEpsilonGreedyActor._tick

  def __init__(self, network_or_learner, num_streams: int, exploration_epsilon: float, rng_key,
               per_stream_noise: bool = False, preprocessor_kwargs: Optional[Mapping[str, Any]] = None, stream=None):
    E = int(num_streams)
    if E < 1 or E > ACTOR_MAX_STREAMS:
      raise ValueError('num_streams must be in [1, %d], got %d' % (ACTOR_MAX_STREAMS, E))
    if isinstance(network_or_learner, learner_lib.Learner):
      shape_learner = network_or_learner
    elif isinstance(network_or_learner, NetworkSpec):
      shape_learner = None
    else:
      raise TypeError('network_or_learner must be a NetworkSpec or a Learner')
    net = network_or_learner.net if shape_learner is not None else network_or_learner
    err = _acting_rows_error(net, E)
    if err:
      raise ValueError(err)
    if per_stream_noise and not learner_lib.noisy_layers(net):
      raise ValueError('per_stream_noise needs a network with noisy layers')
    kwargs = dict(preprocessor_kwargs or {})
    if not kwargs.pop('device_observations', True):
      raise ValueError('the evaluator keeps its frame stacks on the device: device_observations must be True')
    self._stream = stream
    self._E = E
    self._net = net
    self._epsilon = float(exploration_epsilon)
    self._per_stream_noise = bool(per_stream_noise)
    seed = int(np.asarray(rng_key).reshape(-1)[-1]) & 0x7FFFFFFF
    self._rng = np.random.RandomState(seed)
    self._seed = seed
    with self._on_stream():
      if shape_learner is None:            # the frozen actor takes only the configuration; the learner is dropped
        shape_learner = learner_lib.Learner(net)
      kwargs.setdefault('device', shape_learner.device)
      self._actor = shape_learner.actor(E, frozen=True)
      self._pre = processors.VectorizedAtariPreprocessor(E, device_observations=True, **kwargs)
      self._explore_host = torch.zeros((2, E), dtype=torch.float32).pin_memory()
      self._explore_dev = torch.zeros((2, E), dtype=torch.float32, device=shape_learner.device)
      self._actions_host = torch.zeros(E, dtype=torch.int32).pin_memory()
    del shape_learner
    self._actions = np.zeros(E, np.int32)
    self._has_action = np.zeros(E, bool)
    self._episode_return = np.zeros(E)
    self._episode_length = np.zeros(E, np.int64)
    self._num_episodes = np.zeros(E, np.int64)

  def _on_stream(self):
    return torch.cuda.stream(self._stream) if self._stream is not None else contextlib.nullcontext()

  # -- the snapshot ---------------------------------------------------------------------------------------------------
  @property
  def network_params(self):
    """The snapshot as an `hk.Params`-shaped dict of host arrays (None before it is set)."""
    if not self._actor.loaded:
      return None
    with self._on_stream():
      flat = self._actor.get_params()
    out = {}
    for name, value in flat.items():
      mod, leaf = learner_lib.haiku_name(name, self._net.kind)
      out.setdefault(mod, {})[leaf] = value
    return out

  @network_params.setter
  def network_params(self, params) -> None:
    """`EpsilonGreedyActor.network_params`'s inputs: a `Learner` (one device-to-device copy of its online parameters),
    an `hk.Params`-shaped dict or a flat {canonical_name: array} dict.  None leaves the evaluator without parameters."""
    if params is None:
      self._actor.loaded = False
      return
    if self._stream is None:
      self._actor.load_params(params)
      return
    caller = torch.cuda.current_stream()
    caller.wait_stream(self._stream)       # the evaluator's enqueued acts read the previous snapshot
    self._actor.load_params(params)
    done = torch.cuda.Event()
    done.record(caller)
    self._stream.wait_event(done)

  # -- one tick -------------------------------------------------------------------------------------------------------
  def step(self, frames, step_type, reward, discount, lives) -> np.ndarray:
    """`VectorTrainer.step`'s arguments: frames uint8 [E, H, W, 3] raw RGB (device tensor, or host array: one H2D copy);
    step_type int [E]; reward / discount float [E] with NaN for None (FIRST timesteps); lives int [E].  Returns the E
    actions, int32 [E]."""
    if not self._actor.loaded:
      raise RuntimeError('network_params have not been set.')
    step_type, reward, discount, lives = self._check(frames, step_type, reward, discount, lives)
    with self._on_stream():
      out = self._pre.step_arrays(frames, step_type, reward, discount, lives)
      self._track_episodes(step_type, reward)
      emit = out['emit']
      if np.any(~emit & ~self._has_action):
        raise RuntimeError('Cannot repeat if action has never been selected.')
      if emit.any():
        new = self._act()
        self._actions = np.where(emit, new, self._actions).astype(np.int32)
        self._has_action |= emit
    return self._actions.copy()

  def _act(self) -> np.ndarray:
    return self._tick(self._actor, self._pre.stacks, self._epsilon)[0]

  def reset(self, streams=None) -> None:
    """`Agent.reset` for every stream, or for one stream or a sequence of streams (e.g. those whose last timestep was
    LAST): their preprocessor state and their last action."""
    with self._on_stream():
      if streams is None:
        self._pre.reset()
        self._has_action[:] = False
        return
      for e in np.atleast_1d(np.asarray(streams, np.int64)):
        self._pre.reset(int(e))
        self._has_action[e] = False

  # -- surface --------------------------------------------------------------------------------------------------------
  @property
  def num_streams(self) -> int:
    return self._E

  @property
  def actor(self) -> learner_lib.Actor:
    """The frozen acting context."""
    return self._actor

  @property
  def stream(self):
    return self._stream

  @property
  def statistics(self) -> Mapping[str, float]:
    return {}

  @property
  def episode_return(self) -> np.ndarray:
    """Per stream: the summed raw rewards of its current episode (after a LAST timestep: of the episode it ended)."""
    return self._episode_return.copy()

  @property
  def episode_length(self) -> np.ndarray:
    """Per stream: the timesteps of its current episode, FIRST included (after LAST: of the episode it ended)."""
    return self._episode_length.copy()

  @property
  def num_episodes(self) -> np.ndarray:
    """Per stream: the episodes it has completed (LAST timesteps seen)."""
    return self._num_episodes.copy()

  def get_state(self) -> Mapping[str, Any]:
    """The snapshot, the actor's generator counter, the exploration RandomState, the preprocessor, the last actions and
    the episode statistics: a restored evaluator continues bit for bit."""
    with self._on_stream():
      return {
          'network_params': self._actor.get_params() if self._actor.loaded else None,
          'counter': self._actor.counter,
          'rng': self._rng.get_state(),
          'seed': self._seed,
          'preprocessor': self._pre.get_state(),
          'actions': self._actions.copy(),
          'has_action': self._has_action.copy(),
          'episodes': (self._episode_return.copy(), self._episode_length.copy(), self._num_episodes.copy()),
      }

  def set_state(self, state: Mapping[str, Any]) -> None:
    if np.shape(state['actions']) != (self._E,):
      raise ValueError('state is for %d streams, this evaluator has %d' % (len(state['actions']), self._E))
    self.network_params = state['network_params']
    with self._on_stream():
      self._actor.counter = int(state['counter'])
      self._pre.set_state(state['preprocessor'])
    self._rng.set_state(state['rng'])
    self._seed = int(state['seed'])
    self._actions = np.array(state['actions'], np.int32)
    self._has_action = np.array(state['has_action'], bool)
    ret, length, count = state['episodes']
    self._episode_return, self._episode_length, self._num_episodes = (np.array(ret), np.array(length),
                                                                      np.array(count))
