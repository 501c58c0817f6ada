"""GPU: `agent.VectorTrainer`, one training agent fed by E environment streams.  The tick contract (learn and target-sync
cadence behind the minimum-replay gate), equality with the hand composition of the batched parts, E = 1 against
`Agent.step` under `parts.run_loop`, action repeat and input errors, acting beyond the learner's batch, state round
trips and CUDA-graph reuse."""

import itertools

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

FIRST, MID, LAST = 0, 1, 2
RAW = (210, 160, 3)
POOL = 8


# -- fixtures --------------------------------------------------------------------------------------------------------
def _script(E, ticks, seed, max_len=24):
  """Struct-of-arrays timesteps of E streams for `ticks` ticks: (pool index, step_type, reward, discount, lives).
  Every stream starts with FIRST at tick 0; episodes have random lengths, so later episode starts are staggered across
  streams; a life is lost now and then.  A stream whose timestep is LAST is reset before the next tick."""
  rs = np.random.RandomState(seed)
  left = np.zeros(E, np.int64)
  fresh = np.ones(E, bool)
  lives = np.full(E, 3)
  out = []
  for t in range(ticks):
    left = np.where(fresh, rs.randint(3, max_len, E), left - 1)
    st = np.where(fresh, FIRST, np.where(left <= 0, LAST, MID))
    reward = rs.choice([0.0, 0.0, 1.0, -1.0, 2.0], E)
    reward[fresh] = np.nan
    discount = np.where(st == LAST, 0.0, 1.0)
    discount[fresh] = np.nan
    lives = np.where(fresh, 3, lives - ((st == MID) & (rs.uniform(size=E) < 0.03) & (lives > 1)))
    out.append((t % POOL, st, reward, discount, lives.copy()))
    fresh = st == LAST
  return out


def _frames(E, seed):
  """POOL batches of E raw RGB frames, resident on the device."""
  rs = np.random.RandomState(seed)
  return [torch.as_tensor(rs.randint(0, 256, (E,) + RAW).astype(np.uint8), device='cuda') for _ in range(POOL)]


def _agent(kind, min_fill, seed=5, capacity=512, dedup=False, learn_period=4, target_period=16, epsilon=0.1):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  structure = dr.Transition(None, None, None, None, None)
  rs = np.random.RandomState(seed)
  if kind == 'rainbow':
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.5, lambda t: 0.4, 1e-3, True, rs, frame_dedup=dedup)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, frame_dedup=dedup)
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(3 if kind == 'rainbow' else 1), replay=rep,
                batch_size=32, min_replay_capacity_fraction=min_fill / capacity, learn_period=learn_period,
                target_network_update_period=target_period, rng_key=[0, seed])
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common)
  if kind == 'iqn':
    return ag.Iqn(exploration_epsilon=lambda t: epsilon, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                  tau_samples_s_t=64, **common)
  return ag.AGENTS[kind](exploration_epsilon=lambda t: epsilon, grad_error_bound=1.0 / 32, **common)


def _trainer(agent, E, **kw):
  from dqn_zoo_b200 import agent as ag
  return ag.VectorTrainer(agent, num_streams=E, rng_key=[0, 11], **kw)


def _drive(trainer, frames, script, lo, hi, on_tick=None):
  actions = []
  for t in range(lo, hi):
    k, st, rw, dc, lv = script[t]
    t0 = trainer.frame_t
    actions.append(trainer.step(frames[k], st, rw, dc, lv))
    if on_tick is not None:
      on_tick(t0)
    ended = np.nonzero(st == LAST)[0]
    if ended.size:
      trainer.reset(ended)
  return actions


class _Hand:
  """The tick written out with the batched parts, in the order of the tick contract."""

  def __init__(self, agent, E, per_stream_noise=False):
    from dqn_zoo_b200 import agent as ag
    from dqn_zoo_b200 import processors
    from dqn_zoo_b200 import replay as dr
    self.ag, self.E = agent, E
    self.pre = processors.VectorizedAtariPreprocessor(E, device_observations=True)
    self.acc = dr.VectorNStepAccumulator(E, 3 if agent.KIND == 'rainbow' else 1)
    self.actor = ag.BatchedEpsilonGreedyActor(agent.learner, E, exploration_epsilon=0.0, rng_key=[0, 11],
                                              per_stream_noise=per_stream_noise)
    self.actions = np.zeros(E, np.int32)
    self.t = -1

  def tick(self, frames, st, rw, dc, lv):
    ag, E = self.ag, self.E
    t0, self.t = self.t, self.t + E
    out = self.pre.step_arrays(frames, st, rw, dc, lv)
    emit = out['emit']
    if emit.any():
      eps = 0.0 if ag._exploration_epsilon is None else ag._exploration_epsilon(t0 + 1)
      self.actions = np.where(emit, self.actor.step(self.pre.stacks, epsilon=eps), self.actions).astype(np.int32)
      batch = self.acc.step(emit, out['step_type'], out['reward'], out['discount'], self.pre.stacks, self.actions)
      if batch is not None:
        if ag.PRIORITIZED:
          ag._replay.add_batch(batch, ag.learner.max_seen_priority)
        else:
          ag._replay.add_batch(batch)
    if ag._replay.size >= ag._min_replay_capacity:
      for f in range(t0 + 1, t0 + E + 1):
        if f % ag._learn_period == 0:
          ag._learn()
        if f % ag._target_network_update_period == 0:
          ag.learner.sync_target()
    return self.actions.copy()

  def drive(self, frames, script):
    actions = []
    for k, st, rw, dc, lv in script:
      actions.append(self.tick(frames[k], st, rw, dc, lv))
      for e in np.nonzero(st == LAST)[0]:
        self.pre.reset(int(e))
        self.acc.reset(int(e))
    return actions


def _assert_same(a, b, path='state'):
  if isinstance(a, dict):
    assert sorted(a) == sorted(b), path
    for k in a:
      _assert_same(a[k], b[k], '%s[%r]' % (path, k))
  elif isinstance(a, (list, tuple)):
    assert len(a) == len(b), path
    for i, (x, y) in enumerate(zip(a, b)):
      _assert_same(x, y, '%s[%d]' % (path, i))
  elif isinstance(a, (np.ndarray, torch.Tensor)):
    x = a.cpu().numpy() if isinstance(a, torch.Tensor) else a
    y = b.cpu().numpy() if isinstance(b, torch.Tensor) else b
    np.testing.assert_array_equal(x, y, err_msg=path)
  elif isinstance(a, float) and np.isnan(a):
    assert np.isnan(b), path
  else:
    assert a == b, (path, a, b)


def _assert_same_learner(x, y):
  torch.cuda.synchronize()
  assert torch.equal(x.learner.online, y.learner.online)
  assert torch.equal(x.learner.target, y.learner.target)
  assert torch.equal(x.learner.opt_state, y.learner.opt_state)
  assert torch.equal(x.learner.counters, y.learner.counters)


def _min_fill(E):
  return 8 if E == 1 else 3 * E


def _ticks(E):
  return 80 if E == 1 else 36


# -- 1 and 5: cadence, on both sides of the learner's batch ------------------------------------------------------------
@pytest.mark.parametrize('kind,E', list(itertools.product(('dqn', 'rainbow'), (1, 7, 48, 100))))
def test_learn_and_sync_cadence(kind, E):
  """learn_steps equals the gated frames with f % learn_period == 0; each target sync copies the online parameters of
  its frame; nothing is learned or synced before the replay holds min_replay_capacity transitions."""
  ag = _agent(kind, _min_fill(E))
  tr = _trainer(ag, E)
  L = ag.learner
  assert (tr._actor._actor is not None) == (E > L.batch_size)
  events, snapshots = [], []
  learn, sync = ag._learn, L.sync_target

  def spy_learn():
    events.append('L')
    learn()

  def spy_sync():
    events.append('S')
    snapshots.append(L.online.clone())
    sync()

  ag._learn, L.sync_target = spy_learn, spy_sync
  expected_learns, opened = 0, False
  script = _script(E, _ticks(E), seed=E)

  def check(t0):
    nonlocal expected_learns, opened
    want = []
    if ag._replay.size >= ag._min_replay_capacity:
      opened = True
      for f in range(t0 + 1, t0 + E + 1):
        want += ['L'] * (f % ag._learn_period == 0) + ['S'] * (f % ag._target_network_update_period == 0)
    assert events == want, (t0, events, want)
    expected_learns += want.count('L')
    assert tr.learn_steps == expected_learns
    assert tr.frame_t == t0 + E
    if 'S' in events:
      torch.cuda.synchronize()
      assert torch.equal(L.target, snapshots[-1])
    events.clear()

  _drive(tr, _frames(E, 1), script, 0, len(script), on_tick=check)
  assert opened and tr.learn_steps > 0 and snapshots, 'the gate never opened'


# -- 2 and 5: equal to the hand composition ----------------------------------------------------------------------------
@pytest.mark.parametrize('kind,E,dedup,per_stream', [('dqn', 48, False, False), ('rainbow', 48, False, False),
                                                     ('iqn', 24, False, False), ('dqn', 48, True, False),
                                                     ('rainbow', 100, False, True), ('dqn', 100, False, False)])
def test_equals_the_hand_composition(kind, E, dedup, per_stream):
  script = _script(E, _ticks(E), seed=3)
  frames = _frames(E, 2)
  a = _agent(kind, _min_fill(E), dedup=dedup)
  b = _agent(kind, _min_fill(E), dedup=dedup)
  tr = _trainer(a, E, per_stream_noise=per_stream)
  got = _drive(tr, frames, script, 0, len(script))
  want = _Hand(b, E, per_stream_noise=per_stream).drive(frames, script)
  assert tr.learn_steps > 0
  np.testing.assert_array_equal(np.stack(got), np.stack(want))
  _assert_same(a._replay.get_state(), b._replay.get_state())
  _assert_same_learner(a, b)


# -- 3: E = 1 against Agent.step -----------------------------------------------------------------------------------------
class _Env:
  """Host RGB frames and lives, episodes of 10..29 steps."""

  def __init__(self, seed):
    self.rs = np.random.RandomState(seed)
    self.left = 0

  def _obs(self):
    return self.rs.randint(0, 256, RAW).astype(np.uint8), 3

  def reset(self):
    from dqn_zoo_b200 import parts
    self.left = int(self.rs.randint(10, 30))
    return parts.TimeStep(parts.StepType.FIRST, None, None, self._obs())

  def step(self, action):
    from dqn_zoo_b200 import parts
    del action
    self.left -= 1
    last = self.left <= 0
    return parts.TimeStep(parts.StepType.LAST if last else parts.StepType.MID, float(self.rs.randint(-1, 2)),
                          0.0 if last else 1.0, self._obs())


def test_single_stream_equals_agent_step():
  """A greedy dqn trainer with one stream against `Agent.step` under `parts.run_loop`, same environment and seeds:
  same actions, same replay, bit-identical parameters.  Greedy, so neither side draws exploration uniforms.  The two
  sides compute q-values on different paths (`Learner.q_values` and the batched act); with freshly initialised
  parameters on random frames no two actions come within rounding of a tie, so the argmaxes agree."""
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import processors
  N = 240
  a = _agent('dqn', 8, capacity=128, epsilon=0.0)
  a._preprocessor = processors.atari(device_observations=True)
  b = _agent('dqn', 8, capacity=128, epsilon=0.0)
  seq = itertools.islice(parts.run_loop(a, _Env(4)), N)
  want = [None if act is None else int(act) for _, _, _, act in seq]
  tr = _trainer(b, 1)
  env = _Env(4)
  got = []
  ts = env.reset()
  tr.reset()
  for _ in range(N):
    rgb, lives = ts.observation
    r = np.nan if ts.reward is None else ts.reward
    d = np.nan if ts.discount is None else ts.discount
    act = tr.step(rgb[None], [int(ts.step_type)], [r], [d], [lives])
    if ts.last():
      got.append(None)
      tr.reset()
      ts = env.reset()
    else:
      got.append(int(act[0]))
      ts = env.step(int(act[0]))
  assert got == want
  assert tr.frame_t == a._frame_t == N - 1
  assert tr.learn_steps == a._learn_steps > 0
  _assert_same(a._replay.get_state(), b._replay.get_state())
  _assert_same_learner(a, b)


# -- 4: action repeat and errors -----------------------------------------------------------------------------------------
def test_streams_that_do_not_emit_repeat_their_action():
  E = 7
  ag = _agent('dqn', 1024, capacity=1024, epsilon=1.0)    # the gate stays closed; every act explores
  tr = _trainer(ag, E)
  seen = {}
  step_arrays, actor_step = tr._pre.step_arrays, tr._actor.step

  def spy_pre(*args, **kw):
    seen['emit'] = out = step_arrays(*args, **kw)
    return out

  def spy_act(*args, **kw):
    seen['new'] = a = actor_step(*args, **kw)
    return a

  tr._pre.step_arrays, tr._actor.step = spy_pre, spy_act
  script = _script(E, 40, seed=8, max_len=9)
  frames = _frames(E, 0)
  prev = None
  repeats = 0
  for t in range(len(script)):
    seen.clear()
    acts = _drive(tr, frames, script, t, t + 1)[0]
    emit = seen['emit']['emit']
    if 'new' in seen:
      np.testing.assert_array_equal(acts[emit], seen['new'][emit])
    if prev is not None:
      np.testing.assert_array_equal(acts[~emit], prev[~emit])
      repeats += int((~emit).sum())
    prev = acts
  assert repeats > 0


def test_never_acted_stream_and_bad_inputs_raise():
  from dqn_zoo_b200 import agent as ag_lib
  E = 3
  ag = _agent('dqn', 64)
  tr = _trainer(ag, E)
  frames = _frames(E, 0)[0]
  nan = np.full(E, np.nan)
  with pytest.raises(RuntimeError):         # stream 2 has never acted and does not start with FIRST
    tr.step(frames, [FIRST, FIRST, MID], nan, nan, [3, 3, 3])
  tr = _trainer(_agent('dqn', 64), E)
  tr.step(frames, [FIRST] * E, nan, nan, [3] * E)
  # the preprocessor makes every stream's first timestep emit, so only a lost action can reach the check: drop stream
  # 1's and send a tick on which no stream emits
  tr._has_action[1] = False
  with pytest.raises(RuntimeError, match='never been selected'):
    tr.step(frames, [MID] * E, np.zeros(E), np.ones(E), [3] * E)
  tr = _trainer(_agent('dqn', 64), E)
  with pytest.raises(ValueError):
    tr.step(frames[:2], [FIRST] * E, nan, nan, [3] * E)
  with pytest.raises(ValueError):
    tr.step(frames[..., :2], [FIRST] * E, nan, nan, [3] * E)
  with pytest.raises(ValueError):
    tr.step(frames.float(), [FIRST] * E, nan, nan, [3] * E)
  with pytest.raises(ValueError):
    tr.step(frames, [FIRST] * (E + 1), nan, nan, [3] * E)
  with pytest.raises(ValueError):
    tr.step(frames, [FIRST] * E, nan[:2], nan, [3] * E)
  with pytest.raises(ValueError):
    ag_lib.VectorTrainer(_agent('dqn', 64), num_streams=0, rng_key=[0, 1])
  with pytest.raises(ValueError):
    ag_lib.VectorTrainer(_agent('dqn', 64), num_streams=1025, rng_key=[0, 1])
  with pytest.raises(ValueError):
    ag_lib.VectorTrainer(_agent('dqn', 64), num_streams=4, rng_key=[0, 1],
                         preprocessor_kwargs=dict(device_observations=False))


def test_iqn_above_its_acting_cap_raises():
  from dqn_zoo_b200 import agent as ag_lib
  ag = _agent('iqn', 64)                     # 64 tau samples per stream: at most 256 acting streams
  taus = ag.learner.net.tau_samples_policy
  cap = ag_lib.ACTOR_MAX_IQN_ROWS // taus
  ag_lib.VectorTrainer(ag, num_streams=cap, rng_key=[0, 1])
  with pytest.raises(ValueError, match='tau_samples_policy'):
    ag_lib.VectorTrainer(ag, num_streams=cap + 1, rng_key=[0, 1])


# -- 6: state round trip -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind,per_stream', [('rainbow', False), ('rainbow', True), ('iqn', False)])
def test_state_round_trip(kind, per_stream):
  import copy
  E, T = 24, 24
  script = _script(E, 2 * T, seed=6)
  frames = _frames(E, 6)
  a = _agent(kind, _min_fill(E))
  tr = _trainer(a, E, per_stream_noise=per_stream)
  _drive(tr, frames, script, 0, T)
  assert tr.learn_steps > 0
  state = copy.deepcopy(tr.get_state())
  got = _drive(tr, frames, script, T, 2 * T)
  b = _agent(kind, _min_fill(E), seed=99)      # different seeds: everything must come from the state
  tr2 = _trainer(b, E, per_stream_noise=per_stream)
  tr2.set_state(state)
  want = _drive(tr2, frames, script, T, 2 * T)
  np.testing.assert_array_equal(np.stack(got), np.stack(want))
  assert tr.frame_t == tr2.frame_t and tr.learn_steps == tr2.learn_steps
  _assert_same(a._replay.get_state(), b._replay.get_state())
  _assert_same_learner(a, b)
  _assert_same(tr.get_state()['preprocessor'], tr2.get_state()['preprocessor'])
  _assert_same(tr.get_state()['accumulator'], tr2.get_state()['accumulator'])
  np.testing.assert_array_equal(tr.num_episodes, tr2.num_episodes)
  np.testing.assert_array_equal(tr.episode_return, tr2.episode_return)


# -- 7: graph reuse ------------------------------------------------------------------------------------------------------
def test_graph_captured_once_and_replayed():
  E = 48
  ag = _agent('rainbow', _min_fill(E))
  tr = _trainer(ag, E)
  graphs = []

  def note(t0):
    if ag._graph is not None:
      graphs.append(ag._graph)

  replays = []
  orig = torch.cuda.CUDAGraph.replay
  try:
    torch.cuda.CUDAGraph.replay = lambda g: (replays.append(g), orig(g))[1]
    _drive(tr, _frames(E, 5), _script(E, _ticks(E), seed=5), 0, _ticks(E), on_tick=note)
  finally:
    torch.cuda.CUDAGraph.replay = orig
  assert graphs and all(g is graphs[0] for g in graphs)
  assert tr.learn_steps > 2
  assert len(replays) == tr.learn_steps - 1 and all(g is graphs[0] for g in replays)


def test_statistics_and_episode_counts():
  E = 7
  ag = _agent('dqn', 1024, capacity=1024)
  tr = _trainer(ag, E)
  assert np.isnan(tr.statistics['state_value'])
  script = _script(E, 30, seed=2, max_len=8)
  frames = _frames(E, 2)
  returns, lengths = np.zeros(E), np.zeros(E, np.int64)
  done = np.zeros(E, np.int64)
  for t, (k, st, rw, dc, lv) in enumerate(script):
    returns = np.where(st == FIRST, 0.0, returns + np.nan_to_num(rw))
    lengths = np.where(st == FIRST, 1, lengths + 1)
    done += st == LAST
    _drive(tr, frames, script, t, t + 1)
    np.testing.assert_array_equal(tr.episode_return, returns)
    np.testing.assert_array_equal(tr.episode_length, lengths)
    np.testing.assert_array_equal(tr.num_episodes, done)
  assert done.sum() > 0
  emit = tr._q_pending[1]
  q = tr._actor.q_values.cpu().numpy()
  assert tr.statistics['state_value'] == pytest.approx(float(q[emit].max(axis=1).mean()), rel=1e-6)
