"""GPU: frozen acting contexts (`Learner.actor(E, frozen=True)`, `dz_actor_create_frozen`) and `agent.VectorEvaluator`.
Frozen outputs equal live ones bit for bit, the snapshot does not follow the learner, the actor's randomness and acting
leave the learner and a trainer running beside it untouched, overlapped evaluation in the run driver changes no
statistic, streams are independent, state round trips continue bit for bit, and bad inputs are refused."""

import ctypes as C
import itertools
import os
import sys

import numpy as np
import pytest
import torch

from learner_parity import make_batch, make_case, obs_shape, random_noise
from test_gpu_vector_trainer import LAST, _agent, _assert_same, _frames, _script

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ('dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn')
STREAMS = (1, 33, 256)
CASES = ([(k, 84, E) for k in KINDS for E in STREAMS] +
         [(k, hw, E) for k in ('dqn', 'rainbow') for hw in (44, (84, 88)) for E in STREAMS])

_CASES = {}


@pytest.fixture(scope='module', autouse=True)
def _release():
  yield
  _CASES.clear()


def _case(kind, hw):
  k = (kind, hw if isinstance(hw, int) else tuple(hw))
  if k not in _CASES:
    _CASES[k] = make_case(kind, 32, hw, seed=7)
  return _CASES[k]


def _obs(spec, E, seed):
  H, W = obs_shape(spec)
  return torch.as_tensor(np.random.RandomState(seed).randint(0, 256, (E, H, W, 4)).astype(np.uint8), device='cuda')


def _inputs(spec, net, E, rs, per_stream=False):
  """Explicit randomness inputs: IQN taus [E, tau_samples_policy]; rainbow one shared apply or one apply per stream."""
  from dqn_zoo_b200 import learner as dl
  if spec.kind == 'iqn':
    return {'taus': torch.as_tensor(rs.uniform(size=(E, net.tau_samples_policy)).astype(np.float32), device='cuda')}
  if spec.kind == 'rainbow':
    if per_stream:
      raw = [random_noise(spec, rs) for _ in range(E)]
      return {'stream_noise': torch.as_tensor(dl.pack_noise(net, raw), device='cuda').view(E, -1)}
    return {'noise': torch.as_tensor(dl.pack_noise(net, [random_noise(spec, rs)]), device='cuda')}
  return {}


def _act(actor, obs, **kw):
  a, q = actor.act(obs, **kw)
  torch.cuda.synchronize()
  return a.cpu().numpy().copy(), q.cpu().numpy().copy()


def _mma_path(actor, tag):
  from dqn_zoo_b200 import _lib
  path = C.c_int32()
  _lib.call('dz_test_actor_mma_path', actor._h, tag.encode(), C.byref(path))
  return path.value


def _compare(spec, net, frozen, live, E, seed, per_stream=False):
  rs = np.random.RandomState(seed)
  obs = _obs(spec, E, seed)
  kw = _inputs(spec, net, E, rs, per_stream)
  u = torch.as_tensor(rs.uniform(size=(2, E)).astype(np.float32), device='cuda')
  for eps, x in ((0.3, u), (0.0, None)):
    fa, fq = _act(frozen, obs, epsilon=eps, explore=x, **kw)
    la, lq = _act(live, obs, epsilon=eps, explore=x, **kw)
    np.testing.assert_array_equal(fq, lq, err_msg='%s E=%d eps=%g' % (spec.kind, E, eps))
    np.testing.assert_array_equal(fa, la)
  return fq


# -- 1: frozen equals live ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind,hw,E', CASES)
def test_frozen_equals_live(kind, hw, E):
  """Same parameters and randomness inputs: bit-identical q-values and actions (rainbow with one shared apply and with
  one apply per stream)."""
  spec, net, L, _, _ = _case(kind, hw)
  frozen = L.actor(E, frozen=True)
  frozen.load_params(L)
  live = L.actor(E)
  _compare(spec, net, frozen, live, E, seed=E)
  if kind == 'rainbow':
    _compare(spec, net, frozen, live, E, seed=E + 1, per_stream=True)


def test_frozen_actor_runs_the_tensor_core_launches():
  """At 84x84x4 the frozen plan has the live plan's MMA paths; at 84x88 both act on the fp32-FMA kernels."""
  for kind, tags in (('dqn', ('conv1_fwd', 'conv2_fwd', 'conv3_fwd', 'fc1_fwd')),
                     ('rainbow', ('conv1_fwd', 'conv2_fwd', 'conv3_fwd', 'noisy1_fwd')),
                     ('iqn', ('conv1_fwd', 'conv2_fwd', 'conv3_fwd'))):
    _, _, L, _, _ = _case(kind, 84)
    frozen, live = L.actor(64, frozen=True), L.actor(64)
    for tag in tags:
      assert _mma_path(frozen, tag) == _mma_path(live, tag) >= 0, (kind, tag)
  _, _, L, _, _ = _case('dqn', (84, 88))
  with pytest.raises(ValueError):
    _mma_path(L.actor(8, frozen=True), 'conv1_fwd')


@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_load_from_learner_haiku_and_flat_dicts(kind):
  spec, net, L, _, _ = _case(kind, 84)
  E = 20
  actors = [L.actor(E, frozen=True) for _ in range(3)]
  actors[0].load_params(L)
  actors[1].load_params(L.haiku_params())
  actors[2].load_params(L.get_params())
  rs = np.random.RandomState(4)
  obs = _obs(spec, E, 4)
  kw = _inputs(spec, net, E, rs)
  outs = [_act(a, obs, **kw) for a in actors]
  for a, q in outs[1:]:
    np.testing.assert_array_equal(q, outs[0][1])
    np.testing.assert_array_equal(a, outs[0][0])
  got = actors[1].get_params()
  for name, value in L.get_params().items():
    np.testing.assert_array_equal(got[name], value)


# -- 2: the snapshot is frozen -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_snapshot_does_not_follow_the_learner(kind):
  spec, net, L, _, rs = make_case(kind, 32, 84, seed=11)
  E = 40
  frozen, live = L.actor(E, frozen=True), L.actor(E)
  frozen.load_params(L)
  obs = _obs(spec, E, 2)
  kw = _inputs(spec, net, E, np.random.RandomState(3))
  _, before = _act(frozen, obs, **kw)
  _, live_before = _act(live, obs, **kw)
  np.testing.assert_array_equal(before, live_before)
  for _ in range(3):
    (s_tm1, a, r, d, s_t), _, w, _, taus_flat, _, noise_flat = make_batch(spec, net, 32, rs)
    L.update(s_tm1, a, r, d, s_t, weights=w, taus=taus_flat, noise=noise_flat)
  _, after = _act(frozen, obs, **kw)
  _, live_after = _act(live, obs, **kw)
  np.testing.assert_array_equal(after, before)
  assert not np.array_equal(live_after, before)
  frozen.load_params(L)
  _, reloaded = _act(frozen, obs, **kw)
  np.testing.assert_array_equal(reloaded, live_after)


# -- 3: randomness is isolated -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['rainbow', 'iqn'])
def test_frozen_randomness_leaves_the_learner_alone(kind):
  _, _, L, _, _ = _case(kind, 84)
  E, seed = 24, 99
  L.counters[1] = 5
  L.generate_randomness(seed)
  torch.cuda.synchronize()
  want = (L.taus.clone(), L.noise.clone(), L.counters.clone())
  L.counters[1] = 5
  counters = L.counters.clone()
  f1, f2 = L.actor(E, frozen=True), L.actor(E, frozen=True)
  assert f1.counter == 0
  f1.counter = 5
  draws = [f1.generate_randomness(seed).clone() for _ in range(2)]
  if kind == 'rainbow':
    draws.append(f1.generate_randomness(seed, per_stream=True).clone())
  torch.cuda.synchronize()
  assert torch.equal(L.counters, counters)
  assert f1.counter == 5 + len(draws)
  L.generate_randomness(seed)
  torch.cuda.synchronize()
  assert torch.equal(L.taus, want[0]) and torch.equal(L.noise, want[1]) and torch.equal(L.counters, want[2])
  # same seed and counter: two frozen actors, and a live actor on a learner at that counter, draw the same values
  f2.counter = 5
  assert torch.equal(f2.generate_randomness(seed), draws[0])
  L.counters[1] = 6
  live = L.actor(E)
  assert torch.equal(live.generate_randomness(seed), draws[1])


# -- 4: training is isolated -------------------------------------------------------------------------------------------
def _evaluator(net_or_learner, E, eps=0.05, **kw):
  from dqn_zoo_b200 import agent as ag
  return ag.VectorEvaluator(net_or_learner, E, eps, rng_key=[0, 21], **kw)


def _train_run(kind, interleave):
  from dqn_zoo_b200 import agent as ag
  E, ticks = 12, 30
  agent = _agent(kind, min_fill=30, learn_period=2, target_period=8)
  trainer = ag.VectorTrainer(agent, num_streams=E, rng_key=[0, 11], per_stream_noise=kind == 'rainbow')
  script, frames = _script(E, ticks, seed=3), _frames(E, seed=3)
  ev = None
  if interleave:
    EE = 40
    ev = _evaluator(agent.learner, EE, per_stream_noise=kind == 'rainbow', stream=torch.cuda.Stream())
    ev_script, ev_frames = _script(EE, ticks, seed=8), _frames(EE, seed=8)
  actions = []
  for t in range(ticks):
    k, st, rw, dc, lv = script[t]
    actions.append(trainer.step(frames[k], st, rw, dc, lv))
    ended = np.nonzero(st == LAST)[0]
    if ended.size:
      trainer.reset(ended)
    if ev is not None:
      if t % 10 == 0:
        ev.network_params = agent.learner
      k, st, rw, dc, lv = ev_script[t]
      ev.step(ev_frames[k], st, rw, dc, lv)
      ended = np.nonzero(st == LAST)[0]
      if ended.size:
        ev.reset(ended)
  torch.cuda.synchronize()
  assert trainer.learn_steps > 0
  return actions, agent.get_state(), agent.learner.counters.cpu().numpy()


@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_training_is_isolated_from_evaluation_on_a_second_stream(kind):
  """Online and target parameters, optimizer state, replay contents and sum tree, the device counters and the trainer's
  actions are bit-identical with and without evaluator ticks interleaved on a second CUDA stream."""
  alone = _train_run(kind, interleave=False)
  beside = _train_run(kind, interleave=True)
  _assert_same(alone[0], beside[0], 'actions')
  _assert_same(alone[1], beside[1], 'agent')
  np.testing.assert_array_equal(alone[2], beside[2])


# -- 5: overlap changes nothing ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind', ['dqn', 'rainbow'])
def test_overlapped_evaluation_gives_the_same_rows(kind):
  sys.path.insert(0, os.path.join(ROOT, 'tools'))
  try:
    import run_synthetic
  finally:
    sys.path.pop(0)
  argv = ['--agent', kind, '--num_streams', '4', '--num_eval_streams', '6', '--num_iterations', '2',
          '--num_train_frames', '240', '--num_eval_frames', '120', '--replay_capacity', '1000',
          '--min_replay_capacity_fraction', '0.05', '--target_network_update_period', '64',
          '--max_frames_per_episode', '17']
  plain = run_synthetic.run(run_synthetic.parse_args(argv))
  overlapped = run_synthetic.run(run_synthetic.parse_args(argv + ['--overlap_eval']))
  assert len(plain) == len(overlapped) == 3
  rates = ('eval_frame_rate', 'train_frame_rate')
  for a, b in zip(plain, overlapped):
    assert list(a) == list(b)
    _assert_same({k: v for k, v in a.items() if k not in rates}, {k: v for k, v in b.items() if k not in rates}, 'row')
  assert plain[-1]['eval_num_episodes'] > 0


# -- 6: streams are independent ----------------------------------------------------------------------------------------
def test_streams_are_independent():
  """A greedy dqn evaluator on 16 streams acts per stream as 16 one-stream evaluators fed the same timesteps."""
  _, _, L, _, _ = _case('dqn', 84)
  E, ticks = 16, 40
  wide = _evaluator(L, E, eps=0.0)
  wide.network_params = L
  narrow = [_evaluator(L, 1, eps=0.0) for _ in range(E)]
  for ev in narrow:
    ev.network_params = L
  script, frames = _script(E, ticks, seed=5), _frames(E, seed=5)
  for t in range(ticks):
    k, st, rw, dc, lv = script[t]
    got = wide.step(frames[k], st, rw, dc, lv)
    for e, ev in enumerate(narrow):
      one = ev.step(frames[k][e:e + 1], st[e:e + 1], rw[e:e + 1], dc[e:e + 1], lv[e:e + 1])
      assert one[0] == got[e], (t, e)
    ended = np.nonzero(st == LAST)[0]
    if ended.size:
      wide.reset(ended)
      for e in ended:
        narrow[e].reset()
  np.testing.assert_array_equal(wide.num_episodes, [ev.num_episodes[0] for ev in narrow])


def test_one_stream_matches_run_loop_with_truncation():
  """E = 1 through the run driver's loop, truncated at max_frames_per_episode, gives run_loop(EpsilonGreedyActor)'s
  episode returns, lengths and count (SyntheticAtari's rewards do not depend on the actions)."""
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import processors
  from dqn_zoo_b200 import reporting
  sys.path.insert(0, os.path.join(ROOT, 'tools'))
  try:
    import run_synthetic
  finally:
    sys.path.pop(0)
  _, net, L, _, _ = _case('dqn', 84)
  M, frames = 13, 150
  actor = ag.EpsilonGreedyActor(processors.atari(device_observations=True), net, 0.01, rng_key=[0, 5])
  actor.network_params = L
  tracker = reporting.EpisodeTracker()
  tracker.reset()
  lengths, n = [], 0
  for _, ts, _, _ in itertools.islice(parts.run_loop(actor, run_synthetic.SyntheticAtari(seed=9), M), frames):
    tracker.step(None, ts, None, None)
    n += 1
    if ts.last():
      lengths.append(n)
      n = 0
  ev = _evaluator(L, 1, eps=0.01)
  ev.network_params = L
  loop = run_synthetic.StreamLoop(ev, [run_synthetic.SyntheticAtari(seed=9)], frames, M)
  got_lengths = []
  while not loop.done:
    loop.tick()
    if loop._timesteps[0].first():
      got_lengths.append(int(ev.episode_length[0]))
  assert loop._returns == tracker._returns
  assert got_lengths == lengths and len(lengths) >= 5
  assert int(ev.num_episodes[0]) == len(tracker._returns)


# -- 7: state round trip -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('kind,per_stream', [('dqn', False), ('rainbow', True), ('rainbow', False), ('iqn', False)])
def test_state_round_trip_continues_bit_for_bit(kind, per_stream):
  _, _, L, _, _ = _case(kind, 84)
  E, ticks, cut = 9, 36, 17
  script, frames = _script(E, ticks, seed=12), _frames(E, seed=12)

  def drive(ev, lo, hi):
    out = []
    for t in range(lo, hi):
      k, st, rw, dc, lv = script[t]
      a = ev.step(frames[k], st, rw, dc, lv)
      torch.cuda.synchronize()
      out.append((a, ev.actor.q.cpu().numpy().copy()))
      ended = np.nonzero(st == LAST)[0]
      if ended.size:
        ev.reset(ended)
    return out

  ev = _evaluator(L, E, eps=0.2, per_stream_noise=per_stream)
  ev.network_params = L.haiku_params()
  drive(ev, 0, cut)
  state = ev.get_state()
  rest = drive(ev, cut, ticks)
  fresh = _evaluator(L, E, eps=0.2, per_stream_noise=per_stream)
  fresh.set_state(state)
  again = drive(fresh, cut, ticks)
  _assert_same(rest, again, 'ticks')
  _assert_same(ev.episode_return, fresh.episode_return, 'returns')
  assert ev.actor.counter == fresh.actor.counter
  if kind != 'dqn':
    assert ev.actor.counter > state['counter'] > 0


# -- 8: errors ---------------------------------------------------------------------------------------------------------
def test_errors():
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  spec, net, L, _, _ = _case('dqn', 84)
  ev = _evaluator(L, 4)
  script, frames = _script(4, 2, seed=1), _frames(4, seed=1)
  k, st, rw, dc, lv = script[0]
  with pytest.raises(RuntimeError, match='network_params'):
    ev.step(frames[k], st, rw, dc, lv)
  ev.network_params = L
  with pytest.raises(ValueError):
    ev.step(frames[k][:3], st, rw, dc, lv)                     # wrong stream count
  with pytest.raises(ValueError):
    ev.step(frames[k][..., :2], st, rw, dc, lv)                # not RGB
  with pytest.raises(ValueError):
    ev.step(frames[k].float(), st, rw, dc, lv)                 # not uint8
  with pytest.raises(ValueError):
    ev.step(frames[k], st[:3], rw, dc, lv)
  ev.step(frames[k], st, rw, dc, lv)
  with pytest.raises(ValueError):
    ev.step(frames[k][:, :100], *script[1][1:])               # frame shape changed
  for E in (0, 1025):
    with pytest.raises(ValueError):
      _evaluator(L, E)
  _, _, Li, _, _ = _case('iqn', 84)
  with pytest.raises(ValueError):
    _evaluator(Li, 257)                                       # 257 * 64 > 16384
  with pytest.raises(ValueError):
    _evaluator(dl.NetworkSpec('iqn', 6), 257)
  with pytest.raises(ValueError):
    _evaluator(L, 4, per_stream_noise=True)
  # the acting context
  frozen = L.actor(4, frozen=True)
  obs = _obs(spec, 4, 0)
  with pytest.raises(RuntimeError):
    frozen.act(obs)
  q, a = torch.zeros((4, 6), device='cuda'), torch.zeros(4, dtype=torch.int32, device='cuda')
  with pytest.raises(ValueError):                             # the C ABI refuses too
    _lib.call('dz_actor_act', frozen._h, obs.data_ptr(), 0, 0, 0, 0, 0.0, q.data_ptr(), a.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
  live = L.actor(4)
  with pytest.raises(ValueError):
    live.load_params(L)
  with pytest.raises(ValueError):
    live.counter
  with pytest.raises(KeyError):
    frozen.load_params({'conv1/w': L.get_params()['conv1/w']})
  _, _, Lr, _, _ = _case('rainbow', 84)
  with pytest.raises(ValueError):
    frozen.load_params(Lr)
