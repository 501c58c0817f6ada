"""GPU: the acting context (`Learner.actor`, `dz_actor_*`) — batched acting for any number of streams over the learner's
live online parameters: q-values and actions against the float64 oracle, row independence of the stream count, the
learner's tensor-core conv3 features, the MMA paths, randomness, graph capture and BatchedEpsilonGreedyActor beyond the
learner's batch."""

import ctypes as C

import numpy as np
import pytest
import torch

from learner_parity import make_batch, make_case, obs_shape, random_noise, device_buffer
from oracle import learner_oracle as lo

pytestmark = pytest.mark.gpu

KINDS = ('dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn')
STREAMS = (1, 33, 100, 256)
ORACLE_CASES = ([(k, 84, E) for k in KINDS for E in STREAMS] +
                [(k, hw, E) for k in ('rainbow', 'dqn') for hw in (44, (84, 92)) for E in STREAMS])

_CASES = {}


@pytest.fixture(scope='module', autouse=True)
def _release():
  yield
  _CASES.clear()


def _key(hw):
  return hw if isinstance(hw, int) else tuple(hw)


def _case(kind, hw):
  """(spec, net, learner of batch 32, float64 oracle) per (kind, geometry), shared by the module's read-only tests."""
  k = (kind, _key(hw))
  if k not in _CASES:
    _CASES[k] = make_case(kind, 32, hw, seed=3)
  return _CASES[k]


def _obs(spec, E, seed):
  H, W = obs_shape(spec)
  return torch.as_tensor(np.random.RandomState(seed).randint(0, 256, (E, H, W, 4)).astype(np.uint8), device='cuda')


def _inputs(spec, net, E, rs, per_stream=False):
  """Act keyword arguments and the oracle's (taus, noise) for E streams: IQN a distinct tau row per stream; rainbow
  one shared apply, or one apply per stream (oracle: a list of per-row noise dicts)."""
  from dqn_zoo_b200 import learner as dl
  if spec.kind == 'iqn':
    taus = rs.uniform(size=(E, net.tau_samples_policy)).astype(np.float32)
    return {'taus': torch.as_tensor(taus, device='cuda')}, torch.tensor(taus), None
  if spec.kind == 'rainbow':
    if per_stream:
      raw = [random_noise(spec, rs) for _ in range(E)]
      flat = torch.as_tensor(dl.pack_noise(net, raw), device='cuda').view(E, -1)
      return {'stream_noise': flat}, None, [{k: torch.tensor(v) for k, v in one.items()} for one in raw]
    one = random_noise(spec, rs)
    return ({'noise': torch.as_tensor(dl.pack_noise(net, [one]), device='cuda')}, None,
            {k: torch.tensor(v) for k, v in one.items()})
  return {}, None, None


def _oracle_q(spec, params64, obs, taus_o, noise_o):
  x = torch.as_tensor(obs.cpu())
  if isinstance(noise_o, list):
    return np.stack([lo.apply_net(spec, params64, x[e:e + 1], torch.float64, noise=noise_o[e])['q_values'][0].numpy()
                     for e in range(x.shape[0])])
  return lo.apply_net(spec, params64, x, torch.float64, taus=taus_o, noise=noise_o)['q_values'].numpy()


def _act(actor, obs, **kw):
  a, q = actor.act(obs, **kw)
  torch.cuda.synchronize()
  return a.cpu().numpy().copy(), q.cpu().numpy().copy()


def _mma_path(actor, tag):
  from dqn_zoo_b200 import _lib
  path = C.c_int32()
  _lib.call('dz_test_actor_mma_path', actor._h, tag.encode(), C.byref(path))
  return path.value


def _actor_act3(actor):
  from dqn_zoo_b200 import _lib
  ptr, n = C.c_void_p(), C.c_int64()
  _lib.call('dz_test_actor_buffer', actor._h, b'act3', C.byref(ptr), C.byref(n))
  out = torch.empty(n.value, dtype=torch.float32, device='cuda')
  _lib.call('dz_test_copy', out.data_ptr(), ptr, 4 * n.value, torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  return out.cpu().numpy().reshape(actor.num_streams, -1)


def _check_oracle(spec, net, L, O, E, per_stream, seed):
  A = spec.num_actions
  actor = L.actor(E)
  rs = np.random.RandomState(seed)
  obs = _obs(spec, E, seed)
  kw, taus_o, noise_o = _inputs(spec, net, E, rs, per_stream)
  u = rs.uniform(size=(2, E)).astype(np.float32)
  eps = 0.4
  actions, q = _act(actor, obs, epsilon=eps, explore=torch.as_tensor(u, device='cuda'), **kw)
  want = _oracle_q(spec, O.online, obs, taus_o, noise_o)
  np.testing.assert_allclose(q, want, rtol=2e-5, atol=2e-6, err_msg='%s E=%d' % (spec.kind, E))
  for e in range(E):
    expect = min(int(u[1, e] * A), A - 1) if u[0, e] < eps else int(np.argmax(q[e]))
    assert actions[e] == expect, (e, actions[e], expect)
  greedy, q2 = _act(actor, obs, **kw)
  np.testing.assert_array_equal(q2, q)
  np.testing.assert_array_equal(greedy, np.argmax(q, axis=1))


@pytest.mark.parametrize('kind,hw,E', ORACLE_CASES)
def test_q_values_and_actions_match_the_oracle(kind, hw, E):
  """q-values against lo.apply_net in float64 at the acting bar of check_q_values; actions follow
  `u0 < eps ? floor(u1 * A) : first argmax`, greedy acting is the argmax.  Rainbow with one shared apply and with one
  apply per stream."""
  spec, net, L, O, _ = _case(kind, hw)
  _check_oracle(spec, net, L, O, E, False, 11 + E)
  if kind == 'rainbow':
    _check_oracle(spec, net, L, O, E, True, 12 + E)


@pytest.mark.parametrize('kind,per_stream', [('dqn', False), ('c51', False), ('rainbow', False), ('rainbow', True)])
def test_row_results_do_not_depend_on_the_stream_count(kind, per_stream):
  """Row e of a 256-stream actor equals a 1-stream actor on obs[e] with the same noise apply, bit for bit: the fc
  split-K counts and row chunks depend on the geometry only, and the fp32 heads never split K in an actor."""
  spec, net, L, _, _ = _case(kind, 84)
  E = 256
  big, one = L.actor(E), L.actor(1)
  rs = np.random.RandomState(21)
  obs = _obs(spec, E, 21)
  kw, _, _ = _inputs(spec, net, E, rs, per_stream)
  _, q = _act(big, obs, **kw)
  for e in (0, 1, 31, 32, 63, 64, 65, 127, 128, 200, 255):
    kw1 = {k: (v[e:e + 1] if k == 'stream_noise' else v) for k, v in kw.items()}
    _, q1 = _act(one, obs[e:e + 1], **kw1)
    np.testing.assert_array_equal(q1[0], q[e], err_msg='row %d' % e)


@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_conv3_features_equal_the_learners_tensor_core_pass(kind):
  """The actor's conv3 output on the learner's 32 observations equals the learner's pass-0 conv3 output bit for bit
  (same kernels, same reduction order); 33 streams, so conv3 pairs an odd image count."""
  spec, net, L, _, rs = make_case(kind, 32, 84, seed=4)
  arrs, _, w, _, taus_flat, _, noise_flat = make_batch(spec, net, 32, rs)
  s_tm1 = torch.as_tensor(arrs[0], device='cuda')
  obs = torch.cat([s_tm1, _obs(spec, 1, 5)])
  actor = L.actor(33)
  kw, _, _ = _inputs(spec, net, 33, rs)
  _act(actor, obs, **kw)
  got = _actor_act3(actor)
  L.update(*arrs, weights=w, taus=taus_flat, noise=noise_flat, apply_update=False)
  torch.cuda.synchronize()
  want = device_buffer(L, 'act3').numpy().reshape(32, -1)
  np.testing.assert_array_equal(got[:32], want)


@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_tensor_core_paths(kind):
  spec, net, L, O, _ = _case(kind, 84)
  actor = L.actor(100)
  for tag in ('conv1_fwd', 'conv2_fwd', 'conv3_fwd'):
    assert _mma_path(actor, tag) == 2, tag      # wgmma
  if kind != 'iqn':
    fc = 'noisy1_fwd' if kind == 'rainbow' else 'fc1_fwd'
    assert _mma_path(actor, fc) in (1, 2)       # umma_fc_kernel (mma.sync) or wgmma: on the tensor cores
  for tag in ('conv3_dgrad', 'fc1_dgrad', 'conv2_wgrad'):
    with pytest.raises(ValueError):             # a forward-only plan
      _mma_path(actor, tag)


def test_fma_fallback_geometry():
  """84x88 is outside the tensor-core path (odd conv1 width): the actor runs its torso on the fp32-FMA kernels and
  still matches the oracle."""
  spec, net, L, O, _ = _case('dqn', (84, 88))
  actor = L.actor(40)
  with pytest.raises(ValueError):
    _mma_path(actor, 'conv1_fwd')
  _check_oracle(spec, net, L, O, 40, False, 3)


@pytest.mark.parametrize('kind', ['dqn', 'rainbow'])
def test_act_reads_the_learners_live_parameters(kind):
  """An actor created before a learner step acts on the step's new online parameters (read in place)."""
  spec, net, L, O, rs = make_case(kind, 32, 84, seed=6)
  actor = L.actor(64)
  arrs, _, w, _, taus_flat, _, noise_flat = make_batch(spec, net, 32, rs)
  before = L.online.clone()
  L.update(*arrs, weights=w, taus=taus_flat, noise=noise_flat, apply_update=True)
  torch.cuda.synchronize()
  assert not torch.equal(before, L.online)
  params64 = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params().items()}
  obs = _obs(spec, 64, 7)
  kw, taus_o, noise_o = _inputs(spec, net, 64, rs)
  _, q = _act(actor, obs, **kw)
  np.testing.assert_allclose(q, _oracle_q(spec, params64, obs, taus_o, noise_o), rtol=2e-5, atol=2e-6)


@pytest.mark.parametrize('kind,E', [('iqn', 7), ('iqn', 100), ('rainbow', 32), ('rainbow', 100)])
def test_randomness_is_the_learners_generator(kind, E):
  """One counter step per call; for the first min(E, batch) streams the draws equal generate_randomness /
  generate_stream_noise at the same seed and counter."""
  spec, net, L, _, _ = _case(kind, 84)
  actor = L.actor(E)
  k = min(E, L.batch_size)
  modes = (False, True) if kind == 'rainbow' else (False,)
  for per_stream in modes:
    ctr = L.counters.clone()
    got = actor.generate_randomness(41, per_stream=per_stream).clone()
    torch.cuda.synchronize()
    assert int(L.counters[1]) == int(ctr[1]) + 1
    L.counters.copy_(ctr)
    if kind == 'iqn':
      L.generate_randomness(41)
      torch.cuda.synchronize()
      n = k * net.tau_samples_policy
      np.testing.assert_array_equal(got.reshape(-1)[:n].cpu().numpy(), L.taus[:n].cpu().numpy())
    elif per_stream:
      want = L.generate_stream_noise(41, k).clone()
      torch.cuda.synchronize()
      np.testing.assert_array_equal(got[:k].cpu().numpy(), want.cpu().numpy())
    else:
      L.generate_randomness(41)
      torch.cuda.synchronize()
      np.testing.assert_array_equal(got.cpu().numpy(), L.noise[:L.noise_stride].cpu().numpy())
    L.counters.copy_(ctr)


@pytest.mark.parametrize('kind,per_stream', [('dqn', False), ('iqn', False), ('rainbow', False), ('rainbow', True)])
def test_tick_replays_from_a_cuda_graph(kind, per_stream):
  """An actor tick (randomness + act) captured in a CUDA graph and replayed gives the eager tick's bits at the same
  counter."""
  spec, net, L, _, _ = _case(kind, 84)
  E = 100
  actor = L.actor(E)
  obs = _obs(spec, E, 31)
  explore = torch.as_tensor(np.random.RandomState(32).uniform(size=(2, E)).astype(np.float32), device='cuda')

  def tick():
    kw = {}
    if kind in ('iqn', 'rainbow'):
      r = actor.generate_randomness(53, per_stream=per_stream)
      kw = {'taus': r} if kind == 'iqn' else ({'stream_noise': r} if per_stream else {'noise': r})
    return actor.act(obs, epsilon=0.3, explore=explore, **kw)

  ctr = L.counters.clone()
  a, q = tick()
  torch.cuda.synchronize()
  a0, q0 = a.cpu().numpy().copy(), q.cpu().numpy().copy()
  s = torch.cuda.Stream()
  s.wait_stream(torch.cuda.current_stream())
  g = torch.cuda.CUDAGraph()
  with torch.cuda.stream(s):
    with torch.cuda.graph(g, stream=s):
      a, q = tick()
  torch.cuda.current_stream().wait_stream(s)
  L.counters.copy_(ctr)
  actor.q.zero_()
  g.replay()
  torch.cuda.synchronize()
  np.testing.assert_array_equal(q.cpu().numpy(), q0)
  np.testing.assert_array_equal(a.cpu().numpy(), a0)
  assert int(L.counters[1]) == int(ctr[1]) + (1 if kind in ('iqn', 'rainbow') else 0)


@pytest.mark.parametrize('kind,per_stream', [('dqn', False), ('iqn', False), ('rainbow', False), ('rainbow', True)])
def test_batched_epsilon_greedy_actor_beyond_the_learner_batch(kind, per_stream):
  """100 streams on a batch-32 learner: the tick acts through an Actor and returns its actions (one host array)."""
  from dqn_zoo_b200 import agent as agent_lib
  spec, net, L, _, _ = _case(kind, 84)
  E = 100
  obs = _obs(spec, E, 61)
  bega = agent_lib.BatchedEpsilonGreedyActor(L, E, exploration_epsilon=0.3, rng_key=[0, 7], per_stream_noise=per_stream)
  ctr = L.counters.clone()
  got = bega.step(obs)
  assert got.shape == (E,) and got.dtype == np.int32
  L.counters.copy_(ctr)
  ref = L.actor(E)
  u = torch.as_tensor(np.random.RandomState(7).uniform(size=(2, E)).astype(np.float32), device='cuda')
  kw = {}
  if kind in ('iqn', 'rainbow'):
    r = ref.generate_randomness(7, per_stream=per_stream)
    kw = {'taus': r} if kind == 'iqn' else ({'stream_noise': r} if per_stream else {'noise': r})
  want, q = _act(ref, obs, epsilon=0.3, explore=u, **kw)
  np.testing.assert_array_equal(got, want)
  np.testing.assert_array_equal(bega.q_values.cpu().numpy(), q)
  if per_stream:
    assert len({row.tobytes() for row in q}) > E // 2     # the streams' own noise draws


def test_errors_raise_value_error():
  from dqn_zoo_b200 import agent as agent_lib
  spec, net, L, _, _ = _case('rainbow', 44)
  for E in (0, 1025):
    with pytest.raises(ValueError):
      L.actor(E)
    with pytest.raises(ValueError):
      agent_lib.BatchedEpsilonGreedyActor(L, E, exploration_epsilon=0.0, rng_key=[0, 1])
  _, _, I, _, _ = _case('iqn', 84)                    # 64 policy samples: at most 256 streams
  I.actor(256)
  with pytest.raises(ValueError):
    I.actor(257)
  actor = L.actor(40)
  obs = _obs(spec, 41, 1)
  noise = torch.zeros((41, L.noise_stride), dtype=torch.float32, device='cuda')
  with pytest.raises(ValueError):
    actor.act(obs, noise=noise[0])                    # 41 observations for 40 streams
  with pytest.raises(ValueError):
    actor.act(obs[:40], stream_noise=noise)           # one apply per stream
  with pytest.raises(ValueError):
    actor.act(obs[:40], stream_noise=noise[:40, :-4])
  with pytest.raises(ValueError):
    actor.act(obs[:40])                               # rainbow needs noise
  torch.cuda.synchronize()
