"""GPU: rainbow batched acting with one noise apply per actor stream (`dz_learner_act_batch` with noise_ld = stride,
`Learner.act_batch(..., stream_noise=...)`, `Learner.generate_stream_noise`, `BatchedEpsilonGreedyActor(per_stream_noise=True)`)
against the shared-noise mode, the single-observation path and the float64 oracle."""

import numpy as np
import pytest
import torch

from oracle import learner_oracle as lo

pytestmark = pytest.mark.gpu

A = 6
ATOMS = {84: 51, 44: 21}          # 44x44: a ragged head (6 x 21 = 126 outputs) and a 256-wide torso
CASES = [(hw, E) for hw in (84, 44) for E in (1, 7, 32)]


_LEARNERS = {}


@pytest.fixture(scope='module', autouse=True)
def _release_learners():
  yield
  _LEARNERS.clear()


def _case(hw, batch=32):
  """(oracle spec, network spec, learner, params), one learner per geometry for the whole module."""
  if (hw, batch) not in _LEARNERS:
    from dqn_zoo_b200 import learner as dl
    spec = lo.NetSpec('rainbow', A, num_atoms=ATOMS[hw], obs_hw=hw)
    net = dl.NetworkSpec('rainbow', A, num_atoms=ATOMS[hw], obs_shape=(hw, hw, 4))
    params = lo.init_params(spec, 3)
    L = dl.Learner(net, batch_size=batch)
    L.set_params(params, also_target=True)
    _LEARNERS[hw, batch] = (spec, net, L, params)
  return _LEARNERS[hw, batch]


def _obs(hw, E, seed):
  rs = np.random.RandomState(seed)
  return torch.as_tensor(rs.randint(0, 256, size=(E, hw, hw, 4)).astype(np.uint8), device='cuda')


def _act(L, obs, **kw):
  actions, q = L.act_batch(obs, **kw)
  torch.cuda.synchronize()
  return actions.cpu().numpy().copy(), q.cpu().numpy().copy()


def _unpack(net, row):
  """One apply of the device layout -> {name: float64 tensor} for the oracle."""
  from dqn_zoo_b200 import learner as dl
  out, pos = {}, 0
  for name, n in dl.noise_vector_sizes(net):
    out[name] = torch.tensor(row[pos:pos + n].astype(np.float64))
    pos += (n + 3) // 4 * 4
  return out


@pytest.mark.parametrize('hw,E,batch', [(hw, E, 32) for hw, E in CASES] + [(44, 40, 40)])
def test_same_apply_on_every_stream_equals_shared_mode_bit_for_bit(hw, E, batch):
  """Every row carrying one apply: the per-row kernels must reproduce the shared-noise forward exactly (same weight
  formation order, BK chunks and split-K boundaries; E > 32 takes the unsplit path with the fused epilogue)."""
  _, _, L, _ = _case(hw, batch)
  L.generate_randomness(17)
  torch.cuda.synchronize()
  apply = L.noise[:L.noise_stride].clone()
  obs = _obs(hw, E, 1)
  explore = torch.as_tensor(np.random.RandomState(2).uniform(size=(2, E)).astype(np.float32), device='cuda')
  for eps in (0.0, 0.3):
    a_shared, q_shared = _act(L, obs, epsilon=eps, explore=explore, noise=apply)
    a_rows, q_rows = _act(L, obs, epsilon=eps, explore=explore, stream_noise=apply[None, :].repeat(E, 1))
    np.testing.assert_array_equal(q_rows, q_shared)
    np.testing.assert_array_equal(a_rows, a_shared)


@pytest.mark.parametrize('hw,E', CASES)
def test_each_stream_equals_its_own_single_decision_and_the_oracle(hw, E):
  """E distinct applies: row e is `q_values(obs[e], noise=apply e)`, the action follows the documented epsilon rule
  (first argmax when greedy), and the float64 oracle's forward with stream e's noise agrees at the tolerance of
  test_q_values_match_oracle_forward.  A q-value is an expectation over the +-vmax support and often near zero, so its
  fp32 error is absolute rather than relative (the norm of the error over the [E, A] block is 1.0-1.2e-5 of the
  block's norm at 84x84)."""
  spec, net, L, params = _case(hw)
  noise = L.generate_stream_noise(23, E).clone()
  obs = _obs(hw, E, 4)
  u = np.random.RandomState(5).uniform(size=(2, E)).astype(np.float32)
  eps = 0.4
  actions, q = _act(L, obs, epsilon=eps, explore=torch.as_tensor(u, device='cuda'), stream_noise=noise)
  noise_np = noise.cpu().numpy()
  online64 = {k: torch.tensor(v, dtype=torch.float64) for k, v in params.items()}
  want = np.zeros((E, A))
  for e in range(E):
    q1 = L.q_values(obs[e], noise=noise[e]).cpu().numpy()
    np.testing.assert_allclose(q[e], q1, rtol=2e-6, atol=1e-6)
    expect = min(int(u[1, e] * A), A - 1) if u[0, e] < eps else int(np.argmax(q[e]))
    assert actions[e] == expect, (e, actions[e], expect)
    want[e] = lo.apply_net(spec, online64, torch.as_tensor(obs[e:e + 1].cpu()), torch.float64,
                           noise=_unpack(net, noise_np[e]))['q_values'][0].numpy()
  np.testing.assert_allclose(q, want, rtol=2e-5, atol=2e-6)
  greedy, _ = _act(L, obs, stream_noise=noise)
  np.testing.assert_array_equal(greedy, np.argmax(q, axis=1))


@pytest.mark.parametrize('hw,E', CASES)
def test_generated_applies(hw, E):
  """Distinct, finite, |eps| <= sqrt(2); reproducible from (seed, counter); one counter step per call; the first
  min(E, 3) applies are what generate_randomness writes for the same seed and counter."""
  _, _, L, _ = _case(hw)
  S = L.noise_stride
  ctr = L.counters.clone()
  block = L.generate_stream_noise(31, E).clone()
  torch.cuda.synchronize()
  assert tuple(block.shape) == (E, S)
  assert int(L.counters[1]) == int(ctr[1]) + 1
  b = block.cpu().numpy()
  assert np.all(np.isfinite(b)) and np.abs(b).max() <= np.sqrt(2.0)
  for e in range(E):
    for f in range(e):
      assert np.any(b[e] != b[f]), (e, f)
  L.counters.copy_(ctr)
  again = L.generate_stream_noise(31, E).clone()
  torch.cuda.synchronize()
  np.testing.assert_array_equal(again.cpu().numpy(), b)
  L.counters.copy_(ctr)
  L.generate_randomness(31)
  torch.cuda.synchronize()
  k = min(E, 3)
  np.testing.assert_array_equal(b[:k].reshape(-1), L.noise[:k * S].cpu().numpy())
  other = L.generate_stream_noise(32, E).cpu().numpy()
  assert np.any(other != b)


def test_actor_with_per_stream_noise_explores_each_stream_independently():
  from dqn_zoo_b200 import agent as agent_lib
  _, _, L, _ = _case(84)
  obs = _obs(84, 1, 8).repeat(32, 1, 1, 1)        # every stream sees the same observation
  actor = agent_lib.BatchedEpsilonGreedyActor(L, 32, exploration_epsilon=0.0, rng_key=[0, 9], per_stream_noise=True)
  a = actor.step(obs)
  q = actor.q_values.cpu().numpy()
  assert a.shape == (32,) and a.dtype == np.int32
  np.testing.assert_array_equal(a, np.argmax(q, axis=1))
  assert len({row.tobytes() for row in q}) == 32    # each stream's own noise draw
  a2 = actor.step(obs)                              # a new draw every tick
  assert not np.array_equal(actor.q_values.cpu().numpy(), q)
  assert a2.shape == (32,)
  shared = agent_lib.BatchedEpsilonGreedyActor(L, 32, exploration_epsilon=0.0, rng_key=[0, 9])
  shared.step(obs)
  qs = shared.q_values.cpu().numpy()
  assert all(np.array_equal(row, qs[0]) for row in qs)   # one draw for the tick: 32 identical rows
  eps_actor = agent_lib.BatchedEpsilonGreedyActor(L, 32, exploration_epsilon=0.5, rng_key=[0, 4], per_stream_noise=True)
  a3 = eps_actor.step(obs)
  assert a3.min() >= 0 and a3.max() < A


def test_per_stream_errors_raise_value_error_through_act_batch():
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import agent as agent_lib
  from dqn_zoo_b200 import learner as dl
  _, _, L, _ = _case(44)
  B, S = L.batch_size, L.noise_stride
  obs = _obs(44, B + 1, 3)
  noise = torch.zeros((B + 1, S), dtype=torch.float32, device='cuda')
  q = torch.zeros((B + 1, A), dtype=torch.float32, device='cuda')
  act = torch.zeros(B + 1, dtype=torch.int32, device='cuda')
  stream = torch.cuda.current_stream().cuda_stream

  def call(h, E, noise_ptr, noise_ld=S, actions=act.data_ptr()):
    _lib.call('dz_learner_act_batch', h, obs.data_ptr(), E, 0, noise_ptr, noise_ld, 0, 0.0, q.data_ptr(), actions, stream)

  call(L._h, 3, noise.data_ptr())                  # valid call for reference
  call(L._h, 3, noise.data_ptr(), actions=0)       # q-values only
  for E in (0, B + 1):
    with pytest.raises(ValueError):
      call(L._h, E, noise.data_ptr())
    with pytest.raises(ValueError):
      _lib.call('dz_learner_generate_stream_noise', L._h, 1, E, noise.data_ptr(), stream)
  with pytest.raises(ValueError):
    call(L._h, 3, 0)
  with pytest.raises(ValueError):
    call(L._h, 3, noise.data_ptr(), noise_ld=S + 4)   # neither one shared apply nor one per stream
  with pytest.raises(ValueError):
    _lib.call('dz_learner_generate_stream_noise', L._h, 1, 3, 0, stream)
  with pytest.raises(ValueError):
    L.act_batch(obs[:3], stream_noise=noise[:2])   # one apply per stream
  with pytest.raises(ValueError):
    L.act_batch(obs[:3], stream_noise=noise[:3, :S - 4])
  D = dl.Learner(dl.NetworkSpec('dqn', A, obs_shape=(44, 44, 4)), batch_size=8)
  with pytest.raises(ValueError):
    call(D._h, 3, noise.data_ptr())
  with pytest.raises(ValueError):
    D.generate_stream_noise(1, 3)
  with pytest.raises(ValueError):
    agent_lib.BatchedEpsilonGreedyActor(D, 4, exploration_epsilon=0.0, rng_key=[0, 1], per_stream_noise=True)
  torch.cuda.synchronize()
