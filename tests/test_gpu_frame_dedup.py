"""GPU: the frame-deduplicated replay layout (`frame_dedup=True`, csrc/dz_frames.cu).

  * the golden scenarios and the replay contract pass unchanged with every replay constructed in the dedup layout;
  * random frame-stack streams (interleaved actors, static screens, the ring wrapped several times, host and device
    sources): the device plane table, refcounts and frames_in_use equal oracle/frame_pool_oracle.py exactly, and
    everything sampled or read back equals a transition-major replay fed the same stream;
  * agents on either layout with the same seed and contents: sampled ids, loss, priorities and parameters bit-identical;
  * get_state / set_state within and across layouts; the sticky pool-full flag; the 1M x 84x84x4 baseline geometry.
"""

import copy
import functools
import types

import numpy as np
import pytest
import torch

from oracle import frame_pool_oracle as fpo
from oracle import replay_oracle as ro
from oracle import cpu_reference
from oracle import scenarios
import replay_contract as rc

pytestmark = pytest.mark.gpu

STRUCT = (None, None, None, None, None)


@pytest.fixture(scope='module')
def dedup():
  """`dqn_zoo_b200.replay` with both replay classes constructed in the frame-deduplicated layout.  The scenarios store
  iid random observations, which share no planes, so the pool is sized for 2 * C planes per transition, plus one row
  (an add references its planes before the evicted row releases its own) and plane 0, instead of the frame-stack
  default."""
  from dqn_zoo_b200 import replay as dr
  shim = types.SimpleNamespace(**{k: getattr(dr, k) for k in dir(dr) if not k.startswith('__')})

  def dedup_ctor(cls):
    @functools.wraps(cls)
    def make(capacity, *args, **kwargs):
      return cls(capacity, *args, frame_dedup=True, frame_capacity=2 * scenarios.OBS_SHAPE[2] * (capacity + 1) + 1, **kwargs)
    return make
  shim.TransitionReplay = dedup_ctor(dr.TransitionReplay)
  shim.PrioritizedTransitionReplay = dedup_ctor(dr.PrioritizedTransitionReplay)
  return shim


@pytest.mark.parametrize('name', list(scenarios.ALL))
def test_dedup_reproduces_reference_golden(dedup, name):
  rc.check_scenario(dedup, name, 'device')


@pytest.mark.parametrize('fn', rc.CONTRACT, ids=lambda f: f.__name__)
def test_dedup_contract(dedup, fn):
  fn(dedup)


def _stream(seed, n_step, obs_shape):
  rs = np.random.RandomState(seed)
  lengths = [[9, 30, 2, 14], [25, 1, 17], [6, 6, 40]]
  static = {(0, 1), (2, 2)}
  episodes = [[fpo.stacked_episode(rs, L, obs_shape, static=(k, j) in static) for j, L in enumerate(ls)]
              for k, ls in enumerate(lengths)]
  return fpo.interleave_episodes(rs, [ro.NStepTransitionAccumulator(n_step) for _ in lengths], episodes)


def _pool_state(rep):
  st = rep._store
  live = np.asarray(list(rep._live_ids), dtype=np.int64) % rep.capacity
  return st.planes.cpu().numpy()[live], st.refcount.cpu().numpy(), live


def _assert_pool_matches(rep, model):
  planes, ref, live = _pool_state(rep)
  np.testing.assert_array_equal(planes, model.pool.planes[live])
  np.testing.assert_array_equal(ref, model.pool.refcount)
  assert rep.frames_in_use == model.pool.frames_in_use
  ok, msg = rep.check_valid()
  assert ok, msg


@pytest.mark.parametrize('prioritized', [False, True])
@pytest.mark.parametrize('n_step', [1, 3])
def test_random_stacked_streams_match_oracle_and_transition_major(prioritized, n_step):
  from dqn_zoo_b200 import replay as dr
  obs_shape, cap = (8, 6, 4), 24
  trs = _stream(11 + n_step, n_step, obs_shape)
  assert len(trs) > 5 * cap

  def make(dedup_layout):
    rs = np.random.RandomState(7)
    if prioritized:
      return dr.PrioritizedTransitionReplay(cap, dr.Transition(*STRUCT), 0.5, lambda t: 0.6, 0.1, True, rs,
                                            frame_dedup=dedup_layout)
    return dr.TransitionReplay(cap, dr.Transition(*STRUCT), rs, frame_dedup=dedup_layout)

  a, b = make(True), make(False)
  model = fpo.DedupReplayModel(cap, obs_shape, 2 * cap + 64)
  for k, tr in enumerate(trs):
    item = dr.Transition(*tr)
    if k % 2:   # device-resident sources (the processors.atari(device_observations=True) insert path)
      item = item._replace(s_tm1=torch.as_tensor(tr.s_tm1, device='cuda'), s_t=torch.as_tensor(tr.s_t, device='cuda'))
    if prioritized:
      a.add(item, priority=1.0 + k % 5)
      b.add(dr.Transition(*tr), priority=1.0 + k % 5)
    else:
      a.add(item)
      b.add(dr.Transition(*tr))
    model.add(tr.s_tm1, tr.s_t)
    if k % 17 == 16 or k == len(trs) - 1:
      _assert_pool_matches(a, model)
      got = a.sample(16)
      want = b.sample(16)
      for g, w in zip(got, want):
        if isinstance(g, tuple):
          for x, y in zip(g, w):
            np.testing.assert_array_equal(np.asarray(x), np.asarray(y))
        else:
          np.testing.assert_array_equal(g, w)
      if prioritized:
        a.update_priorities(got[1], np.linspace(0.5, 2.0, 16).astype(np.float32))
        b.update_priorities(want[1], np.linspace(0.5, 2.0, 16).astype(np.float32))
      ids = list(a.ids())[::5] if not prioritized else sorted(a._distribution.ids())[::5]
      for x, y in zip(a.get(ids), b.get(ids)):
        for u, v in zip(x, y):
          np.testing.assert_array_equal(np.asarray(u), np.asarray(v))
  # plane 0 and frames shared between streams: far fewer planes than 2 * C per transition
  assert a.frames_in_use < cap * 2 * obs_shape[2] // 2


def _agent(kind, rep, seed, graph, obs_shape):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  net = dl.NetworkSpec(kind, 6, obs_shape=obs_shape)
  common = dict(preprocessor=lambda ts: ts, sample_network_input=np.zeros(obs_shape, np.uint8), network=net,
                optimizer=None, transition_accumulator=dr.NStepTransitionAccumulator(3 if kind == 'rainbow' else 1),
                replay=rep, batch_size=32, min_replay_capacity_fraction=0.05, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=graph)
  eps = lambda t: 0.1
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common)
  if kind == 'c51':
    return ag.C51(support=np.linspace(-10, 10, 51), exploration_epsilon=eps, **common)
  if kind == 'qrdqn':
    return ag.QrDqn(quantiles=(np.arange(201) + 0.5) / 201, exploration_epsilon=eps, huber_param=1.0, **common)
  if kind == 'iqn':
    return ag.Iqn(exploration_epsilon=eps, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                  tau_samples_s_t=64, **common)
  return ag.AGENTS[kind](exploration_epsilon=eps, grad_error_bound=1.0 / 32, **common)


@pytest.mark.parametrize('graph', [False, True])
@pytest.mark.parametrize('kind', ['dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn'])
def test_agents_are_bit_identical_on_both_layouts(kind, graph):
  from dqn_zoo_b200 import replay as dr
  obs_shape, cap, seed = (44, 44, 4), 512, 9
  prioritized = kind in ('prioritized', 'rainbow')
  runs = []
  for dedup_layout in (False, True):
    rs = np.random.RandomState(seed)
    if prioritized:
      rep = dr.PrioritizedTransitionReplay(cap, dr.Transition(*STRUCT), 0.5 if kind == 'rainbow' else 0.6,
                                           lambda t: 0.5, 1e-3, True, rs, frame_dedup=dedup_layout)
    else:
      rep = dr.TransitionReplay(cap, dr.Transition(*STRUCT), rs, frame_dedup=dedup_layout)
    dr.bulk_fill_synthetic_stacked(rep, obs_shape, seed, 6, episode_len=37)
    agent = _agent(kind, rep, seed, graph, obs_shape)
    L = agent.learner
    trace = []
    for _ in range(6):
      agent.learn()
      trace.append((L.sampled_ids.cpu().numpy().copy(), L.loss.cpu().numpy().copy(),
                    L.priorities.cpu().numpy().copy(), L.per_example.cpu().numpy().copy()))
    agent.check_device_flags()
    runs.append((trace, L.online.cpu().numpy(), rep))
  (ta, pa, ra), (tb, pb, rb) = runs
  for step, (x, y) in enumerate(zip(ta, tb)):
    for u, v in zip(x, y):
      np.testing.assert_array_equal(u, v, err_msg='%s step %d' % (kind, step))
  np.testing.assert_array_equal(pa, pb)
  if prioritized:
    np.testing.assert_array_equal(ra.get_state()['distribution']['sum_tree']['storage'],
                                  rb.get_state()['distribution']['sum_tree']['storage'])


def test_stacked_fill_matches_oracle_rows_and_sequential_adds():
  from dqn_zoo_b200 import replay as dr
  obs_shape, cap, L = (8, 6, 4), 50, 7
  filled = dr.TransitionReplay(cap, dr.Transition(*STRUCT), np.random.RandomState(1), frame_dedup=True)
  dr.bulk_fill_synthetic_stacked(filled, obs_shape, 3, 6, episode_len=L)
  tm = dr.TransitionReplay(cap, dr.Transition(*STRUCT), np.random.RandomState(1))
  dr.bulk_fill_synthetic_stacked(tm, obs_shape, 3, 6, episode_len=L)
  obs, a, r, d = fpo.synthetic_stacked_rows(3, np.arange(cap), obs_shape, L, 6)
  added = dr.TransitionReplay(cap, dr.Transition(*STRUCT), np.random.RandomState(1), frame_dedup=True)
  model = fpo.DedupReplayModel(cap, obs_shape, 2 * cap + 64)
  for i in range(cap):
    s0, s1 = obs[i, 0].reshape(obs_shape), obs[i, 1].reshape(obs_shape)
    added.add(dr.Transition(s0, int(a[i]), float(r[i]), float(d[i]), s1))
    model.add(s0, s1)
  for rep in (filled, tm, added):
    got = rep.get(range(cap))
    np.testing.assert_array_equal(np.stack([t.s_tm1 for t in got]).reshape(cap, -1), obs[:, 0])
    np.testing.assert_array_equal(np.stack([t.s_t for t in got]).reshape(cap, -1), obs[:, 1])
    np.testing.assert_array_equal(np.array([t.a_tm1 for t in got]), a)
    np.testing.assert_array_equal(np.array([t.r_t for t in got]), r)
  _assert_pool_matches(filled, model)
  _assert_pool_matches(added, model)
  assert filled.frames_in_use == cap + 8 + 1
  # the filled pool keeps working as adds evict rows
  for i in range(30):
    o = np.full(obs_shape, i, dtype=np.uint8)
    filled.add(dr.Transition(o, 0, 0.0, 1.0, o + 1))
    model.add(o, o + 1)
  _assert_pool_matches(filled, model)
  with pytest.raises(ValueError):
    dr.bulk_fill_synthetic(dr.TransitionReplay(4, dr.Transition(*STRUCT), np.random.RandomState(1), frame_dedup=True),
                           obs_shape, 1, 6)


def test_state_roundtrip_within_and_across_layouts():
  from dqn_zoo_b200 import replay as dr
  obs_shape, cap = (8, 6, 4), 20
  trs = _stream(5, 1, obs_shape)[:47]

  def make(dedup_layout, seed=2):
    return dr.PrioritizedTransitionReplay(cap, dr.Transition(*STRUCT), 0.5, lambda t: 0.6, 0.2, True,
                                          np.random.RandomState(seed), frame_dedup=dedup_layout)
  src = {True: make(True), False: make(False)}
  for k, tr in enumerate(trs):
    for rep in src.values():
      rep.add(dr.Transition(*tr), priority=1.0 + k % 3)
  restored_model = fpo.DedupReplayModel(cap, obs_shape, 2 * cap + 64)
  for i, item in sorted(src[False].get_state()['storage'], key=lambda x: x[0]):
    restored_model.pool.add(i % cap, item.s_tm1, item.s_t, release_row=False)
  restored_model.t = len(trs)
  for from_layout in (True, False):
    st = copy.deepcopy(src[from_layout].get_state())
    for to_layout in (True, False):
      dst = make(to_layout, seed=99)
      dst.set_state(copy.deepcopy(st))
      if to_layout:
        _assert_pool_matches(dst, restored_model)
      sa, sb = np.random.RandomState(4), np.random.RandomState(4)
      rc._rebind_rng(dst, sa)
      ref = make(False, seed=99)
      ref.set_state(copy.deepcopy(st))
      rc._rebind_rng(ref, sb)
      for k in range(25):
        tr = trs[k]
        dst.add(dr.Transition(*tr), priority=2.0)
        ref.add(dr.Transition(*tr), priority=2.0)
        ta, ia, wa = dst.sample(8)
        tb, ib, wb = ref.sample(8)
        np.testing.assert_array_equal(ia, ib)
        np.testing.assert_array_equal(wa, wb)
        np.testing.assert_array_equal(ta.s_tm1, tb.s_tm1)
        np.testing.assert_array_equal(ta.s_t, tb.s_t)
      ok, msg = dst.check_valid()
      assert ok, msg


def test_pool_exhaustion_is_a_sticky_data_error():
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import replay as dr
  obs_shape = (4, 4, 2)
  rs = np.random.RandomState(3)
  for prioritized in (False, True):
    if prioritized:
      rep = dr.PrioritizedTransitionReplay(8, dr.Transition(*STRUCT), 0.5, lambda t: 0.6, 0.1, True,
                                           np.random.RandomState(1), frame_dedup=True, frame_capacity=6)
    else:
      rep = dr.TransitionReplay(8, dr.Transition(*STRUCT), np.random.RandomState(1), frame_dedup=True, frame_capacity=6)
    for _ in range(3):
      item = dr.Transition(rs.randint(1, 256, obs_shape).astype(np.uint8), 0, 0.0, 1.0,
                           rs.randint(1, 256, obs_shape).astype(np.uint8))
      rep.add(item, priority=1.0) if prioritized else rep.add(item)
    assert rep.frames_in_use == 6
    for call in (lambda: rep.sample(4), lambda: rep.check_valid(), lambda: rep.get([0]), lambda: rep.get_state(),
                 lambda: ag.Dqn.check_device_flags(types.SimpleNamespace(_replay=rep, PRIORITIZED=prioritized))):
      with pytest.raises(RuntimeError, match='frame_capacity'):
        call()
  with pytest.raises(ValueError):
    dr.TransitionReplay(8, dr.Transition(*STRUCT), np.random.RandomState(1), frame_dedup=True).add(
        dr.Transition(np.zeros((4, 4), np.uint8), 0, 0.0, 1.0, np.zeros((4, 4), np.uint8)))
  with pytest.raises(ValueError):
    dr.TransitionReplay(8, dr.Transition(*STRUCT), np.random.RandomState(1), frame_dedup=True).add(
        dr.Transition(np.zeros(obs_shape, np.float32), 0, 0.0, 1.0, np.zeros(obs_shape, np.float32)))


def test_dedup_1m_at_the_baseline_geometry_84x84x4():
  """Capacity 1M of 84x84x4 frame stacks in about 14 GB: bytes of rows whose planes sit on both sides of every 2^32
  byte offset of the pool, and 40 fused rainbow steps (ids / weights vs the oracle, sum tree bit-exact)."""
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  free, _ = torch.cuda.mem_get_info()
  if free < 16 * (1 << 30):
    pytest.skip('needs 16 GB of free HBM')
  CAP, obs_shape, seed, L = 1000000, (84, 84, 4), 4, 1000
  beta = lambda t: 0.5
  rep = dr.PrioritizedTransitionReplay(CAP, dr.Transition(*STRUCT), 0.5, beta, 1e-3, True, np.random.RandomState(seed),
                                       frame_dedup=True)
  dr.bulk_fill_synthetic_stacked(rep, obs_shape, seed, 6, episode_len=L)
  assert rep.size == CAP and rep.storage_bytes < 15 * (1 << 30)
  assert rep.frames_in_use == CAP + CAP // L + 1
  stride = rep._store.frame_stride
  rows = [0, 1, CAP - 1]
  k = 1
  while k * (1 << 32) < (CAP + CAP // L + 1) * stride:
    plane = (k * (1 << 32)) // stride             # the plane holding byte k * 2^32 and its neighbours
    for p in (plane - 1, plane, plane + 1):
      e, f = divmod(p - 1, L + 1)
      rows += [e * L + max(f - 1, 0), e * L + min(f, L - 1)]
    k += 1
  rows = np.array(sorted(set(i for i in rows if 0 <= i < CAP)), dtype=np.int64)
  assert k >= 2 and len(rows) >= 6
  got = rep.get(rows)
  obs, a, r, d = fpo.synthetic_stacked_rows(seed, rows, obs_shape, L, 6)
  np.testing.assert_array_equal(np.stack([t.s_tm1 for t in got]).reshape(len(rows), -1), obs[:, 0])
  np.testing.assert_array_equal(np.stack([t.s_t for t in got]).reshape(len(rows), -1), obs[:, 1])
  np.testing.assert_array_equal(np.array([t.a_tm1 for t in got]), a)
  orep, _ = cpu_reference.build_replay('rainbow', CAP, 32, seed, obs_shape=obs_shape)
  orep._beta = beta
  net = dl.NetworkSpec('rainbow', 6, obs_shape=obs_shape)
  agent = ag.Rainbow(preprocessor=lambda ts: ts, sample_network_input=np.zeros(obs_shape, np.uint8), network=net,
                     support=np.linspace(-10, 10, 51), optimizer=None,
                     transition_accumulator=dr.NStepTransitionAccumulator(3), replay=rep, batch_size=32,
                     min_replay_capacity_fraction=0.02, learn_period=16, target_network_update_period=32000,
                     rng_key=[0, seed], use_cuda_graph=True)
  Lr = agent.learner
  for step in range(40):
    agent.learn()
    ids_o, _, w = orep.sample_ids(32)
    pri = Lr.priorities.cpu().numpy()
    np.testing.assert_array_equal(Lr.sampled_ids.cpu().numpy(), ids_o, err_msg='step %d' % step)
    np.testing.assert_allclose(Lr.sampled_weights.cpu().numpy(), w, rtol=1e-14)
    assert np.isfinite(pri).all()
    orep.update_priorities(ids_o, pri)
  agent.check_device_flags()
  tr, ids2, _ = rep.sample(32)
  obs2, _, _, _ = fpo.synthetic_stacked_rows(seed, ids2, obs_shape, L, 6)
  np.testing.assert_array_equal(tr.s_tm1.reshape(32, -1), obs2[:, 0])
  np.testing.assert_array_equal(tr.s_t.reshape(32, -1), obs2[:, 1])
  tree = rep._distribution._sum_tree.get_state()['storage']
  np.testing.assert_array_equal(tree, orep.get_state()['distribution']['sum_tree']['storage'])
