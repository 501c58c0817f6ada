"""GPU: `add_batch` on both replay classes and both storage layouts (csrc/dz_replay.cu, csrc/dz_frames.cu) equals the
same transitions added one `add` at a time: device rows and scalars, the plane table, refcounts, the free stack in
order, the hash table's live set, frames_in_use, the sum tree, the id/index mirrors, ids(), and sample() / get()
under equal RandomStates.  Also: adversarial frame-pool batches, the pool running out mid-batch, the PER priority
forms and their validation, row offsets above 2**32, and the end-to-end many-stream insert path."""

import gc

import numpy as np
import pytest
import torch

from oracle import frame_pool_oracle as fpo
from oracle import learner_oracle as lo
from oracle import replay_oracle as ro

pytestmark = pytest.mark.gpu

STRUCT = (None, None, None, None, None)


def _make(prioritized, dedup, cap, seed=7, frame_capacity=None, alpha=0.5):
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  kw = dict(frame_dedup=dedup, frame_capacity=frame_capacity)
  if prioritized:
    return dr.PrioritizedTransitionReplay(cap, dr.Transition(*STRUCT), alpha, lambda t: 0.6, 0.1, True, rs, **kw)
  return dr.TransitionReplay(cap, dr.Transition(*STRUCT), rs, **kw)


def _table_live_set(st):
  """The plane ids in the hash table; asserts each is found by probing from its hash."""
  table = st.table.cpu().numpy()
  hashes = st.hashes.cpu().numpy().view(np.uint64)
  mask = len(table) - 1
  ids = table[table >= 0]
  for pid in ids:
    t = int(hashes[pid] & np.uint64(mask))
    while table[t] != pid:
      assert table[t] >= 0, 'plane %d is not reachable from its hash' % pid
      t = (t + 1) & mask
  return sorted(ids.tolist())


def _state(rep):
  st = rep._store
  rows = torch.as_tensor(np.asarray(list(rep._live_ids), np.int64) % rep.capacity, device='cuda')   # written rows
  out = {'t': rep._t, 'ids': list(rep._live_ids), 'dist_ids': sorted(rep._distribution.ids()),
         'action': st.action[rows], 'reward': st.reward[rows], 'discount': st.discount[rows], 'flags': rep._flags()}
  dist = rep._distribution
  dist.flush()
  if hasattr(dist, '_sum_tree'):
    host = dist.get_state()
    out.update(tree=dist._sum_tree.device_nodes, live=dist._live_dev.t[:dist.size], id_at=dist._id_at_dev.t,
               host={k: v for k, v in host.items() if k != 'sum_tree'})
  else:
    out.update(mirror=dist.device_ids[:dist.size], host=dist.get_state())
  if hasattr(st, 'frames'):
    top = int(st.counters.item())
    ref = st.refcount.cpu().numpy()
    live = np.nonzero(ref)[0]
    out.update(planes=st.planes, refcount=st.refcount, free=st.free[:top], top=top, hashes=st.hashes[live],
               bytes=st.frames[live], table=_table_live_set(st), live_planes=live)
    assert out['table'] == live.tolist()
  else:
    out.update(obs=st.obs[rows])
  return out


def _assert_same(a, b):
  sa, sb = _state(a), _state(b)
  assert sa.keys() == sb.keys()
  for k in sa:
    x, y = sa[k], sb[k]
    if isinstance(x, torch.Tensor):
      assert torch.equal(x, y), k
    elif isinstance(x, np.ndarray):
      np.testing.assert_array_equal(x, y, err_msg=k)
    else:
      assert x == y, k


def _assert_reads_same(a, b, n=8):
  ga, gb = a.sample(n), b.sample(n)
  for x, y in zip(ga, gb):
    for u, v in zip(x if isinstance(x, tuple) else [x], y if isinstance(y, tuple) else [y]):
      np.testing.assert_array_equal(np.asarray(u), np.asarray(v))
  ids = list(a._live_ids)[::3]
  for x, y in zip(a.get(ids), b.get(ids)):
    for u, v in zip(x, y):
      np.testing.assert_array_equal(np.asarray(u), np.asarray(v))
  for r in (a, b):
    ok, msg = r.check_valid()
    assert ok, msg


def _stacked_stream(seed, obs_shape, n_step=3):
  rs = np.random.RandomState(seed)
  lengths = [[9, 30, 2, 14], [25, 1, 17], [6, 6, 40]]
  static = {(0, 1), (2, 2)}
  episodes = [[fpo.stacked_episode(rs, L, obs_shape, static=(k, j) in static) for j, L in enumerate(ls)]
              for k, ls in enumerate(lengths)]
  return fpo.interleave_episodes(rs, [ro.NStepTransitionAccumulator(n_step) for _ in lengths], episodes)


def _batch(trs, device):
  from dqn_zoo_b200 import replay as dr
  s_tm1, s_t = np.stack([t.s_tm1 for t in trs]), np.stack([t.s_t for t in trs])
  if device:
    s_tm1, s_t = torch.as_tensor(s_tm1, device='cuda'), torch.as_tensor(s_t, device='cuda')
  return dr.Transition(s_tm1, np.array([t.a_tm1 for t in trs]), np.array([t.r_t for t in trs], np.float64),
                       np.array([t.discount_t for t in trs], np.float64), s_t)


def _feed(a, b, trs, K, prioritized, device, model=None, check_every=1):
  from dqn_zoo_b200 import replay as dr
  for n, lo_ in enumerate(range(0, len(trs), K)):
    part = trs[lo_:lo_ + K]
    pri = 1.0 + np.arange(lo_, lo_ + len(part)) % 5
    if prioritized:
      a.add_batch(_batch(part, device), pri)
    else:
      a.add_batch(_batch(part, device))
    for tr, p in zip(part, pri):
      if prioritized:
        b.add(dr.Transition(*tr), priority=float(p))
      else:
        b.add(dr.Transition(*tr))
      if model is not None:
        model.add(tr.s_tm1, tr.s_t)
    if n % check_every == 0 or lo_ + K >= len(trs):
      _assert_same(a, b)
      if model is not None:
        live = np.asarray(list(a._live_ids), np.int64) % a.capacity
        np.testing.assert_array_equal(a._store.planes.cpu().numpy()[live], model.pool.planes[live])
        np.testing.assert_array_equal(a._store.refcount.cpu().numpy(), model.pool.refcount)
        assert a.frames_in_use == model.pool.frames_in_use


@pytest.mark.parametrize('K', [1, 7, 32, 24, 51])
@pytest.mark.parametrize('device', [False, True], ids=['host', 'device'])
@pytest.mark.parametrize('dedup', [False, True], ids=['rows', 'dedup'])
@pytest.mark.parametrize('prioritized', [False, True], ids=['uniform', 'per'])
def test_add_batch_equals_sequential_adds(prioritized, dedup, device, K):
  """K = 24 is the capacity, 51 = 2 * capacity + 3 (split into capacity-sized calls)."""
  obs_shape, cap = (8, 6, 4), 24
  trs = _stacked_stream(11, obs_shape)
  assert len(trs) > 5 * cap
  a, b = _make(prioritized, dedup, cap), _make(prioritized, dedup, cap)
  model = fpo.DedupReplayModel(cap, obs_shape, 2 * cap + 64) if dedup else None
  _feed(a, b, trs, K, prioritized, device, model, check_every=max(1, 24 // K))
  _assert_reads_same(a, b)


def _library_stream(rs, n, obs_shape, frames):
  """Transitions whose channels are drawn from a few planes (plane 0 among them): identical stacks, static screens and
  all-zero planes, planes freed by one add's eviction that reappear in a later add of the same batch, freed ids popped
  again for other bytes."""
  h, w, c = obs_shape
  lib = rs.randint(0, 256, size=(frames, h, w)).astype(np.uint8)
  lib[0] = 0
  out = []
  for _ in range(n):
    s_tm1, s_t = lib[rs.randint(0, frames, size=c)].transpose(1, 2, 0), lib[rs.randint(0, frames, size=c)].transpose(1, 2, 0)
    out.append(ro.Transition(np.ascontiguousarray(s_tm1), int(rs.randint(0, 6)), float(rs.randint(-1, 2)), 0.99,
                             np.ascontiguousarray(s_t)))
  return out


@pytest.mark.parametrize('K', [3, 6, 13])
@pytest.mark.parametrize('frames', [3, 9])
def test_adversarial_pool_batches(K, frames):
  obs_shape, cap = (4, 8, 2), 6
  rs = np.random.RandomState(K * 100 + frames)
  trs = _library_stream(rs, 120, obs_shape, frames)
  # several streams with identical stacks in one batch
  trs[20:28] = [trs[20]] * 8
  a, b = _make(True, True, cap), _make(True, True, cap)
  _feed(a, b, trs, K, True, K % 2 == 1, fpo.DedupReplayModel(cap, obs_shape, 2 * cap + 64))
  _assert_reads_same(a, b, 4)


def test_freed_plane_reappears_and_freed_id_is_reused_in_one_batch():
  obs_shape, cap = (4, 4, 1), 2
  rs = np.random.RandomState(3)
  f = [rs.randint(1, 256, size=obs_shape).astype(np.uint8) for _ in range(8)]
  tr = lambda x, y: ro.Transition(f[x], 0, 0.0, 0.99, f[y])
  first = [tr(0, 1), tr(2, 3)]
  # add 0 releases row 0 (the planes of frames 0 and 1 go back on the free stack); add 1 pops one of those ids for
  # frame 6 and brings frame 1's bytes back under another freed id
  batch = [tr(4, 5), tr(6, 1)]
  a, b = _make(False, True, cap), _make(False, True, cap)
  model = fpo.DedupReplayModel(cap, obs_shape, 2 * cap + 64)
  _feed(a, b, first, 2, False, False, model)
  _feed(a, b, batch, 2, False, False, model)
  _assert_reads_same(a, b, 2)


@pytest.mark.parametrize('prioritized', [False, True])
def test_pool_running_out_mid_batch(prioritized):
  obs_shape, cap = (4, 4, 2), 8
  rs = np.random.RandomState(5)
  trs = [ro.Transition(rs.randint(0, 256, size=obs_shape).astype(np.uint8), 1, 0.0, 0.99,
                       rs.randint(0, 256, size=obs_shape).astype(np.uint8)) for _ in range(6)]
  a = _make(prioritized, True, cap, frame_capacity=9)
  b = _make(prioritized, True, cap, frame_capacity=9)
  from dqn_zoo_b200 import replay as dr
  if prioritized:
    a.add_batch(_batch(trs, False), 1.0)
  else:
    a.add_batch(_batch(trs, False))
  for t in trs:
    b.add(dr.Transition(*t), 1.0) if prioritized else b.add(dr.Transition(*t))
  for r in (a, b):
    assert int(r._flags().item()) & 32
  np.testing.assert_array_equal(a._store.planes.cpu().numpy(), b._store.planes.cpu().numpy())
  assert (a._store.planes.cpu().numpy()[2:6] == 0).all()
  np.testing.assert_array_equal(a._store.refcount.cpu().numpy(), b._store.refcount.cpu().numpy())
  for r in (a, b):
    with pytest.raises(RuntimeError, match='frame pool is full'):
      r.sample(2)
    with pytest.raises(RuntimeError, match='frame pool is full'):
      r.check_valid()


@pytest.mark.parametrize('alpha', [0.5, 1.0, 0.6])
@pytest.mark.parametrize('dedup', [False, True])
def test_priority_forms(alpha, dedup):
  from dqn_zoo_b200 import replay as dr
  obs_shape, cap = (8, 6, 4), 16
  trs = _stacked_stream(4, obs_shape)[:40]
  a, b = _make(True, dedup, cap, alpha=alpha), _make(True, dedup, cap, alpha=alpha)
  dev_pri = torch.tensor(2.75, dtype=torch.float32, device='cuda')
  forms = [(1.5, [1.5] * 10), (np.linspace(0.1, 3.0, 10), list(np.linspace(0.1, 3.0, 10))),
           (np.linspace(0.1, 3.0, 10).astype(np.float32).tolist(), list(np.linspace(0.1, 3.0, 10).astype(np.float32))),
           (dev_pri, [dev_pri] * 10)]
  for k, (batch_pri, seq_pri) in enumerate(forms):
    part = trs[10 * k:10 * k + 10]
    a.add_batch(_batch(part, k % 2 == 0), batch_pri)
    for t, p in zip(part, seq_pri):
      b.add(dr.Transition(*t), priority=p)
    _assert_same(a, b)
  before = _state(a)
  for bad in ([1.0] * 4 + [np.nan] + [1.0] * 5, -1.0, [1.0] * 3):
    with pytest.raises(ValueError):
      a.add_batch(_batch(trs[:10], False), bad)
  after = _state(a)
  for k in before:
    x, y = before[k], after[k]
    if isinstance(x, torch.Tensor):
      assert torch.equal(x, y), k
    elif isinstance(x, np.ndarray):
      np.testing.assert_array_equal(x, y)
    else:
      assert x == y, k
  assert a.size == b.size
  _assert_reads_same(a, b)


def test_shape_mismatch_leaves_the_replay_unchanged():
  from dqn_zoo_b200 import replay as dr
  a = _make(False, False, 8)
  trs = _stacked_stream(2, (8, 6, 4))[:5]
  a.add_batch(_batch(trs, False))
  bad = _batch(trs, False)._replace(s_t=np.zeros((5, 8, 6, 3), np.uint8))
  with pytest.raises(ValueError, match='observation shape/dtype changed'):
    a.add_batch(bad)
  with pytest.raises(ValueError):
    a.add_batch(_batch(trs, False)._replace(r_t=np.zeros(4)))
  assert a.size == 5 and a._t == 5 and list(a.ids()) == list(range(5))


def test_rows_above_4gib_in_the_transition_major_layout():
  """80k rows of 84x84x4 stacks (4.5 GB): the rows at the top of the store start beyond 2**32 bytes; a batch that wraps
  from them to row 0 writes and reads back exactly.  The store is handed back to the driver afterwards, so the
  full-size tests that follow still find the HBM they need."""
  from dqn_zoo_b200 import replay as dr
  cap, obs_shape = 80_000, (84, 84, 4)
  rep = dr.TransitionReplay(cap, dr.Transition(*STRUCT), np.random.RandomState(0))
  try:
    filler = dr.Transition(torch.zeros((256,) + obs_shape, dtype=torch.uint8, device='cuda'), np.zeros(256, np.int64),
                           np.zeros(256), np.zeros(256), torch.zeros((256,) + obs_shape, dtype=torch.uint8, device='cuda'))
    while rep._t + 256 <= cap - 9:
      rep.add_batch(filler)
    rest = cap - 9 - rep._t
    rep.add_batch(dr.Transition(*[f[:rest] for f in filler]))
    assert rep._t == cap - 9 and rep._store.obs[cap - 9].data_ptr() - rep._store.obs.data_ptr() > 2 ** 32
    rs = np.random.RandomState(1)
    part = [ro.Transition(rs.randint(0, 256, size=obs_shape).astype(np.uint8), k, float(k), 0.5,
                          rs.randint(0, 256, size=obs_shape).astype(np.uint8)) for k in range(16)]
    rep.add_batch(_batch(part, False))
    got = rep.get(list(range(cap - 9, cap + 7)))
    for g, w in zip(got, part):
      np.testing.assert_array_equal(g.s_tm1, w.s_tm1)
      np.testing.assert_array_equal(g.s_t, w.s_t)
      assert int(g.a_tm1) == w.a_tm1 and float(g.r_t) == w.r_t
    ok, msg = rep.check_valid()
    assert ok, msg
  finally:
    del rep
    filler = None
    gc.collect()
    torch.cuda.empty_cache()


def _agent(kind, rep, seed, obs_shape):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  net = dl.NetworkSpec(kind, 6, obs_shape=obs_shape)
  common = dict(preprocessor=lambda ts: ts, sample_network_input=np.zeros(obs_shape, np.uint8), network=net,
                optimizer=None, transition_accumulator=dr.NStepTransitionAccumulator(3 if kind == 'rainbow' else 1),
                replay=rep, batch_size=32, min_replay_capacity_fraction=0.05, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=False)
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common)
  return ag.AGENTS[kind](exploration_epsilon=lambda t: 0.1, grad_error_bound=1.0 / 32, **common)


@pytest.mark.parametrize('kind', ['dqn', 'rainbow'])
def test_many_stream_insert_path_end_to_end(kind):
  """E = 8 synthetic streams: VectorizedAtariPreprocessor -> BatchedEpsilonGreedyActor -> VectorNStepAccumulator ->
  add_batch, against the same timesteps through per-stream accumulators and sequential add; then a learner on each
  replay with the same seed: bit-identical loss, priorities and parameters."""
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import processors
  from dqn_zoo_b200 import replay as dr
  E, n_step, cap, seed = 8, 3 if kind == 'rainbow' else 1, 256, 5
  prioritized = kind == 'rainbow'
  rs = np.random.RandomState(seed)
  pre = processors.VectorizedAtariPreprocessor(num_streams=E, device_observations=True)
  L = dl.Learner(dl.NetworkSpec('dqn', 6), batch_size=32)
  L.set_params(lo.init_params(lo.NetSpec('dqn', 6), 2), also_target=True)
  actor = ag.BatchedEpsilonGreedyActor(L, E, exploration_epsilon=0.1, rng_key=[0, seed])
  acc = dr.VectorNStepAccumulator(E, n_step)
  per_stream = [dr.NStepTransitionAccumulator(n_step) for _ in range(E)]
  reps = [_make(prioritized, False, cap, seed) for _ in range(2)]
  remaining = np.zeros(E, np.int64)
  lives = np.full(E, 3)
  for _ in range(120):
    st = np.ones(E, np.int64)
    rw = rs.choice([-1.0, 0.0, 1.0, 2.0], size=E)
    dc = np.ones(E)
    for e in range(E):
      if remaining[e] == 0:
        pre.reset(e)
        st[e], remaining[e] = 0, rs.randint(4, 40)
      else:
        remaining[e] -= 1
        if remaining[e] == 0:
          st[e], dc[e] = 2, 0.0
    rw[st == 0] = np.nan
    dc[st == 0] = np.nan
    frames = torch.as_tensor(rs.randint(0, 256, size=(E, 210, 160, 3)).astype(np.uint8), device='cuda')
    out = pre.step_arrays(frames, st, rw, dc, lives)
    actions = actor.step(pre.stacks)
    batch = acc.step(out['emit'], out['step_type'], out['reward'], out['discount'], pre.stacks, actions)
    if batch is not None:
      reps[0].add_batch(batch, 1.0) if prioritized else reps[0].add_batch(batch)
    for e in np.nonzero(out['emit'])[0]:
      r, d = out['reward'][e], out['discount'][e]
      ts = parts.TimeStep(step_type=parts.StepType(int(out['step_type'][e])), reward=None if np.isnan(r) else float(r),
                          discount=None if np.isnan(d) else float(d), observation=pre.stacks[e].clone())
      for tr in per_stream[e].step(ts, int(actions[e])):
        reps[1].add(tr, 1.0) if prioritized else reps[1].add(tr)
  assert reps[0].size > 100
  _assert_same(reps[0], reps[1])
  runs = []
  for rep in reps:
    agent = _agent(kind, rep, seed, (84, 84, 4))
    trace = []
    for _ in range(4):
      agent.learn()
      trace.append((agent.learner.loss.cpu().numpy().copy(), agent.learner.priorities.cpu().numpy().copy()))
    runs.append((trace, agent.learner.online.cpu().numpy()))
  for (x, y) in zip(runs[0][0], runs[1][0]):
    for u, v in zip(x, y):
      np.testing.assert_array_equal(u, v)
  np.testing.assert_array_equal(runs[0][1], runs[1][1])
