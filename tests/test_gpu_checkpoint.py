"""GPU: checkpoint directories (DESIGN.md §9) — replays, agents, the vector trainer and the run driver.

  * replay round trips, both classes x both layouts x host and device sources, filled by `add` and `add_batch` past
    wrap-around: every device array, the frame pool's plane ids, refcounts, free stack, plane bytes and hashes
    included, and the host bookkeeping equal the saved replay's; the same later adds, samples and priority updates
    then give the same results (new plane ids included);
  * the device digest equals the host twin;
  * agents (dqn, rainbow, iqn with jax taus; CUDA graph on) and a VectorTrainer continue bit-identically after a load;
  * the run driver resumed from `--checkpoint_dir` writes the uninterrupted run's rows;
  * corrupted, truncated or mismatched checkpoints raise, leaving the replay untouched or empty;
  * a 1M x 84x84x4 frame-deduplicated replay round trip with bounded host memory.
"""

import os
import shutil
import sys
import tempfile

import numpy as np
import pytest
import torch

from oracle import checkpoint_oracle as co
from oracle import frame_pool_oracle as fpo
from oracle import replay_oracle as ro
import test_gpu_vector_trainer as vt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCT = (None, None, None, None, None)
OBS = (12, 10, 4)          # 120-byte planes: the pool's 128-byte stride has padding


def _replay(prioritized, dedup, cap=40, seed=7):
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  if prioritized:
    return dr.PrioritizedTransitionReplay(cap, dr.Transition(*STRUCT), 0.5, lambda t: 0.6, 0.1, True, rs,
                                          frame_dedup=dedup)
  return dr.TransitionReplay(cap, dr.Transition(*STRUCT), rs, frame_dedup=dedup)


def _transitions(seed, n_step=1):
  rs = np.random.RandomState(seed)
  lengths = [[9, 30, 2, 14, 11], [25, 1, 17, 8], [6, 6, 40]]
  episodes = [[fpo.stacked_episode(rs, L, OBS, static=(k, j) == (0, 1)) for j, L in enumerate(ls)]
              for k, ls in enumerate(lengths)]
  return fpo.interleave_episodes(rs, [ro.NStepTransitionAccumulator(n_step) for _ in lengths], episodes)


def _feed(rep, trs, source, prioritized, batch_from):
  """`add` for the first `batch_from` transitions, then `add_batch` in batches of 7."""
  from dqn_zoo_b200 import replay as dr
  conv = (lambda x: torch.as_tensor(np.asarray(x), device='cuda')) if source == 'device' else np.asarray
  for k, tr in enumerate(trs[:batch_from]):
    item = dr.Transition(conv(tr.s_tm1), tr.a_tm1, tr.r_t, tr.discount_t, conv(tr.s_t))
    if prioritized:
      rep.add(item, priority=1.0 + k % 5)
    else:
      rep.add(item)
  rest = trs[batch_from:]
  for lo in range(0, len(rest), 7):
    part = rest[lo:lo + 7]
    batch = dr.Transition(conv(np.stack([t.s_tm1 for t in part])), np.array([t.a_tm1 for t in part]),
                          np.array([t.r_t for t in part]), np.array([t.discount_t for t in part]),
                          conv(np.stack([t.s_t for t in part])))
    if prioritized:
      rep.add_batch(batch, 0.5 + (np.arange(len(part)) % 3))
    else:
      rep.add_batch(batch)


def _state(rep):
  """Everything a checkpoint must restore: device arrays (rows / planes, scalars, tree, mirrors, pool) and the host
  bookkeeping, as host values (insertion order of the dicts included)."""
  from dqn_zoo_b200 import replay as dr
  torch.cuda.synchronize()
  st, dist = rep._store, rep._distribution
  dist.flush()
  live = np.asarray(list(rep._live_ids), dtype=np.int64)
  out = {'live_ids': live.tolist(), 't': rep._t}
  if isinstance(dist, dr.UniformDistribution):
    out.update(ids=list(dist._ids), id_to_index=list(dist._id_to_index.items()), mirror=dist._mirror.t.cpu().numpy())
  else:
    out.update(id_to_index=list(dist._id_to_index.items()), index_to_id=list(dist._index_to_id.items()),
               inactive=list(dist._inactive_indices), active=list(dist._active_indices),
               location=list(dist._active_indices_location.items()), size=dist._sum_tree.size,
               tree=dist._sum_tree._nodes.cpu().numpy().view(np.uint64), live_dev=dist._live_dev.t.cpu().numpy(),
               id_at=dist._id_at_dev.t.cpu().numpy())
  if st.obs_shape is None:
    return out
  out.update(action=st.action.cpu().numpy(), reward=st.reward.cpu().numpy().view(np.uint64),
             discount=st.discount.cpu().numpy().view(np.uint64))
  slots = live % rep.capacity
  if isinstance(st, dr._FramePoolStore):
    ref = st.refcount.cpu().numpy()
    ids = np.nonzero(ref)[0]
    top = int(st.counters.item())
    table = st.table.cpu().numpy()
    out.update(planes=st.planes.cpu().numpy(), refcount=ref, free=st.free[:top].cpu().numpy(), top=top,
               frames=st.frames.cpu().numpy()[ids], hashes=st.hashes.cpu().numpy()[ids],
               table=sorted(table[table >= 0].tolist()))
    assert out['table'] == ids.tolist()
  else:
    out['rows'] = st.obs.cpu().numpy()[slots][:, :, :st.obs_bytes]
  return out


def _assert_equal(a, b):
  assert sorted(a) == sorted(b)
  for k in a:
    if isinstance(a[k], np.ndarray):
      np.testing.assert_array_equal(a[k], b[k], err_msg=k)
    else:
      assert a[k] == b[k], k


def _continue(rep, trs, prioritized, source):
  """Further adds, samples and priority updates; returns what they produced."""
  _feed(rep, trs, source, prioritized, batch_from=5)
  out = []
  for _ in range(3):
    got = rep.sample(9)
    if prioritized:
      tr, ids, w = got
      rep.update_priorities(ids, np.linspace(0.25, 3.0, 9).astype(np.float32))
      out.append((ids, w, tr.s_tm1, tr.s_t, tr.r_t))
    else:
      out.append((got.s_tm1, got.s_t, got.a_tm1, got.r_t, got.discount_t))
  return out


@pytest.mark.parametrize('source', ['host', 'device'])
@pytest.mark.parametrize('dedup', [False, True])
@pytest.mark.parametrize('prioritized', [False, True])
def test_replay_round_trip_is_exact(prioritized, dedup, source, tmp_path):
  trs = _transitions(3, n_step=3 if prioritized else 1)
  assert len(trs) > 3 * 40
  a = _replay(prioritized, dedup)
  _feed(a, trs[:100], source, prioritized, batch_from=45)
  if prioritized:
    tr, ids, _ = a.sample(12)
    a.update_priorities(ids, np.linspace(0.5, 2.0, 12).astype(np.float32))
  a.save_checkpoint(str(tmp_path / 'r'))
  b = _replay(prioritized, dedup, seed=1234)
  b.load_checkpoint(str(tmp_path / 'r'))
  _assert_equal(_state(a), _state(b))
  ok, msg = b.check_valid()
  assert ok, msg
  b._random_state.set_state(a._random_state.get_state())     # the run's RandomState, restored by the run
  ga, gb = _continue(a, trs[100:], prioritized, source), _continue(b, trs[100:], prioritized, source)
  for x, y in zip(ga, gb):
    for u, v in zip(x, y):
      np.testing.assert_array_equal(np.asarray(u), np.asarray(v))
  _assert_equal(_state(a), _state(b))          # plane ids of the new adds, free stack order, tree bits


def test_empty_replay_round_trip(tmp_path):
  a = _replay(True, True)
  a.save_checkpoint(str(tmp_path / 'r'))
  b = _replay(True, True)
  b.load_checkpoint(str(tmp_path / 'r'))
  _assert_equal(_state(a), _state(b))


def test_device_digest_equals_the_host_twin_and_oracle():
  import ctypes
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import checkpoint as ck
  rs = np.random.RandomState(0)
  out = torch.zeros(1, dtype=torch.int64, device='cuda')
  for n in [0, 1, 7, 8, 9, 255, 256, 4099, 1 << 20, (1 << 22) + 5]:
    host = rs.randint(0, 256, n).astype(np.uint8)
    dev = torch.as_tensor(host, device='cuda')
    _lib.call('dz_ckpt_digest', dev.data_ptr() if n else None, n, out.data_ptr(), torch.cuda.current_stream().cuda_stream)
    got = int(out.cpu().numpy().view(np.uint64)[0])
    assert got == ck.digest_host(host) == co.digest(host.tobytes()), n
  with pytest.raises(ValueError, match='aligned'):
    _lib.call('dz_ckpt_digest', torch.zeros(16, dtype=torch.uint8, device='cuda').data_ptr() + 1, 8, out.data_ptr(),
              ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))


# -- corruption and mismatches ------------------------------------------------------------------------------------------
def _saved(tmp_path, prioritized, dedup):
  a = _replay(prioritized, dedup)
  _feed(a, _transitions(5)[:90], 'host', prioritized, batch_from=30)
  a.save_checkpoint(str(tmp_path / 'r'))
  return a


def _assert_empty(rep):
  from dqn_zoo_b200 import replay as dr
  assert rep.size == 0 and rep._t == 0 and not rep._distribution._id_to_index
  ok, msg = rep.check_valid()
  assert ok, msg
  if isinstance(rep._store, dr._FramePoolStore):
    assert rep.frames_in_use == 1


@pytest.mark.parametrize('dedup,name', [(True, 'frames'), (False, 'rows'), (True, 'planes'), (True, 'free')])
def test_flipped_byte_raises_and_leaves_the_replay_empty(dedup, name, tmp_path):
  _saved(tmp_path, True, dedup)
  path = tmp_path / 'r' / (name + '.bin')
  raw = bytearray(path.read_bytes())
  raw[len(raw) // 2] ^= 0x01
  path.write_bytes(bytes(raw))
  b = _replay(True, dedup, seed=1)
  _feed(b, _transitions(9)[:20], 'host', True, batch_from=20)
  with pytest.raises(RuntimeError, match=r'%s\.bin: chunk 0 digest' % name):
    b.load_checkpoint(str(tmp_path / 'r'))
  _assert_empty(b)


@pytest.mark.parametrize('dedup', [False, True])
def test_truncated_file_raises_and_leaves_the_replay_empty(dedup, tmp_path):
  _saved(tmp_path, False, dedup)
  path = tmp_path / 'r' / (('frames' if dedup else 'rows') + '.bin')
  raw = path.read_bytes()
  path.write_bytes(raw[:len(raw) - 100])
  b = _replay(False, dedup, seed=1)
  with pytest.raises(RuntimeError, match='truncated'):
    b.load_checkpoint(str(tmp_path / 'r'))
  _assert_empty(b)


def test_inconsistent_pool_raises(tmp_path):
  """A live-plane list that passes its digest but names an unreferenced plane (manifest digests rewritten)."""
  import json
  from dqn_zoo_b200 import checkpoint as ck
  _saved(tmp_path, False, True)
  d = tmp_path / 'r'
  ids = np.fromfile(d / 'pool_ids.bin', dtype=np.int32)
  ids[-1] += 1                                   # still increasing; the plane after the last live one is free
  ids.tofile(d / 'pool_ids.bin')
  m = json.loads((d / ck.MANIFEST).read_text())
  m['files']['pool_ids']['digests'] = ['%016x' % ck.digest_host(ids)]
  (d / ck.MANIFEST).write_text(json.dumps(m))
  b = _replay(False, True, seed=1)
  with pytest.raises(RuntimeError, match='frame pool is inconsistent'):
    b.load_checkpoint(str(d))
  _assert_empty(b)


@pytest.mark.parametrize('other', ['capacity', 'layout', 'kind', 'frame_capacity', 'obs_shape'])
def test_mismatched_manifest_raises_value_error_and_leaves_the_replay_untouched(other, tmp_path):
  from dqn_zoo_b200 import replay as dr
  _saved(tmp_path, False, True)
  rs = np.random.RandomState(1)
  if other == 'capacity':
    b = dr.TransitionReplay(41, dr.Transition(*STRUCT), rs, frame_dedup=True)
  elif other == 'layout':
    b = dr.TransitionReplay(40, dr.Transition(*STRUCT), rs)
  elif other == 'kind':
    b = dr.PrioritizedTransitionReplay(40, dr.Transition(*STRUCT), 0.5, lambda t: 0.6, 0.1, True, rs, frame_dedup=True)
  elif other == 'frame_capacity':
    b = dr.TransitionReplay(40, dr.Transition(*STRUCT), rs, frame_dedup=True, frame_capacity=500)
  else:
    b = dr.TransitionReplay(40, dr.Transition(*STRUCT), rs, frame_dedup=True)
    b.add(dr.Transition(np.zeros((12, 10, 2), np.uint8), 0, 0.0, 1.0, np.zeros((12, 10, 2), np.uint8)))
  if other != 'obs_shape':
    _feed(b, _transitions(9)[:20], 'host', other == 'kind', batch_from=20)
  before = _state(b)
  with pytest.raises(ValueError):
    b.load_checkpoint(str(tmp_path / 'r'))
  _assert_equal(before, _state(b))


# -- agents and the trainer -----------------------------------------------------------------------------------------------
def _agent(kind, rep, seed):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  obs = (44, 44, 4)
  common = dict(preprocessor=lambda ts: ts, sample_network_input=np.zeros(obs, np.uint8),
                network=dl.NetworkSpec(kind, 6, obs_shape=obs), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(3 if kind == 'rainbow' else 1), replay=rep,
                batch_size=32, min_replay_capacity_fraction=0.05, learn_period=4, target_network_update_period=16,
                rng_key=[0, seed], use_cuda_graph=True)
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common)
  if kind == 'iqn':
    return ag.Iqn(exploration_epsilon=lambda t: 0.1, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                  tau_samples_s_t=64, jax_prng_taus=True, **common)
  return ag.Dqn(exploration_epsilon=lambda t: 0.1, grad_error_bound=1.0 / 32, **common)


def _trace(agent, steps):
  L = agent.learner
  out = []
  for _ in range(steps):
    agent.learn()
    out.append([t.cpu().numpy().copy() for t in (L.sampled_ids, L.priorities, L.loss)])
  torch.cuda.synchronize()
  out.append([L.online.cpu().numpy(), L.target.cpu().numpy(), L.opt_state.cpu().numpy(), L.counters.cpu().numpy(),
              L.max_seen_priority.cpu().numpy()])
  return out


@pytest.mark.parametrize('dedup', [False, True])
@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_agent_continues_bit_identically_after_a_load(kind, dedup, tmp_path):
  from dqn_zoo_b200 import replay as dr
  prioritized = kind == 'rainbow'

  def replay(seed):
    rs = np.random.RandomState(seed)
    if prioritized:
      return dr.PrioritizedTransitionReplay(512, dr.Transition(*STRUCT), 0.5, lambda t: 0.4, 1e-3, True, rs,
                                            frame_dedup=dedup)
    return dr.TransitionReplay(512, dr.Transition(*STRUCT), rs, frame_dedup=dedup)
  rep = replay(9)
  dr.bulk_fill_synthetic_stacked(rep, (44, 44, 4), 9, 6, episode_len=37)
  a = _agent(kind, rep, 9)
  _trace(a, 5)
  a.save_checkpoint(str(tmp_path / 'a'))
  rs_state = rep._random_state.get_state()
  want = _trace(a, 6)
  b = _agent(kind, replay(1), 77)            # different seeds and an empty replay: everything comes from the files
  b.load_checkpoint(str(tmp_path / 'a'))
  b._replay._random_state.set_state(rs_state)
  got = _trace(b, 6)
  for x, y in zip(want, got):
    for u, v in zip(x, y):
      np.testing.assert_array_equal(u, v)
  _assert_equal(_state(a._replay), _state(b._replay))


def test_vector_trainer_continues_bit_identically_after_a_load(tmp_path):
  E, T = 8, 40
  script = vt._script(E, 2 * T, seed=4)
  frames = vt._frames(E, 4)
  a = vt._agent('rainbow', vt._min_fill(E), dedup=True)
  tr = vt._trainer(a, E)
  vt._drive(tr, frames, script, 0, T)
  assert tr.learn_steps > 0
  tr.save_checkpoint(str(tmp_path / 't'))
  want = vt._drive(tr, frames, script, T, 2 * T)
  b = vt._agent('rainbow', vt._min_fill(E), seed=99, dedup=True)
  tr2 = vt._trainer(b, E)
  tr2.load_checkpoint(str(tmp_path / 't'))
  got = vt._drive(tr2, frames, script, T, 2 * T)
  np.testing.assert_array_equal(np.stack(want), np.stack(got))
  assert tr.frame_t == tr2.frame_t and tr.learn_steps == tr2.learn_steps
  vt._assert_same_learner(a, b)
  _assert_equal(_state(a._replay), _state(b._replay))
  np.testing.assert_array_equal(tr.episode_return, tr2.episode_return)


def test_run_driver_resumes_from_a_checkpoint_directory(tmp_path):
  """Iterations of the driver's vector-trainer path, stopped after iteration 1 and resumed in fresh objects."""
  sys.path.insert(0, os.path.join(ROOT, 'tools'))
  try:
    import run_synthetic
  finally:
    sys.path.pop(0)
  argv = ['--agent', 'rainbow', '--num_streams', '4', '--num_iterations', '3', '--num_train_frames', '240',
          '--num_eval_frames', '60', '--replay_capacity', '1000', '--min_replay_capacity_fraction', '0.05',
          '--target_network_update_period', '64', '--max_frames_per_episode', '17']
  whole = run_synthetic.run(run_synthetic.parse_args(argv))
  ck = ['--checkpoint_dir', str(tmp_path / 'ck')]
  first = run_synthetic.run(run_synthetic.parse_args(argv[:5] + ['1'] + argv[6:] + ck))
  rest = run_synthetic.run(run_synthetic.parse_args(argv + ck))        # fresh objects, restored from the directory
  assert [r['iteration'] for r in first + rest] == [0, 1, 2, 3]
  rates = ('eval_frame_rate', 'train_frame_rate')
  for x, y in zip(whole, first + rest):
    assert list(x) == list(y)
    for k in x:
      if k not in rates:
        assert x[k] == y[k] or (x[k] != x[k] and y[k] != y[k]), (k, x[k], y[k])


# -- full size ------------------------------------------------------------------------------------------------------------
def _rss_bytes():
  with open('/proc/self/statm') as f:
    return int(f.read().split()[1]) * os.sysconf('SC_PAGE_SIZE')


def test_full_size_frame_dedup_round_trip():
  from dqn_zoo_b200 import replay as dr
  cap, obs = 1_000_000, (84, 84, 4)
  need = (cap + cap // 1000 + 1) * 84 * 84 + 64 * cap          # plane files plus table, scalars and bookkeeping
  tmp = tempfile.gettempdir()
  free = shutil.disk_usage(tmp).free
  if free < need + (2 << 30):
    pytest.skip('%s has %.1f GB free, the checkpoint needs %.1f GB' % (tmp, free / 1e9, need / 1e9))
  directory = tempfile.mkdtemp(prefix='dz_ckpt_')
  try:
    a = dr.TransitionReplay(cap, dr.Transition(*STRUCT), np.random.RandomState(0), frame_dedup=True)
    dr.bulk_fill_synthetic_stacked(a, obs, 5, 6, episode_len=1000)
    torch.cuda.synchronize()
    rss0 = _rss_bytes()
    a.save_checkpoint(directory)
    grown = _rss_bytes() - rss0
    assert grown < (1 << 30), 'host RSS grew by %.2f GiB during the save' % (grown / 2 ** 30)
    b = dr.TransitionReplay(cap, dr.Transition(*STRUCT), np.random.RandomState(0), frame_dedup=True)
    b.load_checkpoint(directory)
    torch.cuda.synchronize()
    sa, sb = a._store, b._store
    for name in ('planes', 'refcount', 'action', 'reward', 'discount'):
      assert torch.equal(getattr(sa, name), getattr(sb, name)), name
    top = int(sa.counters.item())
    assert top == int(sb.counters.item()) and torch.equal(sa.free[:top], sb.free[:top])
    live = torch.nonzero(sa.refcount).reshape(-1)
    assert torch.equal(sa.hashes[live], sb.hashes[live])
    ta, tb = sa.table[sa.table >= 0], sb.table[sb.table >= 0]
    assert torch.equal(torch.sort(ta).values, torch.sort(tb).values)
    pick = live[torch.randperm(live.numel(), generator=torch.Generator().manual_seed(0))[:20000].to(live.device)]
    assert torch.equal(sa.frames[pick], sb.frames[pick])
    slots = torch.as_tensor(np.random.RandomState(1).randint(0, cap, 4096), device='cuda')
    for x, y in zip(sa.gather(slots, 4096), sb.gather(slots, 4096)):
      assert torch.equal(x, y)
    assert list(a._live_ids) == list(b._live_ids) and a._distribution._ids == b._distribution._ids
    ok, msg = b.check_valid()
    assert ok, msg
  finally:
    shutil.rmtree(directory, ignore_errors=True)
