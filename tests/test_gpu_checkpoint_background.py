"""GPU: checkpoints taken without stopping training (DESIGN.md §9).

  * the snapshot pass (`dz_ckpt_snapshot`): for both layouts, record sizes that are and are not multiples of 8 and 16,
    chunks of one record, exactly one chunk, one chunk plus one record, a partial last chunk and n = 0, the packed
    bytes equal the records and every chunk digest equals `dz_ckpt_digest` of that chunk; plane ids and row slots whose
    byte offsets exceed 2^32;
  * replays of both classes and layouts, snapshotted and then changed further, write exactly the files of a blocking
    save at the snapshot point;
  * dqn (frame-deduplicated) and rainbow (PER, n = 3, transition-major) `VectorTrainer`s on `VectorCatch`: a snapshot
    written after further ticks that evict rows and reuse planes leaves training bit-identical to a twin that never
    saved, its directory equals the twin's blocking save, and a trainer loaded from it continues as the twin does;
  * the run driver with `--background_checkpoint` writes the blocking run's rows and resumes as it does;
  * a save forced to fall back to blocking writes the same files.
"""

import ctypes as C
import filecmp
import os
import sys

import numpy as np
import pytest
import torch

import test_gpu_checkpoint as gc
import test_gpu_vector_trainer as vt

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STRUCT = (None, None, None, None, None)


def _assert_same_tree(a, b):
  """Every file under a and b exists in both and is byte-identical."""
  names = lambda root: sorted(os.path.relpath(os.path.join(r, f), root) for r, _, fs in os.walk(root) for f in fs)
  assert names(a) == names(b)
  for name in names(a):
    assert filecmp.cmp(os.path.join(a, name), os.path.join(b, name), shallow=False), name


# -- 1: the snapshot pass ---------------------------------------------------------------------------------------------
def _filled(dedup, obs, cap, episode_len=7):
  """A replay holding `cap` rows: `bulk_fill_synthetic_stacked` where it applies (H*W a multiple of 8), else 1.5 * cap
  `add`s of random stacks (so some rows were evicted)."""
  from dqn_zoo_b200 import replay as dr
  rep = dr.TransitionReplay(cap, dr.Transition(*STRUCT), np.random.RandomState(0), frame_dedup=dedup)
  if obs[0] * obs[1] % 8 == 0:
    dr.bulk_fill_synthetic_stacked(rep, obs, 3, 6, episode_len=episode_len)
    return rep
  rs = np.random.RandomState(1)
  for k in range(cap * 3 // 2):
    s_tm1, s_t = rs.randint(0, 256, (2,) + tuple(obs)).astype(np.uint8)
    rep.add(dr.Transition(s_tm1, k % 6, float(k % 3 - 1), 0.99, s_t))
  return rep


def _records(rep, ids):
  """The records ids as the file stores them, gathered by torch indexing: planes without their stride padding, or
  s_tm1 | s_t of rows."""
  st = rep._store
  idx = ids.long()
  if hasattr(st, 'frames') and st.frames is not None:
    return st.frames[idx, :st.frame_bytes].reshape(-1)
  return st.obs[idx, :, :st.obs_bytes].reshape(-1)


def _snapshot(rep, ids, n, chunk, size=None):
  from dqn_zoo_b200 import _lib
  v = rep._store.fill_view(_lib.ReplayView())
  packed = torch.full((size or max(1, n * _record(rep)),), 0xAB, dtype=torch.uint8, device='cuda')
  digests = torch.full((max(1, -(-n * _record(rep) // chunk)),), -7, dtype=torch.int64, device='cuda')
  _lib.call('dz_ckpt_snapshot', C.byref(v), ids.data_ptr(), n, packed.data_ptr(), chunk, digests.data_ptr(),
            torch.cuda.current_stream().cuda_stream)
  return packed, digests


def _record(rep):
  st = rep._store
  return st.frame_bytes if getattr(st, 'frames', None) is not None else 2 * st.obs_bytes


def _device_digest(data):
  from dqn_zoo_b200 import _lib
  data = data.clone()                                            # a chunk need not start 8-byte aligned
  out = torch.zeros(1, dtype=torch.int64, device='cuda')
  _lib.call('dz_ckpt_digest', data.data_ptr(), data.numel(), out.data_ptr(), torch.cuda.current_stream().cuda_stream)
  return int(out.item())


def _live_ids(rep):
  st = rep._store
  if getattr(st, 'frames', None) is not None:
    return (torch.nonzero(st.refcount[1:] > 0).reshape(-1) + 1).to(torch.int32)
  slots = np.asarray(list(rep._live_ids), np.int64) % rep.capacity
  return torch.as_tensor(slots[::-1].copy().astype(np.int32), device='cuda')   # any order: the file's order is the list's


@pytest.mark.parametrize('obs', [(8, 8, 4), (12, 10, 4), (5, 5, 3), (3, 3, 1)])
@pytest.mark.parametrize('dedup', [False, True])
def test_snapshot_pass_packs_and_digests_every_chunk(dedup, obs):
  """Planes of 64 / 120 / 25 / 9 bytes and rows of 512 / 960 / 150 / 18 bytes: the 16-byte path and the word path,
  with words that straddle two records (25, 9, 150 and 18 are not multiples of 8)."""
  from dqn_zoo_b200 import checkpoint as ck
  rep = _filled(dedup, obs, cap=60)
  ids = _live_ids(rep)
  n, rec = ids.numel(), _record(rep)
  assert n > 10
  want = _records(rep, ids)
  for chunk in (rec, 3 * rec, (n - 1) * rec, n * rec, (n + 5) * rec, ck.CHUNK_BYTES // rec * rec):
    packed, digests = _snapshot(rep, ids, n, chunk)
    torch.cuda.synchronize()
    assert torch.equal(packed[:n * rec], want), chunk
    nchunks = -(-n * rec // chunk)
    got = digests.cpu().numpy()
    for k in range(nchunks):
      part = packed[k * chunk:min(n * rec, (k + 1) * chunk)]
      assert int(got[k]) == _device_digest(part), (chunk, k)
      assert int(got[k:k + 1].view(np.uint64)[0]) == ck.digest_host(part.cpu().numpy()), (chunk, k)
  # one record, and a subrange of the list
  for lo, m in ((0, 1), (n - 1, 1), (3, 5)):
    packed, digests = _snapshot(rep, ids[lo:], m, 2 * rec)
    assert torch.equal(packed[:m * rec], want[lo * rec:(lo + m) * rec])
    for k in range(-(-m // 2)):
      assert int(digests[k].item()) == _device_digest(packed[k * 2 * rec:min(m, 2 * k + 2) * rec])


@pytest.mark.parametrize('dedup', [False, True])
def test_snapshot_pass_with_no_records_writes_nothing(dedup):
  rep = _filled(dedup, (12, 10, 4), cap=20)
  ids = _live_ids(rep)
  packed, digests = _snapshot(rep, ids, 0, _record(rep), size=64)
  torch.cuda.synchronize()
  assert bool((packed == 0xAB).all()) and int(digests[0].item()) == -7


def test_snapshot_pass_rejects_a_chunk_that_splits_records():
  rep = _filled(True, (5, 5, 3), cap=20)
  ids = _live_ids(rep)
  with pytest.raises(ValueError, match='multiple of the record'):
    _snapshot(rep, ids, 3, 24)


@pytest.mark.parametrize('dedup', [False, True])
def test_snapshot_pass_offsets_beyond_4_gib(dedup):
  """A plane id (frame-deduplicated, 84x84 planes) and a row slot (transition-major, 84x84x4 rows) whose byte offsets
  exceed 2^32; only the records named are read back."""
  if dedup:
    rep = _filled(True, (84, 84, 1), cap=640_000, episode_len=1000)
    last = int(torch.nonzero(rep._store.refcount > 0).max().item())
    assert last * rep._store.frame_stride > 2 ** 32
  else:
    rep = _filled(False, (84, 84, 4), cap=80_000, episode_len=1000)
    last = rep.capacity - 1
    assert last * 2 * rep._store.obs_stride > 2 ** 32
  ids = torch.tensor([last, 1, last - 1], dtype=torch.int32, device='cuda')
  rec = _record(rep)
  packed, digests = _snapshot(rep, ids, 3, 2 * rec)
  torch.cuda.synchronize()
  assert torch.equal(packed, _records(rep, ids))
  assert int(digests[0].item()) == _device_digest(packed[:2 * rec])
  assert int(digests[1].item()) == _device_digest(packed[2 * rec:])
  del rep
  torch.cuda.empty_cache()


# -- 2: a replay snapshot writes the blocking save's files -----------------------------------------------------------
@pytest.mark.parametrize('dedup', [False, True])
@pytest.mark.parametrize('prioritized', [False, True])
def test_replay_snapshot_writes_the_blocking_files(prioritized, dedup, tmp_path):
  trs = gc._transitions(3, n_step=3 if prioritized else 1)
  a, b = gc._replay(prioritized, dedup), gc._replay(prioritized, dedup)
  for rep in (a, b):
    gc._feed(rep, trs[:70], 'host', prioritized, batch_from=30)
    gc._continue(rep, trs[70:90], prioritized, 'device')          # adds, samples, priority updates
  want_state = gc._state(b)
  sampling = a._random_state.get_state()                        # the run's, not the checkpoint's (as for get_state)
  snap = a.snapshot_checkpoint()
  assert snap.device_bytes > 0
  after = gc._continue(a, trs[90:], prioritized, 'host')         # rows evicted, planes freed and reused
  assert len(trs[90:]) > a.capacity
  b.save_checkpoint(str(tmp_path / 'blocking'))
  snap.write(str(tmp_path / 'snapshot'))
  snap.release()
  _assert_same_tree(str(tmp_path / 'snapshot'), str(tmp_path / 'blocking'))
  c = gc._replay(prioritized, dedup, seed=8)
  c.load_checkpoint(str(tmp_path / 'snapshot'))
  gc._assert_equal(gc._state(c), want_state)
  c._random_state.set_state(sampling)
  got = gc._continue(c, trs[90:], prioritized, 'host')
  for x, y in zip(after, got):
    for u, v in zip(x, y):
      np.testing.assert_array_equal(u, v)


# -- 3: training goes on while the snapshot is written --------------------------------------------------------------
def _catch_drive(trainer, env, timesteps, ticks):
  actions = []
  for _ in range(ticks):
    frames, step_type, reward, discount, lives = timesteps
    a = trainer.step(frames, step_type, reward, discount, lives)
    actions.append(a)
    last = step_type == vt.LAST
    if last.any():
      trainer.reset(np.nonzero(last)[0])
    timesteps = env.step(a, reset=last)
  return actions, timesteps


def _host_timesteps(ts):
  return (ts[0],) + tuple(np.copy(x) for x in ts[1:])


@pytest.mark.parametrize('kind,dedup', [('dqn', True), ('rainbow', False)])
def test_trainer_snapshot_leaves_training_unaffected(kind, dedup, tmp_path):
  from dqn_zoo_b200 import environments
  E, T, U, cap = 16, 24, 40, 256
  ta = vt._trainer(vt._agent(kind, 3 * E, capacity=cap, dedup=dedup), E)
  tb = vt._trainer(vt._agent(kind, 3 * E, capacity=cap, dedup=dedup), E)
  ea, eb = environments.VectorCatch(E, 9), environments.VectorCatch(E, 9)
  _, tsa = _catch_drive(ta, ea, ea.reset(), T)
  _, tsb = _catch_drive(tb, eb, eb.reset(), T)
  assert ta.learn_steps > 0
  env_at_t, ts_at_t = eb.get_state(), _host_timesteps(tsb)

  snap = ta.snapshot_checkpoint()
  tb.save_checkpoint(str(tmp_path / 'blocking'))
  got, _ = _catch_drive(ta, ea, tsa, U)                         # U * E frames: more than the replay holds
  want, _ = _catch_drive(tb, eb, tsb, U)
  assert U * E > cap
  snap.write(str(tmp_path / 'snapshot'))
  snap.release()
  np.testing.assert_array_equal(np.stack(got), np.stack(want))
  vt._assert_same_learner(ta.agent, tb.agent)
  gc._assert_equal(gc._state(ta.agent._replay), gc._state(tb.agent._replay))
  _assert_same_tree(str(tmp_path / 'snapshot'), str(tmp_path / 'blocking'))

  tc = vt._trainer(vt._agent(kind, 3 * E, seed=99, capacity=cap, dedup=dedup), E)
  tc.load_checkpoint(str(tmp_path / 'snapshot'))
  ec = environments.VectorCatch(E, 9)
  ec.set_state(env_at_t)
  resumed, _ = _catch_drive(tc, ec, (ec.frames,) + ts_at_t[1:], U)
  np.testing.assert_array_equal(np.stack(resumed), np.stack(want))
  vt._assert_same_learner(tc.agent, tb.agent)
  gc._assert_equal(gc._state(tc.agent._replay), gc._state(tb.agent._replay))


def test_directory_checkpoint_background_and_fallback_write_the_blocking_files(tmp_path):
  from dqn_zoo_b200 import environments
  from dqn_zoo_b200 import reporting
  E, T = 8, 20
  trainers = [vt._trainer(vt._agent('rainbow', 3 * E, capacity=128, dedup=True), E) for _ in range(3)]
  envs = [environments.VectorCatch(E, 5) for _ in range(3)]
  for tr, env in zip(trainers, envs):
    _catch_drive(tr, env, env.reset(), T)
  modes = []
  for k, (tr, blocking, budget) in enumerate(zip(trainers, (True, False, False), (None, None, 0))):
    cp = reporting.DirectoryCheckpoint(str(tmp_path / str(k)), snapshot_budget=budget)
    cp.state.trainer = tr
    cp.state.iteration = 4
    modes.append(cp.save(blocking=blocking))
    cp.wait()
  assert modes == ['blocking', 'background', 'blocking']
  for k in (1, 2):
    _assert_same_tree(str(tmp_path / str(k)), str(tmp_path / '0'))


# -- 4: the run driver --------------------------------------------------------------------------------------------
def _driver(argv, csv_path):
  """One run of tools/run_synthetic.py in a fresh process (as a user runs it); its CSV rows."""
  import csv
  import subprocess
  subprocess.run([sys.executable, os.path.join(ROOT, 'tools', 'run_synthetic.py')] + argv +
                 ['--results_csv_path', csv_path], check=True, cwd=ROOT, stdout=subprocess.DEVNULL)
  with open(csv_path) as f:
    return list(csv.DictReader(f))


def test_run_driver_background_checkpoints(tmp_path):
  sys.path.insert(0, os.path.join(ROOT, 'tools'))
  try:
    import run_synthetic
  finally:
    sys.path.pop(0)
  argv = ['--env', 'catch', '--agent', 'rainbow', '--num_streams', '8', '--num_iterations', '3',
          '--num_train_frames', '320', '--num_eval_frames', '80', '--num_eval_streams', '4', '--replay_capacity', '256',
          '--min_replay_capacity_fraction', '0.1', '--target_network_update_period', '64']
  with pytest.raises(SystemExit):
    run_synthetic.parse_args(argv + ['--background_checkpoint'])
  i = argv.index('--num_iterations') + 1
  first = argv[:i] + ['1'] + argv[i + 1:]
  runs = {}
  for mode in ('blocking', 'background'):
    extra = ['--checkpoint_dir', str(tmp_path / mode)] + (['--background_checkpoint'] if mode == 'background' else [])
    whole = _driver(argv + ['--checkpoint_dir', str(tmp_path / (mode + '_whole'))] + extra[2:],
                    str(tmp_path / (mode + '_whole.csv')))
    _driver(first + extra, str(tmp_path / (mode + '.csv')))
    resumed = _driver(argv + extra, str(tmp_path / (mode + '.csv')))   # restored from the directory; appends its rows
    runs[mode] = (whole, resumed)
  for mode in ('blocking', 'background'):
    assert open(os.path.join(str(tmp_path / mode), 'LATEST')).read() == 'gen-000004\n'
  _assert_same_tree(str(tmp_path / 'background' / 'gen-000004' / 'train_agent'),
                    str(tmp_path / 'blocking' / 'gen-000004' / 'train_agent'))
  rates = ('eval_frame_rate', 'train_frame_rate')
  for k, what in enumerate(('uninterrupted run', 'run resumed from the directory')):
    want, got = runs['blocking'][k], runs['background'][k]
    assert [r['iteration'] for r in got] == [r['iteration'] for r in want] == ['0', '1', '2', '3']
    for x, y in zip(want, got):
      assert list(x) == list(y)
      assert {c: v for c, v in x.items() if c not in rates} == {c: v for c, v in y.items() if c not in rates}, what
