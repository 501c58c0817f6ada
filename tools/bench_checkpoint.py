"""Save and load times of full-size checkpoints (DESIGN.md §9).  One JSON line per case:

  * dqn_dedup_1m: a dqn agent whose frame-deduplicated replay holds 1M transitions of 84x84x4 stacks
    (`bulk_fill_synthetic_stacked`), `save_checkpoint` / `load_checkpoint` of the agent directory;
  * dqn_rows_200k: the same with a transition-major replay of 200k transitions;
  * dqn_rows_200k_filecheckpoint: `reporting.FileCheckpoint` (one pickle of `get_state()`) on that 200k agent.

Each line has save and load seconds (host clock around calls that end in a device synchronise), GB/s over the bytes on
disk, the file bytes, and the growth of the process's peak RSS across the save and across the load.  The card's name
and power limit are read in the same run.  A case whose directory lacks room is reported as skipped.

  python tools/bench_checkpoint.py [--dir /tmp] [--cases dqn_dedup_1m,dqn_rows_200k,dqn_rows_200k_filecheckpoint]

`--background` measures `DirectoryCheckpoint.save(blocking=False)` instead, for the two directory cases: the training
stall per save (host clock from the call to its return, with a device synchronise before and after), the snapshot
pass's device time (CUDA events around one `dz_ckpt_snapshot` of the replay's bulk records, with its bytes read plus
written per second against the 3.35 TB/s data-sheet HBM rate), the background write time (return to `wait()`), and,
for dqn_dedup_1m, `VectorTrainer` frames/s at E = 256 on `VectorCatch` over that replay with a background write in
flight and with none, alternated for two rounds each.  `--e2e` adds `run_synthetic.py` wall clock for
`--e2e_iterations` 1M-frame Catch iterations (E = 256, 200k transition-major replay) with blocking and with background
checkpoints.

  python tools/bench_checkpoint.py --background [--e2e] [--dir /tmp]"""

import argparse
import json
import os
import resource
import shutil
import subprocess
import sys
import tempfile
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

OBS = (84, 84, 4)
CASES = ('dqn_dedup_1m', 'dqn_rows_200k', 'dqn_rows_200k_filecheckpoint')


def emit(**kw):
  print(json.dumps(kw), flush=True)


def device_info():
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    q = 'unavailable'
  return {'name': torch.cuda.get_device_name(0), 'name_power_limit': q}


def peak_rss():
  return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024


def tree_bytes(path):
  if os.path.isfile(path):
    return os.path.getsize(path)
  return sum(os.path.getsize(os.path.join(r, f)) for r, _, fs in os.walk(path) for f in fs)


def make_agent(capacity, dedup, seed):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rep = dr.TransitionReplay(capacity, dr.Transition(None, None, None, None, None), np.random.RandomState(seed),
                            frame_dedup=dedup)
  return ag.Dqn(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec('dqn', 6), optimizer=None,
                transition_accumulator=dr.TransitionAccumulator(), replay=rep, batch_size=32,
                exploration_epsilon=lambda t: 0.01, min_replay_capacity_fraction=0.05, learn_period=16,
                target_network_update_period=40000, grad_error_bound=1.0 / 32, rng_key=[0, seed])


def run_case(case, root, info):
  from dqn_zoo_b200 import replay as dr
  from dqn_zoo_b200 import reporting
  capacity, dedup = (1_000_000, True) if case == 'dqn_dedup_1m' else (200_000, False)
  frames = capacity + capacity // 1000 + 1
  need = (frames * 84 * 84 if dedup else capacity * 2 * int(np.prod(OBS))) + 64 * capacity
  free = shutil.disk_usage(root).free
  if free < need + (2 << 30):
    emit(case=case, skipped='%s has %.1f GB free, needs %.1f GB' % (root, free / 1e9, need / 1e9), **info)
    return
  a = make_agent(capacity, dedup, 1)
  dr.bulk_fill_synthetic_stacked(a._replay, OBS, 1, 6, episode_len=1000)
  for _ in range(4):
    a.learn()
  torch.cuda.synchronize()
  b = make_agent(capacity, dedup, 2)
  path = tempfile.mkdtemp(prefix='dz_bench_ckpt_', dir=root)
  try:
    if case.endswith('filecheckpoint'):
      target = os.path.join(path, 'ck.pkl')
      save_cp, load_cp = reporting.FileCheckpoint(target), reporting.FileCheckpoint(target)
      save_cp.state.agent, load_cp.state.agent = a, b
      save, load = save_cp.save, load_cp.restore
    else:
      target = os.path.join(path, 'agent')
      save, load = (lambda: a.save_checkpoint(target)), (lambda: b.load_checkpoint(target))
    r0 = peak_rss()
    t0 = time.perf_counter()
    save()
    torch.cuda.synchronize()
    t_save = time.perf_counter() - t0
    r1 = peak_rss()
    nbytes = tree_bytes(target)
    t0 = time.perf_counter()
    load()
    torch.cuda.synchronize()
    t_load = time.perf_counter() - t0
    r2 = peak_rss()
    same = bool(torch.equal(a.learner.online, b.learner.online)) and b._replay.size == capacity
    emit(case=case, capacity=capacity, layout='frames' if dedup else 'rows', file_bytes=nbytes,
         save_s=round(t_save, 3), load_s=round(t_load, 3), save_GBps=round(nbytes / t_save / 1e9, 3),
         load_GBps=round(nbytes / t_load / 1e9, 3), peak_rss_growth_save_GB=round((r1 - r0) / 1e9, 3),
         peak_rss_growth_load_GB=round((r2 - r1) / 1e9, 3), restored=same, **info)
  finally:
    shutil.rmtree(path, ignore_errors=True)
    del a, b
    torch.cuda.empty_cache()


HBM_BYTES_PER_S = 3.35e12    # H100 SXM data sheet


def snapshot_pass_seconds(rep, repeats=3):
  """Device seconds of one dz_ckpt_snapshot over every live record of `rep` (best of `repeats`), and its bytes."""
  import ctypes as C
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import checkpoint as ck
  from dqn_zoo_b200 import replay as dr
  st = rep._store
  v = st.fill_view(_lib.ReplayView())
  if isinstance(st, dr._FramePoolStore):
    fc = st.frame_capacity
    ids = torch.empty(fc, dtype=torch.int32, device='cuda')
    hashes = torch.empty(fc, dtype=torch.int64, device='cuda')
    count = torch.zeros(1, dtype=torch.int64, device='cuda')
    _lib.call('dz_ckpt_pool_live', C.byref(v), ids.data_ptr(), hashes.data_ptr(), count.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    n, record = int(count.item()), st.frame_bytes
  else:
    live = np.asarray(list(rep._live_ids), np.int64) % rep.capacity
    ids = torch.as_tensor(live.astype(np.int32), device='cuda')
    n, record = len(live), 2 * st.obs_bytes
  chunk = max(1, ck.CHUNK_BYTES // record) * record
  packed = torch.empty(n * record, dtype=torch.uint8, device='cuda')
  digests = torch.empty(-(-n * record // chunk), dtype=torch.int64, device='cuda')
  best = float('inf')
  for _ in range(repeats):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    _lib.call('dz_ckpt_snapshot', C.byref(v), ids.data_ptr(), n, packed.data_ptr(), chunk, digests.data_ptr(),
              torch.cuda.current_stream().cuda_stream)
    b.record()
    b.synchronize()
    best = min(best, a.elapsed_time(b) / 1e3)
  del packed, digests, ids
  torch.cuda.empty_cache()
  return best, n * record


def trainer_rates(a, path, rounds=2, ticks=120):
  """dqn VectorTrainer frames/s at E = 256 on VectorCatch over agent `a`'s replay: `ticks` ticks with a background
  write in flight (started at the first tick) and `ticks` with none, alternated `rounds` times."""
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  from dqn_zoo_b200 import reporting
  E = 256
  tr = ag.VectorTrainer(a, num_streams=E, rng_key=[0, 3])
  env = environments.VectorCatch(E, 7)
  ts = env.reset()
  cp = reporting.DirectoryCheckpoint(path)
  cp.state.trainer = tr

  def run(n, save):
    nonlocal ts
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    in_flight = 0
    if save:
      assert cp.save(blocking=False) == 'background'
    for _ in range(n):
      frames, st, rw, dc, lv = ts
      act = tr.step(frames, st, rw, dc, lv)
      last = st == 2
      if last.any():
        tr.reset(np.nonzero(last)[0])
      ts = env.step(act, reset=last)
      in_flight += bool(save and cp._writer is not None and cp._writer.is_alive())
    torch.cuda.synchronize()
    rate = n * E / (time.perf_counter() - t0)
    cp.wait()
    return rate, in_flight
  run(20, False)                            # warm-up: graph capture, staging rings
  out = {'with_write': [], 'without_write': [], 'ticks_with_write_in_flight': []}
  for _ in range(rounds):
    r, k = run(ticks, True)
    out['with_write'].append(round(r))
    out['ticks_with_write_in_flight'].append(k)
    out['without_write'].append(round(run(ticks, False)[0]))
  return out


def run_background(case, root, info):
  from dqn_zoo_b200 import replay as dr
  from dqn_zoo_b200 import reporting
  capacity, dedup = (1_000_000, True) if case == 'dqn_dedup_1m' else (200_000, False)
  frames = capacity + capacity // 1000 + 1
  need = 2 * ((frames * 84 * 84 if dedup else capacity * 2 * int(np.prod(OBS))) + 64 * capacity)
  free = shutil.disk_usage(root).free
  if free < need + (2 << 30):
    emit(case=case, mode='background', skipped='%s has %.1f GB free, needs %.1f GB' % (root, free / 1e9, need / 1e9),
         **info)
    return
  a = make_agent(capacity, dedup, 1)
  dr.bulk_fill_synthetic_stacked(a._replay, OBS, 1, 6, episode_len=1000)
  for _ in range(4):
    a.learn()
  torch.cuda.synchronize()
  kernel_s, kernel_bytes = snapshot_pass_seconds(a._replay)
  path = tempfile.mkdtemp(prefix='dz_bench_ckpt_', dir=root)
  try:
    cp = reporting.DirectoryCheckpoint(path)
    cp.state.agent = a
    stalls, writes, snapshot_gb = [], [], None
    for _ in range(2):
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      mode = cp.save(blocking=False)
      t1 = time.perf_counter()
      torch.cuda.synchronize()
      t2 = time.perf_counter()
      cp.wait()
      t3 = time.perf_counter()
      stalls.append((round(t1 - t0, 4), round(t2 - t0, 4)))
      writes.append(round(t3 - t1, 3))
      assert mode == 'background', mode
    snapshot_gb = round(a.snapshot_checkpoint_bytes() / 1e9, 3)
    nbytes = tree_bytes(os.path.join(path, open(os.path.join(path, 'LATEST')).read().strip()))
    result = dict(case=case, mode='background', capacity=capacity, layout='frames' if dedup else 'rows',
                  file_bytes=nbytes, snapshot_bound_GB=snapshot_gb,
                  stall_s_return_and_after_sync=stalls, background_write_s=writes,
                  snapshot_pass_s=round(kernel_s, 5), snapshot_pass_bytes=kernel_bytes,
                  snapshot_pass_read_write_TBps=round(2 * kernel_bytes / kernel_s / 1e12, 3),
                  snapshot_pass_fraction_of_hbm_rate=round(2 * kernel_bytes / kernel_s / HBM_BYTES_PER_S, 3))
    if case == 'dqn_dedup_1m':
      result['trainer_E256_frames_per_s'] = trainer_rates(a, os.path.join(path, 'trainer'))
    emit(**result, **info)
  finally:
    shutil.rmtree(path, ignore_errors=True)
    del a
    torch.cuda.empty_cache()


def run_e2e(root, info, iterations):
  """Wall clock of run_synthetic.py: `iterations` 1M-frame Catch iterations, blocking and background checkpoints."""
  sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
  import run_synthetic
  argv = ['--env', 'catch', '--agent', 'dqn', '--num_streams', '256', '--num_iterations', str(iterations),
          '--num_train_frames', '1000000', '--num_eval_frames', '25600', '--num_eval_streams', '256',
          '--replay_capacity', '200000', '--min_replay_capacity_fraction', '0.05']
  free = shutil.disk_usage(root).free
  if free < 30e9:
    emit(case='run_synthetic_catch_e256_rows_200k', skipped='%s has %.1f GB free, needs 30 GB' % (root, free / 1e9),
         **info)
    return
  out = {}
  for mode in ('blocking', 'background'):
    path = tempfile.mkdtemp(prefix='dz_bench_e2e_', dir=root)
    try:
      extra = ['--checkpoint_dir', os.path.join(path, 'ck')] + (['--background_checkpoint'] if mode == 'background' else [])
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      run_synthetic.run(run_synthetic.parse_args(argv + extra))
      torch.cuda.synchronize()
      out.setdefault(mode + '_s', []).append(round(time.perf_counter() - t0, 2))
    finally:
      shutil.rmtree(path, ignore_errors=True)
      torch.cuda.empty_cache()
  emit(case='run_synthetic_catch_e256_rows_200k', iterations=iterations, frames_per_iteration=1_000_000, **out, **info)


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--dir', default=tempfile.gettempdir())
  ap.add_argument('--cases', default=None)
  ap.add_argument('--background', action='store_true')
  ap.add_argument('--e2e', action='store_true')
  ap.add_argument('--e2e_iterations', type=int, default=3)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_checkpoint.py needs a CUDA device')
  info = device_info()
  if args.background:
    for case in (args.cases or 'dqn_dedup_1m,dqn_rows_200k').split(','):
      if case not in CASES[:2]:
        raise SystemExit('--background has the cases %s' % ', '.join(CASES[:2]))
      run_background(case, args.dir, info)
    if args.e2e:
      run_e2e(args.dir, info, args.e2e_iterations)
    return
  for case in (args.cases or ','.join(CASES)).split(','):
    if case not in CASES:
      raise SystemExit('unknown case %r (cases: %s)' % (case, ', '.join(CASES)))
    run_case(case, args.dir, info)


if __name__ == '__main__':
  main()
