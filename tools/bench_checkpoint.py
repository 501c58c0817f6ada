"""Save and load times of full-size checkpoints (DESIGN.md §9).  One JSON line per case:

  * dqn_dedup_1m: a dqn agent whose frame-deduplicated replay holds 1M transitions of 84x84x4 stacks
    (`bulk_fill_synthetic_stacked`), `save_checkpoint` / `load_checkpoint` of the agent directory;
  * dqn_rows_200k: the same with a transition-major replay of 200k transitions;
  * dqn_rows_200k_filecheckpoint: `reporting.FileCheckpoint` (one pickle of `get_state()`) on that 200k agent.

Each line has save and load seconds (host clock around calls that end in a device synchronise), GB/s over the bytes on
disk, the file bytes, and the growth of the process's peak RSS across the save and across the load.  The card's name
and power limit are read in the same run.  A case whose directory lacks room is reported as skipped.

  python tools/bench_checkpoint.py [--dir /tmp] [--cases dqn_dedup_1m,dqn_rows_200k,dqn_rows_200k_filecheckpoint]"""

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


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--dir', default=tempfile.gettempdir())
  ap.add_argument('--cases', default=','.join(CASES))
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_checkpoint.py needs a CUDA device')
  info = device_info()
  for case in args.cases.split(','):
    if case not in CASES:
      raise SystemExit('unknown case %r (cases: %s)' % (case, ', '.join(CASES)))
    run_case(case, args.dir, info)


if __name__ == '__main__':
  main()
