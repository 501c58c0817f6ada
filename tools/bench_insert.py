"""Replay insert rates: sequential `add` against `add_batch`, and the E-stream actor tick with and without the insert.
One JSON line per number.

  * transitions inserted per second, both layouts x host / device sources x uniform / PER: sequential `add`, and
    `add_batch` at K = 1, 8, 32, 128, on 84x84x4 frame stacks whose consecutive stacks share planes (as
    `processors.atari()` builds them), into a 200k-capacity replay whose ring is full (every add evicts).  The host clock
    runs around work that ends in torch.cuda.synchronize(); the device time per batch (kernels and copies, from a
    torch.profiler pass of its own) is printed beside the host time, so the split between host bookkeeping and kernels
    is visible;
  * E-stream actor ticks per second (dqn, rainbow): VectorizedAtariPreprocessor.step_arrays on device-resident synthetic
    RGB frames + BatchedEpsilonGreedyActor.step(pre.stacks); the same + VectorNStepAccumulator.step + add_batch; the same
    with E per-stream NStepTransitionAccumulators + sequential add instead.

  python tools/bench_insert.py [--capacity 200000] [--transitions 4096] [--streams 32] [--ticks 400]"""

import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

OBS = (84, 84, 4)


def emit(**kw):
  print(json.dumps(kw), flush=True)


def device_info():
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    q = 'unavailable'
  return {'name': torch.cuda.get_device_name(0), 'power_limit_and_max_sm_clock': q}


def make_replay(prioritized, dedup, capacity):
  from dqn_zoo_b200 import replay as dr
  st = dr.Transition(None, None, None, None, None)
  rs = np.random.RandomState(1)
  if prioritized:
    rep = dr.PrioritizedTransitionReplay(capacity, st, 0.5, lambda t: 0.4, 1e-3, True, rs, frame_dedup=dedup)
  else:
    rep = dr.TransitionReplay(capacity, st, rs, frame_dedup=dedup)
  dr.bulk_fill_synthetic_stacked(rep, OBS, 1, 6, episode_len=1000)   # ring full: every add below evicts
  return rep


def stacks(n, seed):
  """n + 1 frame stacks of one stream: stack t holds frames t .. t+3, so consecutive stacks share three planes."""
  frames = np.random.RandomState(seed).randint(0, 256, size=(n + 4, OBS[0], OBS[1])).astype(np.uint8)
  return np.ascontiguousarray(np.stack([frames[c:c + n + 1] for c in range(4)], axis=-1))


def insert(rep, prioritized, src, lo, hi, k):
  from dqn_zoo_b200 import replay as dr
  if k == 0:
    for t in range(lo, hi):
      item = dr.Transition(src[t], t % 6, 1.0, 0.99, src[t + 1])
      rep.add(item, 1.0) if prioritized else rep.add(item)
    return
  for b in range(lo, hi, k):
    e = min(hi, b + k)
    items = dr.Transition(src[b:e], np.arange(b, e) % 6, np.ones(e - b), np.full(e - b, 0.99), src[b + 1:e + 1])
    rep.add_batch(items, 1.0) if prioritized else rep.add_batch(items)


def device_us_per_call(rep, prioritized, src, lo, k, calls):
  """Kernel + copy time per insert call (k = 0: per add), from torch.profiler CUDA activity."""
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    insert(rep, prioritized, src, lo, lo + max(1, k) * calls, k)
    torch.cuda.synchronize()
  total = sum(e.self_device_time_total for e in prof.key_averages())
  return total / calls


def bench_rates(capacity, n):
  host = stacks(n * 6 + 8, 5)
  dev = torch.as_tensor(host, device='cuda')
  for dedup in (False, True):
    for prioritized in (False, True):
      rep = make_replay(prioritized, dedup, capacity)
      for source in ('host', 'device'):
        src = dev if source == 'device' else host
        pos = 0
        for k in (0, 1, 8, 32, 128):
          insert(rep, prioritized, src, pos, pos + 256, k)       # warm-up of this shape
          pos += 256
          torch.cuda.synchronize()
          t0 = time.perf_counter()
          insert(rep, prioritized, src, pos, pos + n, k)
          t_host = time.perf_counter() - t0
          torch.cuda.synchronize()
          dt = time.perf_counter() - t0
          pos += n
          calls = 16
          dev_us = device_us_per_call(rep, prioritized, src, pos, k, calls)
          pos += max(1, k) * calls
          emit(metric='insert_transitions_per_sec', method='add' if k == 0 else 'add_batch', K=k or None,
               layout='frame_dedup' if dedup else 'transition_major', source=source,
               replay='per' if prioritized else 'uniform', value=round(n / dt, 1), transitions=n,
               host_us_per_call=round(1e6 * t_host / (n / max(1, k)), 2), device_us_per_call=round(dev_us, 2),
               capacity=capacity)
        if pos > len(host) - 1:
          raise AssertionError('source stacks exhausted')
      ok, msg = rep.check_valid()
      assert ok, msg
      del rep
      torch.cuda.empty_cache()


def bench_ticks(kind, E, ticks, capacity):
  from dqn_zoo_b200 import agent as agent_lib
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import processors
  from dqn_zoo_b200 import replay as dr
  from oracle import learner_oracle as lo
  prioritized, n_step = (True, 3) if kind == 'rainbow' else (False, 1)
  L = dl.Learner(dl.NetworkSpec(kind, 6), batch_size=max(32, E))
  L.set_params(lo.init_params(lo.NetSpec(kind, 6), 2), also_target=True)
  rs = np.random.RandomState(0)
  frames = [torch.as_tensor(rs.randint(0, 256, size=(E, 210, 160, 3)).astype(np.uint8), device='cuda') for _ in range(8)]
  mid, zeros, ones, lives = np.ones(E, np.int64), np.zeros(E), np.ones(E), np.full(E, 3)
  nan = np.full(E, np.nan)
  for variant in ('act', 'act+batched_insert', 'act+sequential_insert'):
    pre = processors.VectorizedAtariPreprocessor(num_streams=E, device_observations=True)
    actor = agent_lib.BatchedEpsilonGreedyActor(L, E, exploration_epsilon=0.01, rng_key=[0, 3])
    rep = make_replay(prioritized, True, capacity) if variant != 'act' else None
    acc = dr.VectorNStepAccumulator(E, n_step)
    per_stream = [dr.NStepTransitionAccumulator(n_step) for _ in range(E)]
    inserted = 0

    def tick(t):
      nonlocal inserted
      first = t == 0
      out = pre.step_arrays(frames[t % 8], np.zeros(E, np.int64) if first else mid, nan if first else zeros,
                            nan if first else ones, lives)
      actions = actor.step(pre.stacks)
      if variant == 'act+batched_insert':
        batch = acc.step(out['emit'], out['step_type'], out['reward'], out['discount'], pre.stacks, actions)
        if batch is not None:
          rep.add_batch(batch, 1.0) if prioritized else rep.add_batch(batch)
          inserted += len(batch.r_t)
      elif variant == 'act+sequential_insert':
        for e in np.nonzero(out['emit'])[0]:
          r, d = out['reward'][e], out['discount'][e]
          ts = parts.TimeStep(step_type=parts.StepType(int(out['step_type'][e])),
                              reward=None if np.isnan(r) else float(r), discount=None if np.isnan(d) else float(d),
                              observation=pre.stacks[e].clone())
          for tr in per_stream[e].step(ts, int(actions[e])):
            rep.add(tr, 1.0) if prioritized else rep.add(tr)
            inserted += 1

    for t in range(40):
      tick(t)
    torch.cuda.synchronize()
    inserted = 0
    t0 = time.perf_counter()
    for t in range(40, 40 + ticks):
      tick(t)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    emit(metric='actor_ticks_per_sec', agent=kind, streams=E, variant=variant, value=round(ticks / dt, 1),
         decisions_per_sec=round(ticks * E / dt, 1), transitions_inserted=inserted, ticks=ticks,
         note='frame_dedup replay (capacity %d, full); action repeat 4: a stream emits a timestep every 4th tick' % capacity)
    del rep
    torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--capacity', type=int, default=200000)
  ap.add_argument('--transitions', type=int, default=4096)
  ap.add_argument('--streams', type=int, default=32)
  ap.add_argument('--ticks', type=int, default=400)
  ap.add_argument('--skip', default='', help='comma-separated parts to skip: rates,ticks')
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_insert.py needs a CUDA device')
  torch.cuda.set_device(0)
  emit(metric='device', **device_info())
  skip = set(a.skip.split(','))
  if 'rates' not in skip:
    bench_rates(a.capacity, a.transitions)
  if 'ticks' not in skip:
    for kind in ('dqn', 'rainbow'):
      bench_ticks(kind, a.streams, a.ticks, a.capacity)


if __name__ == '__main__':
  main()
