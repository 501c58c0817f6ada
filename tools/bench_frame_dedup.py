"""Frame-deduplicated replay (`frame_dedup=True`) against the transition-major layout, one JSON line per number:

  * HBM bytes of a 1M-transition replay of 84x84x4 frame stacks in each layout, and frames_in_use after the stacked fill;
  * fused learner grad-steps/s (rainbow, dqn) on identical stacked contents in both layouts, alternated, three runs each;
  * add() calls/s in both layouts, from host arrays and from device tensors;
  * aggregate grad-steps/s of K learners with a 1M dedup replay each on one GPU, K = 1, 2, 4, ... while HBM lasts.

  python tools/bench_frame_dedup.py [--capacity 200000] [--steps 1000] [--learners 1,2,4]
The step timing uses --capacity (both layouts must fit at once); the sampled rows are spread over the whole store."""

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

OBS = (84, 84, 4)
EPISODE_LEN = 1000
SETUP = {'rainbow': (True, 0.5, 3), 'dqn': (False, 1.0, 1)}   # prioritized, alpha, n-step


def emit(**kw):
  print(json.dumps(kw), flush=True)


def make_replay(kind, capacity, dedup, seed):
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import replay as dr
  pri, alpha, n_step = SETUP[kind]
  rs = np.random.RandomState(seed)
  st = dr.Transition(None, None, None, None, None)
  if pri:
    sched = parts.LinearSchedule(begin_t=int(0.02 * capacity), end_t=200 * 250000, begin_value=0.4, end_value=1.0)
    rep = dr.PrioritizedTransitionReplay(capacity, st, alpha, sched, 1e-3, True, rs, frame_dedup=dedup)
  else:
    rep = dr.TransitionReplay(capacity, st, rs, frame_dedup=dedup)
  dr.bulk_fill_synthetic_stacked(rep, OBS, seed, 6, episode_len=EPISODE_LEN, discount=0.99 ** n_step)
  return rep


def make_agent(kind, rep, seed):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  common = dict(preprocessor=lambda ts: ts, sample_network_input=np.zeros(OBS, np.uint8),
                network=dl.NetworkSpec(kind, 6), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(SETUP[kind][2]), replay=rep, batch_size=32,
                min_replay_capacity_fraction=0.02, learn_period=16, target_network_update_period=32000,
                rng_key=[0, seed], use_cuda_graph=True)
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common)
  return ag.Dqn(exploration_epsilon=lambda t: 0.01, grad_error_bound=1.0 / 32, **common)


def time_steps(agent, draws, steps, warmup):
  for i in range(warmup):
    agent.learn_from_device_draws(draws[i % len(draws)])
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for i in range(steps):
    agent.learn_from_device_draws(draws[i % len(draws)])
  e1.record()
  torch.cuda.synchronize()
  agent.check_device_flags()
  return e0.elapsed_time(e1) / steps


def bench_bytes():
  from dqn_zoo_b200 import replay as dr
  cap = 1000000
  obs_stride = (int(np.prod(OBS)) + 15) // 16 * 16
  tm_bytes = cap * 2 * obs_stride + cap * (4 + 8 + 8) + 4     # rows + action/reward/discount + flags
  emit(metric='replay_hbm_bytes', layout='transition_major', capacity=cap, obs=list(OBS), bytes=tm_bytes,
       note='computed from the row layout (not allocated)')
  rep = make_replay('rainbow', cap, True, 1)
  emit(metric='replay_hbm_bytes', layout='frame_dedup', capacity=cap, obs=list(OBS), bytes=rep.storage_bytes,
       frame_capacity=rep._store.frame_capacity, frames_in_use=rep.frames_in_use, episode_len=EPISODE_LEN)
  del rep
  torch.cuda.empty_cache()


def bench_steps(capacity, steps, warmup):
  for kind in ('rainbow', 'dqn'):
    agents = {}
    for dedup in (False, True):
      rep = make_replay(kind, capacity, dedup, 3)
      agent = make_agent(kind, rep, 3)
      draws = torch.as_tensor(np.stack([agent.host_draws() for _ in range(64)]), device='cuda')
      agents[dedup] = (agent, rep, draws)
    ms = {False: [], True: []}
    for _ in range(3):
      for dedup in (False, True):
        agent, _, draws = agents[dedup]
        ms[dedup].append(time_steps(agent, draws, steps, warmup))
    for dedup in (False, True):
      emit(metric='fused_grad_steps_per_sec', agent=kind, layout='frame_dedup' if dedup else 'transition_major',
           capacity=capacity, runs_us_per_step=[round(1e3 * m, 2) for m in ms[dedup]],
           value=1e3 / float(np.median(ms[dedup])), steps=steps, warmup=warmup,
           timing='CUDA events around %d CUDA-graph replays; layouts alternated, median of 3' % steps)
    agent, rep, _ = agents[True]
    slots = torch.as_tensor(np.random.RandomState(0).randint(capacity, size=32), device='cuda')
    out = torch.empty((32, 2, rep._store.obs_stride), dtype=torch.uint8, device='cuda')
    from dqn_zoo_b200 import _lib
    import ctypes as C
    v = rep.device_view()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for rnd in range(2):
      e0.record()
      for _ in range(steps):
        _lib.call('dz_replay_gather', C.byref(v), slots.data_ptr(), 32, out.data_ptr(), out.data_ptr() + rep._store.obs_stride,
                  None, None, None, torch.cuda.current_stream().cuda_stream)
      e1.record()
      torch.cuda.synchronize()
    emit(metric='frame_reconstruct_us', agent=kind, batch=32,
         value=1e3 * e0.elapsed_time(e1) / steps, note='dz_replay_gather of a dedup replay: reconstruct kernel + '
         'scalar gather, eager launches back to back')
    del agents
    torch.cuda.empty_cache()


def bench_adds(n=3000):
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(0)
  frames = rs.randint(0, 256, size=(n + 4, 84, 84)).astype(np.uint8)
  stacks = np.stack([np.stack([frames[t + c] for c in range(4)], axis=-1) for t in range(n + 1)])
  dev = torch.as_tensor(stacks, device='cuda')
  for dedup in (False, True):
    for source in ('host', 'device'):
      rep = dr.TransitionReplay(2000, dr.Transition(None, None, None, None, None), np.random.RandomState(1),
                                frame_dedup=dedup)
      src = dev if source == 'device' else stacks
      for t in range(50):
        rep.add(dr.Transition(src[t], 0, 0.0, 0.99, src[t + 1]))
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      for t in range(n):
        rep.add(dr.Transition(src[t], 0, 0.0, 0.99, src[t + 1]))
      torch.cuda.synchronize()
      dt = time.perf_counter() - t0
      emit(metric='replay_add_calls_per_sec', layout='frame_dedup' if dedup else 'transition_major', source=source,
           value=n / dt, adds=n, note='one host thread, synchronised at the end; ring wraps (capacity 2000)')


def bench_multi(ks, steps, warmup):
  from dqn_zoo_b200 import replay as dr  # noqa: F401
  cap = 1000000
  for k in ks:
    free, _ = torch.cuda.mem_get_info()
    if k * 15.5e9 > free:
      emit(metric='learner_grad_steps_per_sec (aggregate, 1M dedup replay each)', learners=k, value=None,
           note='not run: %.1f GB of HBM free' % (free / 1e9))
      break
    shards = []
    for j in range(k):
      stream = torch.cuda.Stream()
      with torch.cuda.stream(stream):
        rep = make_replay('rainbow', cap, True, 1 + 17 * j)
        agent = make_agent('rainbow', rep, 1 + 17 * j)
        draws = torch.as_tensor(np.stack([agent.host_draws() for _ in range(64)]), device='cuda')
        for i in range(3):
          agent.learn_from_device_draws(draws[i])
      stream.synchronize()
      shards.append((agent, rep, stream, draws))

    def sweep(n):
      for i in range(n):
        for agent, _, stream, draws in shards:
          with torch.cuda.stream(stream):
            agent.learn_from_device_draws(draws[i % 64])
    sweep(warmup)
    torch.cuda.synchronize()
    e0 = [torch.cuda.Event(enable_timing=True) for _ in shards]
    e1 = [torch.cuda.Event(enable_timing=True) for _ in shards]
    for (_, _, stream, _), ev in zip(shards, e0):
      ev.record(stream)
    sweep(steps)
    for (_, _, stream, _), ev in zip(shards, e1):
      ev.record(stream)
    torch.cuda.synchronize()
    ms = max(a.elapsed_time(b) for a, b in zip(e0, e1))
    value = k * steps / (ms / 1e3)
    emit(metric='learner_grad_steps_per_sec (aggregate, 1M dedup replay each)', learners=k, agent='rainbow',
         value=value, per_learner=value / k, replay_gb_total=sum(s[1].storage_bytes for s in shards) / 1e9,
         steps=steps, timing='CUDA events on each shard stream, max over shards; round-robin graph replays')
    del shards
    torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--capacity', type=int, default=200000)
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--learners', default='1,2,4')
  ap.add_argument('--skip', default='', help='comma-separated parts to skip: bytes,steps,adds,multi')
  a = ap.parse_args()
  torch.cuda.set_device(0)
  emit(metric='device', name=torch.cuda.get_device_name(0))
  skip = set(a.skip.split(','))
  if 'bytes' not in skip:
    bench_bytes()
  if 'steps' not in skip:
    bench_steps(a.capacity, a.steps, a.warmup)
  if 'adds' not in skip:
    bench_adds()
  if 'multi' not in skip:
    bench_multi([int(x) for x in a.learners.split(',')], a.steps, a.warmup)


if __name__ == '__main__':
  main()
