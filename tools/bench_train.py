"""End-to-end training rate of `agent.VectorTrainer`: the full tick (preprocess, act, insert, learn and sync) for E
environment streams on device-resident synthetic RGB frames, for dqn and rainbow at E in {1, 32, 128, 256}.  One JSON
line per point:

  * train_frames_per_sec: environment frames consumed per second (E per tick), host clock around ticks that end in a
    device synchronise;
  * learner_steps_per_sec: learner steps run per second in the same window (one per learn_period = 16 frames);
  * learner_only_frames_per_sec: the bound set by the learner alone, 16 x the rate of back-to-back CUDA-graph learner
    steps on the same agent, so the gap between the tick and the learner is visible.

Batch-32 learner, replay of `--capacity` transitions (frame-deduplicated, prefilled, so the minimum-replay gate is open),
target sync every 40000 frames; streams emit a timestep every 4th tick (action repeat 4), long episodes.

  python tools/bench_train.py [--frames 16384] [--streams 1,32,128,256] [--agents dqn,rainbow] [--repeats 2]"""

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
RAW = (210, 160, 3)
LEARN_PERIOD = 16


def emit(**kw):
  print(json.dumps(kw), flush=True)


def device_info():
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm,clocks.sm', '--format=csv,noheader'],
                       capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
  except (OSError, subprocess.SubprocessError, IndexError):
    q = 'unavailable'
  return {'name': torch.cuda.get_device_name(0), 'power_limit_max_sm_clock_sm_clock': q}


def make_agent(kind, capacity):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  structure = dr.Transition(None, None, None, None, None)
  rs = np.random.RandomState(1)
  if kind == 'rainbow':
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.5, lambda t: 0.4, 1e-3, True, rs, frame_dedup=True)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, frame_dedup=True)
  dr.bulk_fill_synthetic_stacked(rep, OBS, 1, 6, episode_len=1000)
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(3 if kind == 'rainbow' else 1), replay=rep,
                batch_size=32, min_replay_capacity_fraction=0.05, learn_period=LEARN_PERIOD,
                target_network_update_period=40000, rng_key=[0, 7])
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common)
  return ag.Dqn(exploration_epsilon=lambda t: 0.01, grad_error_bound=1.0 / 32, **common)


def learner_only_steps_per_sec(agent, steps):
  for _ in range(20):
    agent.learn()
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(steps):
    agent.learn()
  torch.cuda.synchronize()
  return steps / (time.perf_counter() - t0)


def bench(kind, E, frames_target, capacity, repeats):
  from dqn_zoo_b200 import agent as ag
  agent = make_agent(kind, capacity)
  trainer = ag.VectorTrainer(agent, num_streams=E, rng_key=[0, 3])
  rs = np.random.RandomState(0)
  pool = [torch.as_tensor(rs.randint(0, 256, (E,) + RAW).astype(np.uint8), device='cuda') for _ in range(8)]
  mid, first = np.ones(E, np.int64), np.zeros(E, np.int64)
  zeros, ones, nan, lives = np.zeros(E), np.ones(E), np.full(E, np.nan), np.full(E, 3)
  tick = 0

  def run(n):
    nonlocal tick
    for _ in range(n):
      if tick == 0:
        trainer.step(pool[0], first, nan, nan, lives)
      else:
        trainer.step(pool[tick % 8], mid, zeros, ones, lives)
      tick += 1

  run(max(64, 4 * LEARN_PERIOD // E + 8))             # warm-up: every tick shape, the graph capture
  torch.cuda.synchronize()
  ticks = max(100, frames_target // E)
  for r in range(repeats):
    steps0 = trainer.learn_steps
    t0 = time.perf_counter()
    run(ticks)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    graph = learner_only_steps_per_sec(agent, 400)
    emit(metric='train_frames_per_sec', agent=kind, streams=E, repeat=r, value=round(ticks * E / dt, 1),
         learner_steps_per_sec=round((trainer.learn_steps - steps0) / dt, 1),
         learner_only_frames_per_sec=round(LEARN_PERIOD * graph, 1), graph_steps_per_sec=round(graph, 1),
         ticks=ticks, learn_period=LEARN_PERIOD, batch=32, capacity=capacity)
  del trainer, agent, pool
  torch.cuda.empty_cache()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--frames', type=int, default=16384, help='frames per timed window (at least 100 ticks)')
  ap.add_argument('--streams', default='1,32,128,256')
  ap.add_argument('--agents', default='dqn,rainbow')
  ap.add_argument('--capacity', type=int, default=100000)
  ap.add_argument('--repeats', type=int, default=2)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_train.py needs a CUDA device')
  torch.cuda.set_device(0)
  emit(metric='device', **device_info())
  for kind in a.agents.split(','):
    for E in (int(s) for s in a.streams.split(',')):
      bench(kind, E, a.frames, a.capacity, a.repeats)
  emit(metric='device_after', **device_info())


if __name__ == '__main__':
  main()
