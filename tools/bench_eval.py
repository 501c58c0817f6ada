"""Measures the evaluation phase on many streams (`agent.VectorEvaluator` over a frozen acting context):

  (a) evaluation frames/s of the evaluator tick at E streams, against one `EpsilonGreedyActor` step per frame (the
      one-stream evaluation path of the run drivers); both read raw frames from a pool already in memory, so no
      environment is timed;
  (b) GPU time per act of a frozen actor against a live one at E streams (the live actor packs the conv weight images
      on every act, the frozen one once per snapshot);
  (c) wall time of `tools/run_synthetic.py`'s train-then-evaluate iterations against `--overlap_eval`.

The compared modes alternate within one process, `--repeats` times.  Prints one JSON line per measurement, the first
with the GPU's power limit and SM clocks.

  python tools/bench_eval.py --agents dqn rainbow iqn --streams 1 32 128 256
"""
import argparse
import json
import os
import subprocess
import sys
import timeit

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

RAW = (210, 160, 3)


def gpu_info():
  try:
    out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                         capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    out = ''
  return {'gpu': torch.cuda.get_device_name(0), 'nvidia_smi': out}


def script(E, ticks, episode=400):
  """step types of E streams: FIRST at tick 0, LAST every `episode` ticks (staggered), then FIRST again."""
  st = np.ones((ticks, E), np.int64)
  for e in range(E):
    t = 0
    while t < ticks:
      st[t, e] = 0
      end = t + episode - (e * 37) % (episode // 2)
      if end < ticks:
        st[end, e] = 2
      t = end + 1
  reward = np.where(st == 0, np.nan, 1.0)
  discount = np.where(st == 0, np.nan, np.where(st == 2, 0.0, 1.0))
  return st, reward, discount


def eval_rate(kind, E, ticks, warmup):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  net = dl.NetworkSpec(kind, 6)
  L = dl.Learner(net)
  L.init_params(1)
  ev = ag.VectorEvaluator(L, E, 0.01, rng_key=[0, 3])
  ev.network_params = L
  rs = np.random.RandomState(0)
  pool = [torch.as_tensor(rs.randint(0, 256, (E,) + RAW).astype(np.uint8), device='cuda') for _ in range(4)]
  st, rw, dc = script(E, warmup + ticks)
  lives = np.full(E, 3)
  t0 = None
  for t in range(warmup + ticks):
    if t == warmup:
      torch.cuda.synchronize()
      t0 = timeit.default_timer()
    ev.step(pool[t % 4], st[t], rw[t], dc[t], lives)
    last = np.nonzero(st[t] == 2)[0]
    if last.size:
      ev.reset(last)
  torch.cuda.synchronize()
  return E * ticks / (timeit.default_timer() - t0)


def single_rate(kind, frames, warmup):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import processors
  net = dl.NetworkSpec(kind, 6)
  L = dl.Learner(net)
  L.init_params(1)
  actor = ag.EpsilonGreedyActor(processors.atari(device_observations=True), net, 0.01, rng_key=[0, 3])
  actor.network_params = L
  rs = np.random.RandomState(0)
  pool = [rs.randint(0, 256, RAW).astype(np.uint8) for _ in range(4)]
  st, rw, dc = script(1, warmup + frames)
  t0 = None
  for t in range(warmup + frames):
    if t == warmup:
      torch.cuda.synchronize()
      t0 = timeit.default_timer()
    s = int(st[t, 0])
    ts = parts.TimeStep(parts.StepType(s), None if s == 0 else float(rw[t, 0]), None if s == 0 else float(dc[t, 0]),
                        (pool[t % 4], 3))
    actor.step(ts)
    if s == 2:
      actor.reset()
  torch.cuda.synchronize()
  return frames / (timeit.default_timer() - t0)


def act_time(kind, E, acts, frozen):
  from dqn_zoo_b200 import learner as dl
  net = dl.NetworkSpec(kind, 6)
  L = dl.Learner(net)
  L.init_params(1)
  actor = L.actor(E, frozen=frozen)
  if frozen:
    actor.load_params(L)
  obs = torch.randint(0, 256, (E, 84, 84, 4), dtype=torch.uint8, device='cuda')
  kw = {}
  if dl.uses_iqn_network(kind):
    kw['taus'] = actor.generate_randomness(1)
  elif kind == 'rainbow':
    kw['noise'] = actor.generate_randomness(1)
  for _ in range(5):
    actor.act(obs, **kw)
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(acts):
    actor.act(obs, **kw)
  end.record()
  end.synchronize()
  return 1000.0 * start.elapsed_time(end) / acts    # us per act


def iteration_time(kind, overlap, train_streams, eval_streams):
  import run_synthetic
  argv = ['--agent', kind, '--num_streams', str(train_streams), '--num_eval_streams', str(eval_streams),
          '--num_iterations', '2', '--num_train_frames', '20000', '--num_eval_frames', '10000', '--replay_capacity', '20000',
          '--min_replay_capacity_fraction', '0.05', '--max_frames_per_episode', '2000']
  if overlap:
    argv.append('--overlap_eval')
  t0 = timeit.default_timer()
  rows = run_synthetic.run(run_synthetic.parse_args(argv))
  return timeit.default_timer() - t0, rows


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--agents', nargs='+', default=['dqn', 'rainbow', 'iqn'])
  ap.add_argument('--streams', nargs='+', type=int, default=[1, 32, 128, 256])
  ap.add_argument('--frames', type=int, default=20000, help='evaluated frames per rate measurement')
  ap.add_argument('--repeats', type=int, default=2)
  ap.add_argument('--parts', default='abc')
  args = ap.parse_args()
  print(json.dumps(gpu_info()), flush=True)
  for _ in range(args.repeats):
    if 'a' in args.parts:
      for kind in args.agents:
        single = single_rate(kind, min(args.frames, 3000), 200)
        print(json.dumps({'part': 'a', 'agent': kind, 'mode': 'EpsilonGreedyActor+run_loop', 'E': 1,
                          'frames_per_s': round(single, 1)}), flush=True)
        for E in args.streams:
          ticks = max(args.frames // E, 50)
          rate = eval_rate(kind, E, ticks, 20)
          print(json.dumps({'part': 'a', 'agent': kind, 'mode': 'VectorEvaluator', 'E': E, 'frames_per_s': round(rate, 1)}),
                flush=True)
    if 'b' in args.parts:
      for kind in args.agents:
        for E in (32, 256):
          for frozen in (False, True):
            us = act_time(kind, E, 200, frozen)
            print(json.dumps({'part': 'b', 'agent': kind, 'E': E, 'actor': 'frozen' if frozen else 'live',
                              'us_per_act': round(us, 2)}), flush=True)
    if 'c' in args.parts:
      for kind in ('dqn',):
        for overlap in (False, True):
          wall, rows = iteration_time(kind, overlap, 64, 64)
          print(json.dumps({'part': 'c', 'agent': kind, 'overlap_eval': overlap, 'wall_s': round(wall, 2),
                            'eval_frame_rate': [round(r['eval_frame_rate'], 1) for r in rows],
                            'train_frame_rate': [round(r['train_frame_rate'], 1) for r in rows]}), flush=True)


if __name__ == '__main__':
  main()
