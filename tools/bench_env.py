"""The device Catch environment (`environments.VectorCatch`, DESIGN.md §10) alone and in the loop.  One JSON line per
point:

  * env_step: E in {32, 256, 1024}.  device_us_per_tick: CUDA events around back-to-back ticks (actions copy, kernel,
    record copy) without host synchronisation; store_GBps: the E x 100,800 frame bytes a tick writes over that time;
    frames_per_sec: E over the host time of a full `step` (which synchronises once);
  * env_train / env_eval: E in {32, 256}, `VectorCatch.step` + `VectorTrainer.step` (dqn, rainbow; replay prefilled so
    the learner runs every 16 frames) or + `VectorEvaluator.step`, frames per second over the host clock, beside
    bench_train.py / bench_eval.py's device-pool figures;
  * driver: `tools/run_synthetic.py --env catch --num_streams 64 --num_eval_streams 64`, with and without
    `--overlap_eval`, wall time of the whole run;
  * learning (`--learning FRAMES`): the learning curve of the GPU learning test (tests/test_gpu_catch.py): dqn, E = 32,
    evaluated with epsilon 0.01 on 64 streams every `--eval_every` frames.

The card's name and power limit are read in the same run.

  python tools/bench_env.py [--parts env,train,eval,driver] [--learning 0]"""

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench_train  # noqa: E402

FRAME_BYTES = 210 * 160 * 3


def emit(**kw):
  print(json.dumps(kw), flush=True)


def bench_env_step(E, ticks=400):
  import ctypes as C
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import environments
  env = environments.VectorCatch(E, seed=1)
  env.reset()
  rs = np.random.RandomState(0)
  for _ in range(20):
    env.step(rs.randint(0, 6, E))
  args = (C.byref(env._cfg), env._state.data_ptr(), env._control_host.data_ptr(), env._control.data_ptr(),
          env._frames.data_ptr(), env._record.data_ptr(), env._record_host.data_ptr())
  s = torch.cuda.current_stream()
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(ticks):
    _lib.call('dz_catch_step', *args, s.cuda_stream)
  end.record()
  end.synchronize()
  device_s = start.elapsed_time(end) / 1e3 / ticks
  actions = [rs.randint(0, 6, E) for _ in range(16)]
  t0 = time.perf_counter()
  for t in range(ticks):
    env.step(actions[t % 16])
  host_s = (time.perf_counter() - t0) / ticks
  emit(metric='env_step', streams=E, device_us_per_tick=round(device_s * 1e6, 2),
       store_GBps=round(E * FRAME_BYTES / device_s / 1e9, 1), frames_per_sec=round(E / host_s, 1),
       host_us_per_step=round(host_s * 1e6, 2), ticks=ticks)


def _loop(agent, env, ticks):
  from dqn_zoo_b200 import parts
  frames, st, rw, dc, lv = env.reset()
  agent.reset()
  for _ in range(ticks):
    actions = agent.step(frames, st, rw, dc, lv)
    last = st == int(parts.StepType.LAST)
    if last.any():
      agent.reset(np.nonzero(last)[0])
    frames, st, rw, dc, lv = env.step(actions, reset=last)


def bench_env_agent(what, kind, E, frames_target, repeats=2):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  from dqn_zoo_b200 import learner as dl
  env = environments.VectorCatch(E, seed=2)
  if what == 'train':
    agent = bench_train.make_agent(kind, 100000)
    runner = ag.VectorTrainer(agent, num_streams=E, rng_key=[0, 3])
  else:
    learner = dl.Learner(dl.NetworkSpec(kind, 6))
    runner = ag.VectorEvaluator(learner, E, 0.01, [0, 3])
    runner.network_params = learner
  _loop(runner, env, max(64, 72 // E + 8))             # warm-up: every tick shape, the graph capture
  torch.cuda.synchronize()
  ticks = max(100, frames_target // E)
  for r in range(repeats):
    t0 = time.perf_counter()
    _loop(runner, env, ticks)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    emit(metric='env_' + what, agent=kind, streams=E, repeat=r, frames_per_sec=round(ticks * E / dt, 1), ticks=ticks)


def bench_driver():
  import run_synthetic
  base = ['--env', 'catch', '--num_streams', '64', '--num_eval_streams', '64', '--num_iterations', '2',
          '--num_train_frames', '65536', '--num_eval_frames', '32768', '--replay_capacity', '20000',
          '--min_replay_capacity_fraction', '0.05']
  for overlap in (False, True, False, True):
    argv = base + (['--overlap_eval'] if overlap else [])
    t0 = time.perf_counter()
    rows = run_synthetic.run(run_synthetic.parse_args(argv))
    dt = time.perf_counter() - t0
    emit(metric='driver', overlap_eval=overlap, wall_s=round(dt, 2),
         train_frame_rate=[round(r['train_frame_rate'], 1) for r in rows],
         eval_frame_rate=[round(r['eval_frame_rate'], 1) for r in rows])


# -- learning ----------------------------------------------------------------------------------------------------------
def learning_agent(seed, train_frames):
  """dqn at the reference's hyper-parameters but for a faster schedule: replay of 100k transitions, learning from 10k,
  epsilon 1 -> 0.01 over the first quarter of the frames, target sync every 8000 frames."""
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  capacity, min_fill = 100000, 10000
  rep = dr.TransitionReplay(capacity, dr.Transition(None, None, None, None, None), rs, frame_dedup=True)
  epsilon = parts.LinearSchedule(begin_t=4 * min_fill, decay_steps=max(train_frames // 4, 1), begin_value=1.0,
                                 end_value=0.01)
  return ag.Dqn(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec('dqn', 6), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=min_fill / capacity, learn_period=16, target_network_update_period=8000,
                rng_key=[0, seed + 1], exploration_epsilon=epsilon, grad_error_bound=1.0 / 32)


def evaluate(learner, seed, num_streams=64):
  """Mean return of the episodes that `num_streams` Catch streams complete in 1,900 ticks (every stream completes at
  least one: an episode is at most 20 x 91 + 30 frames) at epsilon 0.01, and their number."""
  import run_synthetic
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  ev = ag.VectorEvaluator(learner, num_streams, 0.01, [0, seed + 2])
  ev.network_params = learner
  env = environments.VectorCatch(num_streams, seed + 3)
  stats = run_synthetic.StreamLoop(ev, env, 1900 * num_streams, 0).run()
  return stats['episode_return'], stats['num_episodes']


def learning_run(train_frames, seed=0, num_streams=32, eval_every=0, log=None):
  """Trains `learning_agent` from `num_streams` Catch streams for `train_frames` frames; evaluates every `eval_every`
  frames (0: at the end only).  Returns [(frames, mean eval return, eval episodes, train episode return)]."""
  import run_synthetic
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  agent = learning_agent(seed, train_frames)
  trainer = ag.VectorTrainer(agent, num_streams=num_streams, rng_key=[0, seed + 4])
  env = environments.VectorCatch(num_streams, seed + 5)
  loop = run_synthetic.StreamLoop(trainer, env, train_frames, 0)
  curve = []
  every = max(eval_every // num_streams, 1) if eval_every else None
  while not loop.done:
    loop.tick()
    if (every and loop._tick % every == 0) or loop.done:
      ret, n = evaluate(agent.learner, seed)
      curve.append((loop._tick * num_streams, ret, n, loop.stats()['episode_return']))
      if log:
        log(frames=curve[-1][0], eval_return=round(ret, 3), eval_episodes=n, train_return=round(curve[-1][3], 3))
  return curve


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parts', default='env,train,eval,driver')
  ap.add_argument('--frames', type=int, default=65536, help='frames per timed window of env_train / env_eval')
  ap.add_argument('--learning', type=int, default=0, help='frames of the learning curve (0: none)')
  ap.add_argument('--eval_every', type=int, default=200000)
  ap.add_argument('--seed', type=int, default=0)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bench_env.py needs a CUDA device')
  torch.cuda.set_device(0)
  emit(metric='device', **bench_train.device_info())
  parts = a.parts.split(',') if a.parts else []
  if 'env' in parts:
    for E in (32, 256, 1024):
      bench_env_step(E)
  for what in ('train', 'eval'):
    if what in parts:
      for kind in ('dqn', 'rainbow'):
        for E in (32, 256):
          bench_env_agent(what, kind, E, a.frames)
  if 'driver' in parts:
    bench_driver()
  if a.learning:
    t0 = time.perf_counter()
    learning_run(a.learning, a.seed, eval_every=a.eval_every,
                 log=lambda **kw: emit(metric='learning', seed=a.seed, wall_s=round(time.perf_counter() - t0, 1), **kw))
  emit(metric='device_after', **bench_train.device_info())


if __name__ == '__main__':
  main()
