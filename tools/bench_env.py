"""A device game (`--game catch`: `environments.VectorCatch`, DESIGN.md §10, the default; `--game breakout`:
`environments.VectorBreakout`, §11; `--game pong`: `environments.VectorPong`, §12) alone and in the loop.  One JSON line
per point (with `--game breakout` or `pong` each carries `game`):

  * env_step: E in {32, 256, 1024}.  device_us_per_tick: CUDA events around back-to-back ticks (actions copy, kernel,
    record copy) without host synchronisation; store_GBps: the E x 100,800 frame bytes a tick writes over that time;
    frames_per_sec: E over the host time of a full `step` (which synchronises once);
  * env_train / env_eval: E in {32, 256}, `VectorCatch.step` + `VectorTrainer.step` (dqn, rainbow; replay prefilled so
    the learner runs every 16 frames) or + `VectorEvaluator.step`, frames per second over the host clock, beside
    bench_train.py / bench_eval.py's device-pool figures;
  * driver: `tools/run_synthetic.py --env <game> --num_streams 64 --num_eval_streams 64`, with and without
    `--overlap_eval`, wall time of the whole run;
  * learning (`--learning FRAMES`): the learning curve of the GPU learning tests (tests/test_gpu_catch.py,
    tests/test_gpu_breakout.py, tests/test_gpu_pong.py): `--agent` (dqn; also rainbow), E = 32, evaluated with epsilon 0.01 on 64 streams every
    `--eval_every` frames (`evaluate` says what an evaluation episode is).

The card's name and power limit are read in the same run.

  python tools/bench_env.py [--game catch] [--parts env,train,eval,driver] [--learning 0] [--agent dqn]"""

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
# Breakout evaluation: episodes are truncated at this many frames, and every stream plays one frame more than that, so
# each completes at least one episode (a good policy can keep the ball alive far longer).
BREAKOUT_EVAL_FRAMES = 4500
# Pong evaluation, the same way: a game of a random policy lasts about 2,000 frames, and one whose rallies go on can
# last far longer.
PONG_EVAL_FRAMES = 6000


def make_env(game, num_streams, seed, num_actions=6):
  """`VectorCatch`, `VectorBreakout` (whose actions 4.. do nothing, so 6-action agents drive it) or `VectorPong`."""
  from dqn_zoo_b200 import environments
  if game == 'breakout':
    return environments.VectorBreakout(num_streams, seed, num_actions=num_actions)
  if game == 'pong':
    return environments.VectorPong(num_streams, seed, num_actions=num_actions)
  return environments.VectorCatch(num_streams, seed, num_actions=num_actions)


def _tag(game):
  return {} if game == 'catch' else {'game': game}


def emit(**kw):
  print(json.dumps(kw), flush=True)


def bench_env_step(E, ticks=400, game='catch'):
  import ctypes as C
  from dqn_zoo_b200 import _lib
  env = make_env(game, E, seed=1)
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
    _lib.call(env._STEP, *args, s.cuda_stream)
  end.record()
  end.synchronize()
  device_s = start.elapsed_time(end) / 1e3 / ticks
  actions = [rs.randint(0, 6, E) for _ in range(16)]
  t0 = time.perf_counter()
  for t in range(ticks):
    env.step(actions[t % 16])
  host_s = (time.perf_counter() - t0) / ticks
  emit(metric='env_step', **_tag(game), streams=E, device_us_per_tick=round(device_s * 1e6, 2),
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


def bench_env_agent(what, kind, E, frames_target, repeats=2, game='catch'):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  env = make_env(game, E, seed=2)
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
    emit(metric='env_' + what, **_tag(game), agent=kind, streams=E, repeat=r, frames_per_sec=round(ticks * E / dt, 1), ticks=ticks)


def bench_driver(game='catch'):
  import run_synthetic
  base = ['--env', game, '--num_streams', '64', '--num_eval_streams', '64', '--num_iterations', '2',
          '--num_train_frames', '65536', '--num_eval_frames', '32768', '--replay_capacity', '20000',
          '--min_replay_capacity_fraction', '0.05']
  for overlap in (False, True, False, True):
    argv = base + (['--overlap_eval'] if overlap else [])
    t0 = time.perf_counter()
    rows = run_synthetic.run(run_synthetic.parse_args(argv))
    dt = time.perf_counter() - t0
    emit(metric='driver', **_tag(game), overlap_eval=overlap, wall_s=round(dt, 2),
         train_frame_rate=[round(r['train_frame_rate'], 1) for r in rows],
         eval_frame_rate=[round(r['eval_frame_rate'], 1) for r in rows])


# -- learning ----------------------------------------------------------------------------------------------------------
def learning_agent(seed, train_frames, kind='dqn', num_actions=6, dueling=False, noisy=False, random_shift_pad=0,
                   prioritized=False, n_step=None):
  """dqn at the reference's hyper-parameters but for a faster schedule: replay of 100k transitions, learning from 10k,
  epsilon 1 -> 0.01 over the first quarter of the frames, target sync every 8000 frames.  `kind='rainbow'`: the same
  schedule with rainbow's prioritized replay (exponent 0.5, importance exponent 0.4 -> 1 over the run), 3-step returns,
  noisy greedy acting and its 51-atom support on [-10, 10].  `kind='double_q'`: dqn's schedule with the double Q-learning
  target.  `dueling`: the dueling network (DESIGN.md §16) in place of dqn's fc1 / head.  `noisy`: noisy networks
  (DESIGN.md §17) with an epsilon schedule that is zero throughout, so that the agent explores through its noise alone
  (NoisyNet-DQN for dqn).  `random_shift_pad`: random-shift augmentation of every learner step (DESIGN.md §18); with
  kind='double_q' and `dueling` that is DrQ-epsilon's agent on this schedule.  `prioritized`: any kind on rainbow's
  prioritized replay (DESIGN.md §19).  `n_step`: the returns' step count (None: 3 for rainbow, 1 otherwise)."""
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  capacity, min_fill = 100000, 10000
  structure = dr.Transition(None, None, None, None, None)
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, num_actions, dueling=dueling,
                                                                                          noisy=noisy),
                optimizer=None, batch_size=32, min_replay_capacity_fraction=min_fill / capacity, learn_period=16,
                target_network_update_period=8000, rng_key=[0, seed + 1], random_shift_pad=random_shift_pad)
  n = dr.NStepTransitionAccumulator(n_step or (3 if kind == 'rainbow' else 1))
  if kind == 'rainbow' or prioritized:
    importance = parts.LinearSchedule(begin_t=min_fill, decay_steps=max(train_frames, 1), begin_value=0.4,
                                      end_value=1.0)
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.5, importance, 1e-3, True, rs, frame_dedup=True)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, frame_dedup=True)
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), transition_accumulator=n, replay=rep, **common)
  epsilon = parts.LinearSchedule(begin_t=4 * min_fill, decay_steps=max(train_frames // 4, 1), begin_value=1.0,
                                 end_value=0.01)
  if noisy:
    epsilon = lambda t: 0.0
  if kind == 'fqf':   # dqn's schedule, 32 fractions, kappa 1 and the fraction layer's default RMSProp
    return ag.Fqf(transition_accumulator=n, replay=rep, exploration_epsilon=epsilon,
                  huber_param=1.0, **common)
  if dl.uses_iqn_network(kind):   # iqn / munchausen_iqn: dqn's schedule, iqn's 64 / 64 / 64 taus and kappa 1
    return ag.AGENTS[kind](transition_accumulator=n, replay=rep, exploration_epsilon=epsilon, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                           tau_samples_s_t=64, **common)
  if kind == 'c51':   # dqn's schedule, 51 atoms on [-10, 10]
    return ag.C51(support=np.linspace(-10, 10, 51), transition_accumulator=n, replay=rep, exploration_epsilon=epsilon,
                  **common)
  if kind == 'qrdqn':   # dqn's schedule, 201 quantiles, kappa 1
    return ag.QrDqn(quantiles=(np.arange(201) + 0.5) / 201, transition_accumulator=n, replay=rep,
                    exploration_epsilon=epsilon, huber_param=1.0, **common)
  # munchausen: dqn's schedule, the paper's alpha / tau / l0; double_q: dqn's schedule
  agent_cls = {'munchausen': ag.Munchausen, 'double_q': ag.DoubleQ}.get(kind, ag.Dqn)
  return agent_cls(transition_accumulator=n, replay=rep, exploration_epsilon=epsilon, grad_error_bound=1.0 / 32,
                   **common)


def evaluate(learner, seed, num_streams=64, game='catch', num_actions=6):
  """Mean return of the episodes that `num_streams` streams complete at epsilon 0.01, and their number.  Catch: 1,900
  ticks, no truncation (every stream completes at least one episode: one is at most 20 x 91 + 30 frames).  Breakout:
  an episode runs from its FIRST step to its LAST step or to its BREAKOUT_EVAL_FRAMES-th frame, where it is
  truncated; every stream plays BREAKOUT_EVAL_FRAMES + 1 ticks, so it completes at least one, and the episodes still
  running at the end are not counted.  Pong: the same with PONG_EVAL_FRAMES."""
  import run_synthetic
  from dqn_zoo_b200 import agent as ag
  ev = ag.VectorEvaluator(learner, num_streams, 0.01, [0, seed + 2])
  ev.network_params = learner
  env = make_env(game, num_streams, seed + 3, num_actions)
  if game in ('breakout', 'pong'):
    limit = BREAKOUT_EVAL_FRAMES if game == 'breakout' else PONG_EVAL_FRAMES
    loop = run_synthetic.StreamLoop(ev, env, (limit + 1) * num_streams, limit)
  else:
    loop = run_synthetic.StreamLoop(ev, env, 1900 * num_streams, 0)
  stats = loop.run()
  return stats['episode_return'], stats['num_episodes']


def learning_run(train_frames, seed=0, num_streams=32, eval_every=0, log=None, game='catch', num_actions=6,
                 kind='dqn', dueling=False, noisy=False, random_shift_pad=0, prioritized=False, n_step=None):
  """Trains `learning_agent` (of `kind`, on the dueling network with `dueling`, with noisy layers with `noisy`) from `num_streams` streams of `game` for `train_frames` frames (training episodes are not
  truncated); evaluates every `eval_every` frames (0: at the end only).  Returns [(frames, mean eval return, eval
  episodes, train episode return)]."""
  import run_synthetic
  from dqn_zoo_b200 import agent as ag
  agent = learning_agent(seed, train_frames, kind, num_actions, dueling, noisy, random_shift_pad, prioritized, n_step)
  trainer = ag.VectorTrainer(agent, num_streams=num_streams, rng_key=[0, seed + 4])
  env = make_env(game, num_streams, seed + 5, num_actions)
  loop = run_synthetic.StreamLoop(trainer, env, train_frames, 0)
  curve = []
  every = max(eval_every // num_streams, 1) if eval_every else None
  while not loop.done:
    loop.tick()
    if (every and loop._tick % every == 0) or loop.done:
      ret, n = evaluate(agent.learner, seed, game=game, num_actions=num_actions)
      curve.append((loop._tick * num_streams, ret, n, loop.stats()['episode_return']))
      if log:
        log(frames=curve[-1][0], eval_return=round(ret, 3), eval_episodes=n, train_return=round(curve[-1][3], 3))
  return curve


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--game', default='catch', choices=['catch', 'breakout', 'pong'])
  ap.add_argument('--agent', default='dqn', choices=['dqn', 'double_q', 'c51', 'qrdqn', 'rainbow', 'munchausen', 'iqn',
                                                       'munchausen_iqn', 'fqf'],
                  help='the agent of the learning curve')
  ap.add_argument('--dueling', action='store_true', help='the learning curve on the dueling network (DESIGN.md §16)')
  ap.add_argument('--noisy', action='store_true',
                  help='the learning curve on noisy networks with a zero epsilon schedule (DESIGN.md §17)')
  ap.add_argument('--random_shift_pad', type=int, default=0,
                  help='the learning curve with random-shift augmentation at pad N (DESIGN.md §18)')
  ap.add_argument('--prioritized', action='store_true',
                  help='the learning curve on rainbow\'s prioritized replay, for any agent (DESIGN.md §19)')
  ap.add_argument('--n_step', type=int, default=None, help='the returns\' step count (default: 3 for rainbow, else 1)')
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
      bench_env_step(E, game=a.game)
  for what in ('train', 'eval'):
    if what in parts:
      for kind in ('dqn', 'rainbow'):
        for E in (32, 256):
          bench_env_agent(what, kind, E, a.frames, game=a.game)
  if 'driver' in parts:
    bench_driver(a.game)
  if a.learning:
    t0 = time.perf_counter()
    learning_run(a.learning, a.seed, eval_every=a.eval_every, game=a.game, kind=a.agent, dueling=a.dueling,
                 noisy=a.noisy, random_shift_pad=a.random_shift_pad, prioritized=a.prioritized, n_step=a.n_step, log=lambda **kw: emit(metric='learning', **_tag(a.game), **({} if a.agent == 'dqn' else
                                                                              {'agent': a.agent}),
                                       **({'dueling': True} if a.dueling else {}),
                                       **({'noisy': True} if a.noisy else {}),
                                       **({'random_shift_pad': a.random_shift_pad} if a.random_shift_pad else {}),
                                       **({'prioritized': True} if a.prioritized else {}),
                                       **({'n_step': a.n_step} if a.n_step else {}),
                                       seed=a.seed, wall_s=round(time.perf_counter() - t0, 1), **kw))
  emit(metric='device_after', **bench_train.device_info())


if __name__ == '__main__':
  main()
