"""A run driver with the structure of the reference's `<agent>/run_atari.py` (dqn/run_atari.py:98-290) on a SYNTHETIC
Atari-shaped environment (no ALE/ROMs in this image): raw 210x160x3 frames + lives -> device preprocessing
(`processors.atari`, frame stacks stay in HBM) -> agent.step (act / insert / fused learner step) -> trackers ->
evaluation actor with the online parameters -> CSV row (`dqn_zoo_plots.ipynb` column names, minus the human-normalised
score which needs real game scores) -> checkpoint.  It exists to show how the pieces replace the reference's; the same
sequence of calls is what tests/test_gpu_agent.py::test_train_eval_iteration_with_trackers_actor_and_checkpoint checks.

  python tools/run_synthetic.py --agent rainbow --num_iterations 3 --num_train_frames 2000 --num_eval_frames 500 \
      --results_csv_path /tmp/results.csv --checkpoint_path /tmp/ck.pkl

`--num_streams E` (E > 1) trains from E environments at once through `agent.VectorTrainer`: each tick stages the E raw
frames in pinned memory, sends them to the device in one copy and makes one trainer step; `--num_train_frames` then
counts the frames of all streams.

`--num_eval_streams E` evaluates on E environments of their own through `agent.VectorEvaluator` (a frozen parameter
snapshot taken after each training phase); `--num_eval_frames` then counts the frames of all evaluation streams.  Both
phases share `StreamLoop`'s truncation and episode bookkeeping.  `--overlap_eval` (with `--num_streams` > 1) runs
iteration i's evaluation on its own CUDA stream, one tick after each training tick of iteration i + 1; every column of
the CSV rows but the rates is as without it.  CSV columns and checkpoints are otherwise as with one stream.

`--env catch` plays Catch (`dqn_zoo_b200.environments`, DESIGN.md §10) instead of the synthetic frames: a game that is
simulated and rendered on the device, so its returns measure learning.  With E > 1 streams each phase steps one
`VectorCatch` whose frames tensor goes to the trainer or evaluator as it is, with no host staging; with one stream the
phases play `Catch` through `parts.run_loop`.  `--env breakout` does the same with the device Breakout (DESIGN.md §11;
`VectorBreakout` / `Breakout`, `--num_actions` in [4, 18]).  Breakout has no frame limit of its own:
`--max_frames_per_episode` truncates its episodes.  `--env pong` plays the device Pong against a scripted opponent
(DESIGN.md §12; `VectorPong` / `Pong`, `--num_actions` in [6, 18]), which has no frame limit either.

`--checkpoint_dir D --background_checkpoint` ends each iteration with `DirectoryCheckpoint.save(blocking=False)`: the
agent and its replay are snapshotted in device memory and the generation is written by a background thread while the
next iteration trains (DESIGN.md §9); the run waits for the last write before it returns.  The rows are those of the
blocking saves.
"""
import argparse
import collections
import itertools
import math
import os
import sys
import timeit

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402


class SyntheticAtari:
  """Random RGB frames with Atari's geometry; episodes of random length; a life is lost now and then."""

  def __init__(self, seed, num_actions=6, height=210, width=160):
    self._rs = np.random.RandomState(seed)
    self._shape = (height, width, 3)
    self.num_actions = num_actions
    self._left = 0
    self._lives = 3

  def _observation(self):
    return self._rs.randint(0, 256, size=self._shape, dtype=np.uint8), self._lives

  def reset(self):
    from dqn_zoo_b200 import parts
    self._left = int(self._rs.randint(200, 800))
    self._lives = 3
    return parts.TimeStep(parts.StepType.FIRST, None, None, self._observation())

  def step(self, action):
    from dqn_zoo_b200 import parts
    del action
    self._left -= 1
    if self._rs.uniform() < 0.002 and self._lives > 1:
      self._lives -= 1
    last = self._left <= 0
    reward = float(self._rs.choice([0.0, 0.0, 0.0, 1.0, -1.0]))
    return parts.TimeStep(parts.StepType.LAST if last else parts.StepType.MID, reward, 0.0 if last else 1.0,
                          self._observation())


def build_train_agent(args, random_state, preprocessor):
  from dqn_zoo_b200 import agent as agent_lib
  from dqn_zoo_b200 import learner as learner_lib
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import replay as replay_lib
  kind = args.agent
  prioritized = kind in ('prioritized', 'rainbow') or args.prioritized
  n_step = 3 if kind == 'rainbow' else 1
  structure = replay_lib.Transition(None, None, None, None, None)
  if prioritized:
    schedule = parts.LinearSchedule(begin_t=int(args.min_replay_capacity_fraction * args.replay_capacity),
                                    decay_steps=max(args.num_iterations * args.num_train_frames // 4, 1), begin_value=0.4,
                                    end_value=1.0)
    replay = replay_lib.PrioritizedTransitionReplay(args.replay_capacity, structure, 0.6 if kind == 'prioritized' else 0.5, schedule,
                                                    1e-3, True, random_state)
  else:
    replay = replay_lib.TransitionReplay(args.replay_capacity, structure, random_state)
  network = learner_lib.NetworkSpec(kind, args.num_actions, dueling=args.dueling, noisy=args.noisy)
  epsilon = parts.LinearSchedule(begin_t=int(args.min_replay_capacity_fraction * args.replay_capacity * 4),
                                 decay_steps=max(args.num_train_frames, 1), begin_value=1.0, end_value=0.01)
  if args.noisy:   # noisy networks explore through their noise: a zero schedule (NoisyNet-DQN for dqn)
    epsilon = lambda t: 0.0
  common = dict(preprocessor=preprocessor, sample_network_input=np.zeros((84, 84, 4), np.uint8), network=network, optimizer=None,
                transition_accumulator=replay_lib.NStepTransitionAccumulator(n_step), replay=replay, batch_size=32,
                min_replay_capacity_fraction=args.min_replay_capacity_fraction, learn_period=16,
                target_network_update_period=args.target_network_update_period,
                rng_key=[0, int(random_state.randint(1, 2 ** 31))], random_shift_pad=args.random_shift_pad)
  if kind == 'rainbow':
    return agent_lib.Rainbow(support=np.linspace(-10, 10, 51), **common), network
  if kind == 'c51':
    return agent_lib.C51(support=np.linspace(-10, 10, 51), exploration_epsilon=epsilon, **common), network
  if kind == 'qrdqn':
    return agent_lib.QrDqn(quantiles=(np.arange(201) + 0.5) / 201, exploration_epsilon=epsilon, huber_param=1.0, **common), network
  if kind == 'fqf':
    return agent_lib.Fqf(exploration_epsilon=epsilon, huber_param=1.0, **common), network
  if learner_lib.uses_iqn_network(kind):
    return agent_lib.AGENTS[kind](exploration_epsilon=epsilon, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                         tau_samples_s_t=64, **common), network
  return agent_lib.AGENTS[kind](exploration_epsilon=epsilon, grad_error_bound=1.0 / 32, **common), network


class StreamLoop:
  """E environments stepped through a vectorised agent (`agent.VectorTrainer` or `agent.VectorEvaluator`) for
  `num_frames` frames (rounded up to whole ticks), with `parts.run_loop`'s truncation at `max_frames_per_episode` and the
  episode bookkeeping the CSV row reads.  One `tick()` per call, so an evaluation loop can be interleaved tick by tick
  with a training loop; `stats()` gives the keys of `reporting.EpisodeTracker` / `StepRateTracker` plus the mean
  `state_value` of the acting ticks.  The raw frames go to the device in one copy per tick, staged in pinned memory
  (double-buffered, so the staging of tick t + 1 overlaps the copy of tick t), on `stream` when one is given.

  `envs` is a list of E dm_env-style environments, or one vectorised device environment (`environments.VectorCatch`)
  whose frames tensor the agent reads in place, stepped on `stream`."""

  def __init__(self, agent, envs, num_frames, max_frames_per_episode, stream=None):
    import torch
    self._torch = torch
    self._agent, self._envs, self._max = agent, envs, max_frames_per_episode
    self._stream = stream
    self._vector = not isinstance(envs, (list, tuple))
    if self._vector:
      E = envs.num_streams
      with self._on_stream():
        first = envs.reset()
    else:
      E = len(envs)
      first = [env.reset() for env in envs]
      shape = first[0].observation[0].shape
      with self._on_stream():
        self._stage = [torch.zeros((E,) + shape, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self._frames = [torch.zeros((E,) + shape, dtype=torch.uint8, device='cuda') for _ in range(2)]
      self._copied = [None, None]
    self._E = E
    agent.reset()
    self._timesteps = first
    self._steps = np.zeros(E, np.int64)
    self._returns, self._values = [], []
    self._ticks = -(-num_frames // E)
    self._tick = 0
    self._duration = 0.0

  def _on_stream(self):
    import contextlib
    return self._torch.cuda.stream(self._stream) if self._stream is not None else contextlib.nullcontext()

  @property
  def done(self) -> bool:
    return self._tick >= self._ticks

  def tick(self) -> None:
    from dqn_zoo_b200 import parts
    torch = self._torch
    t0 = timeit.default_timer()
    E, agent, envs = self._E, self._agent, self._envs
    if self._vector:
      frames, step_type, reward, discount, lives = self._timesteps
      step_type = step_type.copy()
    else:
      frames, step_type, reward, discount, lives = self._stage_timesteps()
    self._steps = np.where(step_type == int(parts.StepType.FIRST), 0, self._steps) + 1
    if self._max > 0:                            # run_loop's truncation: relabel the timestep LAST
      step_type[self._steps > self._max] = int(parts.StepType.LAST)
    actions = agent.step(frames, step_type, reward, discount, lives)
    value = agent.statistics.get('state_value', math.nan)
    if not math.isnan(value):
      self._values.append(value)
    last = step_type == int(parts.StepType.LAST)
    if last.any():
      self._returns.extend(agent.episode_return[last].tolist())
      agent.reset(np.nonzero(last)[0])
    if self._vector:
      with self._on_stream():
        self._timesteps = envs.step(actions, reset=last)
    else:
      self._timesteps = [envs[e].reset() if last[e] else envs[e].step(int(actions[e])) for e in range(E)]
    self._tick += 1
    self._duration += timeit.default_timer() - t0

  def _stage_timesteps(self):
    """The E host timesteps as struct-of-arrays, their frames sent to the device in one staged copy."""
    torch = self._torch
    slot = self._tick % 2
    if self._copied[slot] is not None:
      self._copied[slot].synchronize()           # the copy out of this staging buffer has finished
    host = self._stage[slot].numpy()
    timesteps = self._timesteps
    for e, ts in enumerate(timesteps):
      host[e] = ts.observation[0]
    step_type = np.array([int(ts.step_type) for ts in timesteps], np.int64)
    reward = np.array([np.nan if ts.reward is None else ts.reward for ts in timesteps])
    discount = np.array([np.nan if ts.discount is None else ts.discount for ts in timesteps])
    lives = np.array([ts.observation[1] for ts in timesteps], np.int64)
    with self._on_stream():
      self._frames[slot].copy_(self._stage[slot], non_blocking=True)
      self._copied[slot] = torch.cuda.Event()
      self._copied[slot].record()
    return self._frames[slot], step_type, reward, discount, lives

  def run(self):
    while not self.done:
      self.tick()
    return self.stats()

  def stats(self):
    running = float(self._agent.episode_return.mean())
    frames_done = self._tick * self._E
    return {
        'episode_return': float(np.mean(self._returns)) if self._returns else (running if frames_done else math.nan),
        'num_episodes': len(self._returns),
        'step_rate': frames_done / self._duration if frames_done else math.nan,
        'state_value': float(np.mean(self._values)) if self._values else math.nan,
    }


def train_streams(trainer, envs, num_frames, max_frames_per_episode):
  """`num_frames` frames (rounded up to whole ticks) of E environments through `trainer` (a `StreamLoop` run to the
  end); returns its statistics."""
  return StreamLoop(trainer, envs, num_frames, max_frames_per_episode).run()


def eval_streams(evaluator, envs, num_frames, max_frames_per_episode):
  """The evaluation phase on E environments through an `agent.VectorEvaluator`, on the evaluator's CUDA stream."""
  return StreamLoop(evaluator, envs, num_frames, max_frames_per_episode, stream=evaluator.stream).run()


def iteration_row(iteration, args, train_stats, eval_stats, train_epsilon):
  """The CSV row of one iteration (the column names and order of the reference's run_atari)."""
  return [
      ('iteration', iteration, '%3d'),
      ('frame', iteration * args.num_train_frames, '%5d'),
      ('eval_episode_return', eval_stats['episode_return'], '% 2.2f'),
      ('train_episode_return', train_stats['episode_return'], '% 2.2f'),
      ('eval_num_episodes', eval_stats['num_episodes'], '%3d'),
      ('train_num_episodes', train_stats['num_episodes'], '%3d'),
      ('eval_frame_rate', eval_stats['step_rate'], '%4.0f'),
      ('train_frame_rate', train_stats['step_rate'], '%4.0f'),
      ('train_exploration_epsilon', train_epsilon, '%.3f'),
      ('train_state_value', train_stats['state_value'], '%.3f'),
  ]


def parse_args(argv=None):
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--env', default='synthetic', choices=['synthetic', 'catch', 'breakout', 'pong'],
                  help='synthetic: random host frames; catch / breakout / pong: a game simulated and rendered on the device '
                       '(dqn_zoo_b200.environments)')
  ap.add_argument('--agent', default='dqn',
                  choices=['dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn', 'munchausen',
                           'munchausen_iqn', 'fqf'])
  ap.add_argument('--dueling', action='store_true',
                  help='the dueling network (DESIGN.md §16): dqn, double_q, prioritized and munchausen only')
  ap.add_argument('--noisy', action='store_true',
                  help='noisy networks (DESIGN.md §17) with a zero epsilon schedule: dqn, double_q, prioritized and '
                       'munchausen only; combines with --dueling')
  ap.add_argument('--random_shift_pad', type=int, default=0,
                  help='random-shift augmentation of every learner step at pad N in [0, 16] (DESIGN.md §18); 0: off')
  ap.add_argument('--prioritized', action='store_true',
                  help='prioritized replay for any agent (DESIGN.md §19): rainbow\'s exponent 0.5, importance exponent '
                       '0.4 -> 1 and uniform-sample probability 1e-3; prioritized and rainbow always use it')
  ap.add_argument('--num_actions', type=int, default=6)
  ap.add_argument('--replay_capacity', type=int, default=20000)
  ap.add_argument('--min_replay_capacity_fraction', type=float, default=0.05)
  ap.add_argument('--target_network_update_period', type=int, default=4000)
  ap.add_argument('--num_iterations', type=int, default=2)
  ap.add_argument('--num_train_frames', type=int, default=4000)
  ap.add_argument('--num_eval_frames', type=int, default=1000)
  ap.add_argument('--max_frames_per_episode', type=int, default=108000)
  ap.add_argument('--eval_exploration_epsilon', type=float, default=0.01)
  ap.add_argument('--seed', type=int, default=1)
  ap.add_argument('--results_csv_path', default='')
  ap.add_argument('--checkpoint_path', default='', help='pickle the whole run state into one file (FileCheckpoint)')
  ap.add_argument('--checkpoint_dir', default='',
                  help='checkpoint into a directory (DirectoryCheckpoint): the agent and its replay are streamed to '
                       'files with bounded host memory')
  ap.add_argument('--background_checkpoint', action='store_true',
                  help='with --checkpoint_dir: snapshot the agent and its replay in device memory at the end of each '
                       'iteration and write the directory on a background thread while training goes on')
  ap.add_argument('--num_streams', type=int, default=1, help='E > 1: train from E environments with agent.VectorTrainer')
  ap.add_argument('--num_eval_streams', type=int, default=0,
                  help='E >= 1: evaluate on E environments of their own with agent.VectorEvaluator')
  ap.add_argument('--overlap_eval', action='store_true',
                  help="run iteration i's evaluation on its own CUDA stream, interleaved tick by tick with iteration "
                       "i + 1's training (needs --num_streams > 1 and --num_eval_streams; rows are written one "
                       "iteration late)")
  args = ap.parse_args(argv)
  if args.num_streams < 1:
    ap.error('--num_streams must be >= 1')
  if args.num_eval_streams < 0:
    ap.error('--num_eval_streams must be >= 0')
  if args.overlap_eval and (args.num_streams < 2 or args.num_eval_streams < 1):
    ap.error('--overlap_eval needs --num_streams > 1 and --num_eval_streams >= 1')
  if args.overlap_eval and (args.checkpoint_path or args.checkpoint_dir):
    ap.error('--overlap_eval does not checkpoint: an iteration ends while the previous evaluation is still running')
  if args.env == 'catch' and not 3 <= args.num_actions <= 18:
    ap.error('--env catch needs --num_actions in [3, 18]')
  if args.env == 'breakout' and not 4 <= args.num_actions <= 18:
    ap.error('--env breakout needs --num_actions in [4, 18]')
  if args.env == 'pong' and not 6 <= args.num_actions <= 18:
    ap.error('--env pong needs --num_actions in [6, 18]')
  if args.checkpoint_path and args.checkpoint_dir:
    ap.error('give --checkpoint_path or --checkpoint_dir, not both')
  if args.background_checkpoint and not args.checkpoint_dir:
    ap.error('--background_checkpoint needs --checkpoint_dir')
  return args


def run(args):
  """The iterations of the run driver; returns the CSV rows (OrderedDicts) in order."""
  import torch
  if not torch.cuda.is_available():
    raise SystemExit('run_synthetic.py needs a CUDA device (the package has no CPU fallback)')
  from dqn_zoo_b200 import agent as agent_lib
  from dqn_zoo_b200 import environments
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import processors
  from dqn_zoo_b200 import reporting

  random_state = np.random.RandomState(args.seed)
  writer = reporting.CsvWriter(args.results_csv_path) if args.results_csv_path else reporting.NullWriter()

  def environment_builder(num_streams=0):
    """A new environment seeded from the run's RandomState; with a device game and num_streams > 0, its vectorised
    form (VectorCatch, VectorBreakout, VectorPong)."""
    seed = int(random_state.randint(1, 2 ** 31))
    if args.env == 'catch':
      if num_streams:
        return environments.VectorCatch(num_streams, seed, num_actions=args.num_actions)
      return environments.Catch(seed, num_actions=args.num_actions)
    if args.env == 'breakout':
      if num_streams:
        return environments.VectorBreakout(num_streams, seed, num_actions=args.num_actions)
      return environments.Breakout(seed, num_actions=args.num_actions)
    if args.env == 'pong':
      if num_streams:
        return environments.VectorPong(num_streams, seed, num_actions=args.num_actions)
      return environments.Pong(seed, num_actions=args.num_actions)
    return SyntheticAtari(seed=seed, num_actions=args.num_actions)

  def preprocessor_builder():
    return processors.atari(device_observations=True)

  train_agent, network = build_train_agent(args, random_state, preprocessor_builder())
  trainer = None
  if args.num_streams > 1:
    trainer = agent_lib.VectorTrainer(train_agent, num_streams=args.num_streams,
                                      rng_key=[0, int(random_state.randint(1, 2 ** 31))])
  eval_key = [0, int(random_state.randint(1, 2 ** 31))]
  if args.num_eval_streams:
    eval_agent = agent_lib.VectorEvaluator(network, args.num_eval_streams, args.eval_exploration_epsilon, eval_key,
                                           stream=torch.cuda.Stream() if args.overlap_eval else None)
  else:
    eval_agent = agent_lib.EpsilonGreedyActor(preprocessor=preprocessor_builder(), network=network,
                                              exploration_epsilon=args.eval_exploration_epsilon, rng_key=eval_key)

  if args.checkpoint_dir:
    checkpoint = reporting.DirectoryCheckpoint(args.checkpoint_dir)
  elif args.checkpoint_path:
    checkpoint = reporting.FileCheckpoint(args.checkpoint_path)
  else:
    checkpoint = reporting.NullCheckpoint()
  state = checkpoint.state
  state.iteration = 0
  state.train_agent = train_agent if trainer is None else trainer
  state.eval_agent = eval_agent
  state.random_state = random_state
  state.writer = writer
  if checkpoint.can_be_restored():
    checkpoint.restore()

  rows = []

  def write(iteration, train_stats, eval_stats, train_epsilon):
    log_output = iteration_row(iteration, args, train_stats, eval_stats, train_epsilon)
    print(', '.join(('%s: ' + f) % (n, v) for n, v, f in log_output), flush=True)
    row = collections.OrderedDict((n, v) for n, v, _ in log_output)
    writer.write(row)
    rows.append(row)

  pending = None                         # overlap: (iteration, train stats, epsilon, evaluation loop) still evaluating
  device_game = args.env in ('catch', 'breakout', 'pong')
  vector_game = device_game and trainer is not None
  while state.iteration <= args.num_iterations:
    # a new environment per iteration: deterministic after a restore
    env = environment_builder(args.num_streams if vector_game else 0)
    eval_env = env                       # the one-stream evaluation (no --num_eval_streams) plays the first stream
    num_train_frames = 0 if state.iteration == 0 else args.num_train_frames
    if trainer is None:
      train_seq = parts.run_loop(train_agent, env, args.max_frames_per_episode)
      train_stats = reporting.generate_statistics(reporting.make_default_trackers(train_agent),
                                                  itertools.islice(train_seq, num_train_frames))
      if device_game and args.num_eval_streams:
        eval_envs = environment_builder(args.num_eval_streams)
      else:
        eval_envs = [environment_builder() for _ in range(args.num_eval_streams)]
    else:
      if vector_game:
        envs = env
        if args.num_eval_streams:
          eval_envs = environment_builder(args.num_eval_streams)
        else:
          eval_env = environment_builder()
      else:
        envs = [env] + [environment_builder() for _ in range(args.num_streams - 1)]
        eval_envs = [environment_builder() for _ in range(args.num_eval_streams)]
      train_loop = StreamLoop(trainer, envs, num_train_frames, args.max_frames_per_episode)
      while not train_loop.done:
        train_loop.tick()
        if pending is not None and not pending[3].done:
          pending[3].tick()              # the previous iteration's evaluation, on the evaluator's stream
      train_stats = train_loop.stats()
    if pending is not None:
      write(pending[0], pending[1], pending[3].run(), pending[2])
      pending = None
    train_epsilon = train_agent.exploration_epsilon
    eval_agent.network_params = train_agent.learner      # device-to-device copy of the online parameters
    if args.num_eval_streams:
      eval_loop = StreamLoop(eval_agent, eval_envs, args.num_eval_frames, args.max_frames_per_episode,
                             stream=eval_agent.stream)
      if args.overlap_eval:
        pending = (state.iteration, train_stats, train_epsilon, eval_loop)
        state.iteration += 1
        continue
      eval_stats = eval_loop.run()
    else:
      eval_seq = parts.run_loop(eval_agent, eval_env, args.max_frames_per_episode)
      eval_stats = reporting.generate_statistics(reporting.make_default_trackers(eval_agent),
                                                 itertools.islice(eval_seq, args.num_eval_frames))
    write(state.iteration, train_stats, eval_stats, train_epsilon)
    state.iteration += 1
    if args.background_checkpoint:
      checkpoint.save(blocking=False)   # a snapshot; the directory is written while the next iteration trains
    else:
      checkpoint.save()
  if pending is not None:
    write(pending[0], pending[1], pending[3].run(), pending[2])
  if args.background_checkpoint:
    checkpoint.wait()
  writer.close()
  return rows


def main():
  run(parse_args())


if __name__ == '__main__':
  main()
