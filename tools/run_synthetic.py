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
counts the frames of all streams.  Evaluation, CSV rows and checkpoints are as with one stream.
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
  prioritized = kind in ('prioritized', 'rainbow')
  n_step = 3 if kind == 'rainbow' else 1
  structure = replay_lib.Transition(None, None, None, None, None)
  if prioritized:
    schedule = parts.LinearSchedule(begin_t=int(args.min_replay_capacity_fraction * args.replay_capacity),
                                    decay_steps=max(args.num_iterations * args.num_train_frames // 4, 1), begin_value=0.4,
                                    end_value=1.0)
    replay = replay_lib.PrioritizedTransitionReplay(args.replay_capacity, structure, 0.5 if kind == 'rainbow' else 0.6, schedule,
                                                    1e-3, True, random_state)
  else:
    replay = replay_lib.TransitionReplay(args.replay_capacity, structure, random_state)
  network = learner_lib.NetworkSpec(kind, args.num_actions)
  epsilon = parts.LinearSchedule(begin_t=int(args.min_replay_capacity_fraction * args.replay_capacity * 4),
                                 decay_steps=max(args.num_train_frames, 1), begin_value=1.0, end_value=0.01)
  common = dict(preprocessor=preprocessor, sample_network_input=np.zeros((84, 84, 4), np.uint8), network=network, optimizer=None,
                transition_accumulator=replay_lib.NStepTransitionAccumulator(n_step), replay=replay, batch_size=32,
                min_replay_capacity_fraction=args.min_replay_capacity_fraction, learn_period=16,
                target_network_update_period=args.target_network_update_period,
                rng_key=[0, int(random_state.randint(1, 2 ** 31))])
  if kind == 'rainbow':
    return agent_lib.Rainbow(support=np.linspace(-10, 10, 51), **common), network
  if kind == 'c51':
    return agent_lib.C51(support=np.linspace(-10, 10, 51), exploration_epsilon=epsilon, **common), network
  if kind == 'qrdqn':
    return agent_lib.QrDqn(quantiles=(np.arange(201) + 0.5) / 201, exploration_epsilon=epsilon, huber_param=1.0, **common), network
  if kind == 'iqn':
    return agent_lib.Iqn(exploration_epsilon=epsilon, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                         tau_samples_s_t=64, **common), network
  return agent_lib.AGENTS[kind](exploration_epsilon=epsilon, grad_error_bound=1.0 / 32, **common), network


def train_streams(trainer, envs, num_frames, max_frames_per_episode):
  """`num_frames` frames (rounded up to whole ticks) of E environments through `trainer`; returns the keys of
  `reporting.EpisodeTracker` / `StepRateTracker` the CSV row reads, plus the mean `state_value` of the acting ticks.
  The raw frames go to the device in one copy per tick, staged in pinned memory (double-buffered, so the staging of
  tick t + 1 overlaps the copy of tick t)."""
  import torch
  from dqn_zoo_b200 import parts
  E = len(envs)
  first = [env.reset() for env in envs]
  shape = first[0].observation[0].shape
  stage = [torch.zeros((E,) + shape, dtype=torch.uint8).pin_memory() for _ in range(2)]
  frames = [torch.zeros((E,) + shape, dtype=torch.uint8, device='cuda') for _ in range(2)]
  copied = [None, None]
  trainer.reset()
  timesteps = first
  steps = np.zeros(E, np.int64)
  returns, values = [], []
  ticks = -(-num_frames // E)
  t0 = timeit.default_timer()
  for tick in range(ticks):
    slot = tick % 2
    if copied[slot] is not None:
      copied[slot].synchronize()                 # the copy out of this staging buffer has finished
    host = stage[slot].numpy()
    for e, ts in enumerate(timesteps):
      host[e] = ts.observation[0]
    step_type = np.array([int(ts.step_type) for ts in timesteps], np.int64)
    reward = np.array([np.nan if ts.reward is None else ts.reward for ts in timesteps])
    discount = np.array([np.nan if ts.discount is None else ts.discount for ts in timesteps])
    lives = np.array([ts.observation[1] for ts in timesteps], np.int64)
    steps = np.where(step_type == int(parts.StepType.FIRST), 0, steps) + 1
    if max_frames_per_episode > 0:               # run_loop's truncation: relabel the timestep LAST
      step_type[steps > max_frames_per_episode] = int(parts.StepType.LAST)
    frames[slot].copy_(stage[slot], non_blocking=True)
    copied[slot] = torch.cuda.Event()
    copied[slot].record()
    actions = trainer.step(frames[slot], step_type, reward, discount, lives)
    value = trainer.statistics['state_value']
    if not math.isnan(value):
      values.append(value)
    last = step_type == int(parts.StepType.LAST)
    if last.any():
      returns.extend(trainer.episode_return[last].tolist())
      trainer.reset(np.nonzero(last)[0])
    timesteps = [envs[e].reset() if last[e] else envs[e].step(int(actions[e])) for e in range(E)]
  duration = timeit.default_timer() - t0
  running = float(trainer.episode_return.mean())
  frames_done = ticks * E
  return {
      'episode_return': float(np.mean(returns)) if returns else (running if frames_done else math.nan),
      'num_episodes': len(returns),
      'step_rate': frames_done / duration if frames_done else math.nan,
      'state_value': float(np.mean(values)) if values else math.nan,
  }


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--agent', default='dqn', choices=['dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn'])
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
  ap.add_argument('--checkpoint_path', default='')
  ap.add_argument('--num_streams', type=int, default=1, help='E > 1: train from E environments with agent.VectorTrainer')
  args = ap.parse_args()
  if args.num_streams < 1:
    ap.error('--num_streams must be >= 1')

  import torch
  if not torch.cuda.is_available():
    raise SystemExit('run_synthetic.py needs a CUDA device (the package has no CPU fallback)')
  from dqn_zoo_b200 import agent as agent_lib
  from dqn_zoo_b200 import parts
  from dqn_zoo_b200 import processors
  from dqn_zoo_b200 import reporting

  random_state = np.random.RandomState(args.seed)
  writer = reporting.CsvWriter(args.results_csv_path) if args.results_csv_path else reporting.NullWriter()

  def environment_builder():
    return SyntheticAtari(seed=int(random_state.randint(1, 2 ** 31)), num_actions=args.num_actions)

  def preprocessor_builder():
    return processors.atari(device_observations=True)

  train_agent, network = build_train_agent(args, random_state, preprocessor_builder())
  trainer = None
  if args.num_streams > 1:
    trainer = agent_lib.VectorTrainer(train_agent, num_streams=args.num_streams,
                                      rng_key=[0, int(random_state.randint(1, 2 ** 31))])
  eval_agent = agent_lib.EpsilonGreedyActor(preprocessor=preprocessor_builder(), network=network,
                                            exploration_epsilon=args.eval_exploration_epsilon,
                                            rng_key=[0, int(random_state.randint(1, 2 ** 31))])

  checkpoint = reporting.FileCheckpoint(args.checkpoint_path) if args.checkpoint_path else reporting.NullCheckpoint()
  state = checkpoint.state
  state.iteration = 0
  state.train_agent = train_agent if trainer is None else trainer
  state.eval_agent = eval_agent
  state.random_state = random_state
  state.writer = writer
  if checkpoint.can_be_restored():
    checkpoint.restore()

  while state.iteration <= args.num_iterations:
    env = environment_builder()          # a new environment per iteration: deterministic after a restore
    num_train_frames = 0 if state.iteration == 0 else args.num_train_frames
    if trainer is None:
      train_seq = parts.run_loop(train_agent, env, args.max_frames_per_episode)
      train_stats = reporting.generate_statistics(reporting.make_default_trackers(train_agent),
                                                  itertools.islice(train_seq, num_train_frames))
    else:
      envs = [env] + [environment_builder() for _ in range(args.num_streams - 1)]
      train_stats = train_streams(trainer, envs, num_train_frames, args.max_frames_per_episode)
    eval_agent.network_params = train_agent.learner      # device-to-device copy of the online parameters
    eval_seq = parts.run_loop(eval_agent, env, args.max_frames_per_episode)
    eval_stats = reporting.generate_statistics(reporting.make_default_trackers(eval_agent),
                                               itertools.islice(eval_seq, args.num_eval_frames))
    log_output = [
        ('iteration', state.iteration, '%3d'),
        ('frame', state.iteration * args.num_train_frames, '%5d'),
        ('eval_episode_return', eval_stats['episode_return'], '% 2.2f'),
        ('train_episode_return', train_stats['episode_return'], '% 2.2f'),
        ('eval_num_episodes', eval_stats['num_episodes'], '%3d'),
        ('train_num_episodes', train_stats['num_episodes'], '%3d'),
        ('eval_frame_rate', eval_stats['step_rate'], '%4.0f'),
        ('train_frame_rate', train_stats['step_rate'], '%4.0f'),
        ('train_exploration_epsilon', train_agent.exploration_epsilon, '%.3f'),
        ('train_state_value', train_stats['state_value'], '%.3f'),
    ]
    print(', '.join(('%s: ' + f) % (n, v) for n, v, f in log_output), flush=True)
    writer.write(collections.OrderedDict((n, v) for n, v, _ in log_output))
    state.iteration += 1
    checkpoint.save()
  writer.close()


if __name__ == '__main__':
  main()
