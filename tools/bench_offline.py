"""Offline training with conservative Q-learning (DESIGN.md §20): the CQL term's step time and a runnable offline RL
recipe on Catch.  One JSON line per point.

  * step: CUDA-graph learner steps (`agent.learn()`) at cql_alpha 0 and 1, alternated in one process, for dqn, double_q,
    munchausen, c51, qrdqn, rainbow, iqn and fqf on a 2^17-transition synthetic frame-deduplicated replay at 84x84x4,
    B 32: `--steps` steps x `--rounds` rounds per alpha, median and spread of us per step, and launches per step at
    both alphas (`dz_launch_count` over one eager step).
  * offline (`--offline UPDATES`): a dataset of `--dataset` transitions recorded on 3-action Catch (noop, left, right)
    by a uniformly random behaviour policy through a `VectorTrainer` whose agent never reaches its learning gate, saved
    with `replay.save_checkpoint` and loaded into a fresh replay; then dqn and qrdqn trained on it offline
    (`agent.OfflineTrainer`) with 6-action networks at cql_alpha 0 and 1, so that actions 3-5 never appear in the
    data.  Every `--eval_every` updates: the evaluation return on 6-action Catch (bench_env.evaluate; actions >= 3 are
    no-ops there), and on 4096 dataset states the share whose greedy action lies outside {0, 1, 2} and the mean of
    max_{a>=3} Q - max_{a<3} Q.

The card's name, power limit and SM clock are read in the same run.

  python tools/bench_offline.py [--parts step,offline] [--offline 30000]"""

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

OBS = (84, 84, 4)
STEP_KINDS = ('dqn', 'double_q', 'munchausen', 'c51', 'qrdqn', 'rainbow', 'iqn', 'fqf')


def emit(**kw):
  print(json.dumps(kw), flush=True)


def device_info():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True)
  return {'device': torch.cuda.get_device_name(), 'nvidia_smi': q.stdout.strip()}


def make_agent(kind, replay, cql_alpha, num_actions=6, seed=7, graph=True, learn_period=4, target_period=8000):
  """An agent of `kind` on `replay` with `cql_alpha`: the reference's hyper-parameters for its kind (rainbow: its
  support and noisy greedy acting; iqn 64 / 64 / 64 taus; fqf 32 fractions) and dqn's epsilon-greedy acting."""
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, num_actions), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(1), replay=replay, batch_size=32,
                min_replay_capacity_fraction=0.0, learn_period=learn_period, target_network_update_period=target_period,
                rng_key=[0, seed], use_cuda_graph=graph, cql_alpha=cql_alpha)
  eps = lambda t: 0.01
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common)
  if kind == 'c51':
    return ag.C51(support=np.linspace(-10, 10, 51), exploration_epsilon=eps, **common)
  if kind == 'qrdqn':
    return ag.QrDqn(quantiles=(np.arange(201) + 0.5) / 201, exploration_epsilon=eps, huber_param=1.0, **common)
  if kind == 'fqf':
    return ag.Fqf(exploration_epsilon=eps, huber_param=1.0, **common)
  if dl.uses_iqn_network(kind):
    return ag.AGENTS[kind](exploration_epsilon=eps, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                           tau_samples_s_t=64, **common)
  return ag.AGENTS[kind](exploration_epsilon=eps, grad_error_bound=1.0 / 32, **common)


# -- step time -----------------------------------------------------------------------------------------------------------
def launches_per_step(agent):
  from dqn_zoo_b200 import _lib
  agent.learn()
  torch.cuda.synchronize()
  c0 = _lib.lib.dz_launch_count()
  agent.learn()
  torch.cuda.synchronize()
  return int(_lib.lib.dz_launch_count() - c0)


def bench_steps(steps, rounds):
  from dqn_zoo_b200 import replay as dr
  for kind in STEP_KINDS:
    agents = {}
    launches = {}
    for alpha in (0.0, 1.0):
      rep = dr.PrioritizedTransitionReplay(1 << 17, dr.Transition(None, None, None, None, None), 0.5, lambda t: 0.4,
                                           1e-3, True, np.random.RandomState(1), frame_dedup=True) \
          if kind == 'rainbow' else dr.TransitionReplay(1 << 17, dr.Transition(None, None, None, None, None),
                                                        np.random.RandomState(1), frame_dedup=True)
      dr.bulk_fill_synthetic_stacked(rep, OBS, 1, 6, episode_len=1000)
      launches[alpha] = launches_per_step(make_agent(kind, rep, alpha, graph=False))
      agents[alpha] = make_agent(kind, rep, alpha)
      for _ in range(50):
        agents[alpha].learn()
    torch.cuda.synchronize()
    us = {0.0: [], 1.0: []}
    for _ in range(rounds):
      for alpha in (0.0, 1.0):
        a = agents[alpha]
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for _ in range(steps):
          a.learn()
        end.record()
        end.synchronize()
        us[alpha].append(start.elapsed_time(end) * 1e3 / steps)
    emit(metric='cql_step', agent=kind, steps=steps, rounds=rounds,
         us_alpha0=[round(x, 2) for x in us[0.0]], us_alpha1=[round(x, 2) for x in us[1.0]],
         median_us_alpha0=round(float(np.median(us[0.0])), 2), median_us_alpha1=round(float(np.median(us[1.0])), 2),
         added_us=round(float(np.median(us[1.0]) - np.median(us[0.0])), 2),
         launches_per_step_alpha0=launches[0.0], launches_per_step_alpha1=launches[1.0])
    del agents


# -- offline learning on Catch ---------------------------------------------------------------------------------------------
DATA_ACTIONS = 3
NET_ACTIONS = 6


def record_dataset(size, seed=0, num_streams=64):
  """A frame-deduplicated replay of `size` transitions of 3-action Catch under a uniformly random policy: a
  `VectorTrainer` over a dqn agent at epsilon 1 whose learning gate (min_replay_capacity) is never reached."""
  import run_synthetic
  import bench_env
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rep = dr.TransitionReplay(size, dr.Transition(None, None, None, None, None), np.random.RandomState(seed),
                            frame_dedup=True)
  behaviour = ag.Dqn(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec('dqn', DATA_ACTIONS),
                     optimizer=None, transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                     exploration_epsilon=lambda t: 1.0, min_replay_capacity_fraction=2.0, learn_period=16,
                     target_network_update_period=8000, grad_error_bound=1.0 / 32, rng_key=[0, seed + 1])
  trainer = ag.VectorTrainer(behaviour, num_streams=num_streams, rng_key=[0, seed + 2])
  env = bench_env.make_env('catch', num_streams, seed + 3, DATA_ACTIONS)
  loop = run_synthetic.StreamLoop(trainer, env, 1 << 40, 0)
  while rep.size < size:
    loop.tick()
  torch.cuda.synchronize()
  assert behaviour._learn_steps == 0
  return rep, loop.stats()['episode_return']


def load_dataset(rep, seed=0):
  """The recipe's second half: the dataset written with `save_checkpoint` and read back into a fresh replay."""
  from dqn_zoo_b200 import replay as dr
  fresh = dr.TransitionReplay(rep.capacity, dr.Transition(None, None, None, None, None), np.random.RandomState(seed),
                              frame_dedup=True)
  with tempfile.TemporaryDirectory() as d:
    rep.save_checkpoint(os.path.join(d, 'dataset'))
    fresh.load_checkpoint(os.path.join(d, 'dataset'))
  return fresh


def dataset_states(rep, n=4096, seed=5):
  ids = np.random.RandomState(seed).choice(rep.size, n, replace=False)
  return torch.tensor(np.stack([t.s_tm1 for t in rep.get(ids)]))


def conservatism(learner, states):
  """(share of states whose greedy action is >= 3, mean of max_{a>=3} Q - max_{a<3} Q) under the online network."""
  qs = []
  B = learner.batch_size
  kw = {}
  for i in range(0, states.shape[0], B):
    chunk = states[i:i + B].to(learner.device)
    if learner.kind == 'iqn':
      kw = {'taus': torch.rand(chunk.shape[0] * learner.net.tau_samples_policy, device=learner.device)}
    _, q = learner.act_batch(chunk, epsilon=0.0, **kw)
    qs.append(q.clone().cpu())
  q = torch.cat(qs).double()
  out = q[:, DATA_ACTIONS:].max(1).values
  seen = q[:, :DATA_ACTIONS].max(1).values
  return float((q.argmax(1) >= DATA_ACTIONS).double().mean()), float((out - seen).mean())


def offline_run(rep, kind, cql_alpha, updates, eval_every, seed=0, states=None, log=None):
  """Trains a 6-action `kind` agent offline on `rep`; returns [(updates, eval return, eval episodes, out-of-data
  greedy share, mean out-of-data gap)]."""
  import bench_env
  from dqn_zoo_b200 import agent as ag
  agent = make_agent(kind, rep, cql_alpha, num_actions=NET_ACTIONS, seed=seed + 11, learn_period=16)
  trainer = ag.OfflineTrainer(agent)
  states = dataset_states(rep) if states is None else states
  curve = []
  while trainer.updates < updates:
    trainer.step(min(eval_every, updates - trainer.updates))
    ret, n = bench_env.evaluate(agent.learner, seed, num_actions=NET_ACTIONS)
    share, gap = conservatism(agent.learner, states)
    curve.append((trainer.updates, ret, n, share, gap))
    if log:
      log(agent=kind, cql_alpha=cql_alpha, updates=trainer.updates, eval_return=round(ret, 3), eval_episodes=n,
          out_of_data_greedy=round(share, 4), out_of_data_gap=round(gap, 4))
  return curve


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--parts', default='step,offline')
  ap.add_argument('--steps', type=int, default=500)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--offline', type=int, default=30000, help='updates per offline run')
  ap.add_argument('--eval_every', type=int, default=5000)
  ap.add_argument('--dataset', type=int, default=1 << 17)
  args = ap.parse_args()
  emit(metric='device', **device_info())
  parts = args.parts.split(',')
  if 'step' in parts:
    bench_steps(args.steps, args.rounds)
  if 'offline' in parts:
    t0 = time.perf_counter()
    rep, behaviour_return = record_dataset(args.dataset)
    emit(metric='dataset', transitions=rep.size, behaviour_return=round(behaviour_return, 3),
         seconds=round(time.perf_counter() - t0, 1))
    rep = load_dataset(rep)
    states = dataset_states(rep)
    for kind in ('dqn', 'qrdqn'):
      for alpha in (0.0, 1.0):
        offline_run(rep, kind, alpha, args.offline, args.eval_every, states=states,
                    log=lambda **kw: emit(metric='offline', **kw))
  emit(metric='device', **device_info())


if __name__ == '__main__':
  main()
