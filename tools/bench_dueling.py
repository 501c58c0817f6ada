#!/usr/bin/env python
"""The dueling network (DESIGN.md §16) and noisy networks (§17) beside the plain one, for dqn, double_q, prioritized and
munchausen: CUDA-graph `_learn()` steps (sample -> update -> priority write-back) on a 1M-capacity frame-deduplicated
synthetic replay (uniform; prioritized: PER at exponent 0.6), batch 32, 84x84x4, 6 actions.  Per kind, the agents of
the chosen networks (plain, dueling, noisy, noisy_dueling) run in alternated rounds in one process, so that they share
the machine's state.  Then one eager profiled pass of each
(per-launch CUDA events, dz_profile_begin / end): the library launches per step and the times of fc1_fwd, fc1_dgrad,
fc1_wgrad, dueling_head_fwd, dueling_head_bwd, head_wgrad and the plain head's launches they replace (head_fwd,
head_dgrad and their finishes; for noisy networks the noisy launches), and the act time of a live actor at E in
{1, 32, 256} (noisy networks: with one shared noise apply and with one apply per stream).  One JSON line per result; the
first and the last name the card, its power limit and its clocks.

  python tools/bench_dueling.py [--steps 2000] [--rounds 3] [--kinds dqn,double_q,prioritized,munchausen]
                                [--networks plain,dueling,noisy,noisy_dueling]

The expectation this checks: the dueling step adds a second 3136 -> 512 stream (6.4 MB more fc weights per blob in the
forward, the input gradient and the weight gradient) and replaces the head's grouped GEMM, split finish and input
gradient by the two dueling kernels, so it should cost the plain step plus about one more fc1 stream's weight traffic.
"""

import argparse
import ctypes as C
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench_train  # noqa: E402

KINDS = ('dqn', 'double_q', 'prioritized', 'munchausen')
NETWORKS = {'plain': (False, False), 'dueling': (True, False), 'noisy': (False, True), 'noisy_dueling': (True, True)}
CAPACITY = 1 << 20


def emit(**kw):
  print(json.dumps(kw), flush=True)


def make_agent(kind, network, capacity, seed=1):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  structure = dr.Transition(None, None, None, None, None)
  if kind == 'prioritized':
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.6, lambda t: 0.4, 1e-3, True, rs, frame_dedup=True)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, frame_dedup=True)
  dr.bulk_fill_synthetic_stacked(rep, (84, 84, 4), seed, 6, episode_len=1000)
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6, dueling=NETWORKS[network][0],
                                                                           noisy=NETWORKS[network][1]),
                optimizer=None, transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=0.05, learn_period=16, target_network_update_period=40000, rng_key=[0, 7])
  return ag.AGENTS[kind](exploration_epsilon=lambda t: 0.01, grad_error_bound=1.0 / 32, **common)


def time_steps(agent, steps):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  start.record()
  for _ in range(steps):
    agent.learn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) * 1e3 / steps


def profile_step(agent, reps=50):
  """Per-launch event times of `reps` eager steps: ({tag: us per step}, library launches per step)."""
  from dqn_zoo_b200 import _lib
  agent._use_graph = False
  agent.learn()
  _lib.call('dz_profile_begin')
  for _ in range(reps):
    agent.learn()
  buf = C.create_string_buffer(1 << 16)
  _lib.call('dz_profile_end', buf, len(buf))
  agent._use_graph = True
  prof = json.loads(buf.value.decode())
  return {k: round(v[1] * 1e3 / reps, 2) for k, v in prof.items()}, sum(v[0] for v in prof.values()) // reps


def act_us(learner, E, reps=300, noise=None):
  """One live actor act at E streams; noise 'shared' / 'stream': a noisy network's one apply / one apply per stream."""
  obs = torch.as_tensor(np.random.RandomState(E).randint(0, 256, (E, 84, 84, 4)).astype(np.uint8), device='cuda')
  x = learner.actor(E)
  kw = {}
  if noise == 'shared':
    kw = {'noise': x.generate_randomness(1).clone()}
  elif noise == 'stream':
    kw = {'stream_noise': x.generate_randomness(1, per_stream=True).clone()}
  for _ in range(30):
    x.act(obs, **kw)
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  start.record()
  for _ in range(reps):
    x.act(obs, **kw)
  end.record()
  end.synchronize()
  return round(start.elapsed_time(end) * 1e3 / reps, 2)


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--steps', type=int, default=2000)
  ap.add_argument('--warmup', type=int, default=200)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--capacity', type=int, default=CAPACITY)
  ap.add_argument('--kinds', default=','.join(KINDS))
  ap.add_argument('--networks', default='plain,dueling', help='from %s' % ', '.join(NETWORKS))
  a = ap.parse_args()
  kinds = tuple(a.kinds.split(','))
  if not kinds or any(k not in KINDS for k in kinds):
    raise SystemExit('--kinds: choose from %s' % ', '.join(KINDS))
  networks = tuple(a.networks.split(','))
  if not networks or any(n not in NETWORKS for n in networks):
    raise SystemExit('--networks: choose from %s' % ', '.join(NETWORKS))
  if not torch.cuda.is_available():
    raise SystemExit('bench_dueling.py needs a CUDA device')
  torch.cuda.set_device(0)
  emit(metric='device', **bench_train.device_info())
  for kind in kinds:
    agents = {n: make_agent(kind, n, a.capacity) for n in networks}
    for ag in agents.values():
      for _ in range(a.warmup):
        ag.learn()
    times = {d: [] for d in agents}
    for r in range(a.rounds):
      for d, ag in agents.items():
        us = time_steps(ag, a.steps)
        times[d].append(us)
        emit(metric='learn_step_us', agent=kind, network=d, round=r, steps=a.steps, us=round(us, 2))
    for d, ag in agents.items():
      prof, launches = profile_step(ag)
      acting = {'act_us': {E: act_us(ag.learner, E) for E in (1, 32, 256)}} if not NETWORKS[d][1] else {
          'act_us_shared_noise': {E: act_us(ag.learner, E, noise='shared') for E in (1, 32, 256)},
          'act_us_stream_noise': {E: act_us(ag.learner, E, noise='stream') for E in (1, 32, 256)}}
      emit(metric='learn_step_summary', agent=kind, network=d, median_us=round(float(np.median(times[d])), 2),
           min_us=round(min(times[d]), 2), max_us=round(max(times[d]), 2), launches_per_step=launches,
           launch_us=prof, **acting)
    del agents
    torch.cuda.empty_cache()
  emit(metric='device_after', **bench_train.device_info())


if __name__ == '__main__':
  main()
