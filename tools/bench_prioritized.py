#!/usr/bin/env python
"""Prioritized replay for every agent kind (DESIGN.md §19) against the uniform replay: the CUDA-graph `_learn()` step
(sample -> update -> priority write-back on PER; sample -> update on uniform) of each kind, batch 32, 84x84x4, 6
actions, on a full synthetic replay of `--capacity` transitions in each storage layout (transition-major:
bulk_fill_synthetic; frame-deduplicated: bulk_fill_synthetic_stacked).  The PER replay has rainbow's exponent 0.5,
importance exponent 0.4 and uniform-sample probability 1e-3.  Per kind and layout the uniform and PER agents run in
alternated rounds in one process, so that they share the machine's state; the median step time of the rounds and the
PER - uniform difference are reported.  prioritized and rainbow are not listed: they learn by priority whatever their
replay, and double_q on PER is prioritized's step (the same launches and arithmetic).  One JSON line per result; the
first and the last name the card, its power limit and its clocks.

  python tools/bench_prioritized.py [--steps 500] [--rounds 5] [--kinds dqn,c51,...] [--layouts dense,dedup]
"""

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench_train  # noqa: E402

KINDS = ('dqn', 'double_q', 'munchausen', 'c51', 'qrdqn', 'iqn', 'munchausen_iqn', 'fqf')
LAYOUTS = ('dense', 'dedup')


def emit(**kw):
  print(json.dumps(kw), flush=True)


def make_agent(kind, prioritized, layout, capacity, seed=1):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  structure = dr.Transition(None, None, None, None, None)
  dedup = layout == 'dedup'
  if prioritized:
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.5, lambda t: 0.4, 1e-3, True, rs, frame_dedup=dedup)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, frame_dedup=dedup)
  if dedup:
    dr.bulk_fill_synthetic_stacked(rep, (84, 84, 4), seed, 6, episode_len=1000)
  else:
    dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6)
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6), optimizer=None,
                replay=rep, batch_size=32, min_replay_capacity_fraction=0.05, learn_period=16,
                target_network_update_period=40000, rng_key=[0, 7], transition_accumulator=dr.NStepTransitionAccumulator(1))
  eps = lambda t: 0.01
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


def time_steps(agent, steps):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  start.record()
  for _ in range(steps):
    agent.learn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) * 1e3 / steps


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--steps', type=int, default=500)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--capacity', type=int, default=1 << 17)
  ap.add_argument('--kinds', default=','.join(KINDS))
  ap.add_argument('--layouts', default=','.join(LAYOUTS))
  a = ap.parse_args()
  kinds, layouts = tuple(a.kinds.split(',')), tuple(a.layouts.split(','))
  if not kinds or any(k not in KINDS for k in kinds):
    raise SystemExit('--kinds: choose from %s' % ', '.join(KINDS))
  if not layouts or any(x not in LAYOUTS for x in layouts):
    raise SystemExit('--layouts: choose from %s' % ', '.join(LAYOUTS))
  if not torch.cuda.is_available():
    raise SystemExit('bench_prioritized.py needs a CUDA device')
  torch.cuda.set_device(0)
  emit(metric='device', **bench_train.device_info())
  for layout in layouts:
    for kind in kinds:
      agents = {per: make_agent(kind, per, layout, a.capacity) for per in (False, True)}
      for ag in agents.values():
        for _ in range(a.warmup):
          ag.learn()
      times = {per: [] for per in agents}
      for _ in range(a.rounds):
        for per, ag in agents.items():
          times[per].append(time_steps(ag, a.steps))
      med = {per: float(np.median(t)) for per, t in times.items()}
      emit(metric='learn_step_us', kind=kind, layout=layout, uniform=round(med[False], 2), per=round(med[True], 2),
           per_minus_uniform_us=round(med[True] - med[False], 2), rounds_uniform=[round(t, 2) for t in times[False]],
           rounds_per=[round(t, 2) for t in times[True]])
      del agents
      torch.cuda.empty_cache()
  emit(metric='device_after', **bench_train.device_info())


if __name__ == '__main__':
  main()
