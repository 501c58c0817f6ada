"""Munchausen DQN's learner step beside double_q's and dqn's: CUDA-graph `_learn()` steps (sample -> update) at
84x84x4, batch 32, 6 actions, on a synthetic uniform replay, the three agents alternated over `--rounds` rounds in one
process so that they share the machine's state.  Then one eager profiled pass of each (per-launch CUDA events,
dz_profile_begin / end) for the loss kernels' times.  One JSON line per result.
  python tools/bench_munchausen.py [--steps 2000] [--rounds 3] [--kinds munchausen,double_q,dqn]

`--kinds munchausen_iqn,iqn` times Munchausen-IQN beside iqn (64 / 64 / 64 taus drawn on the device each step): it adds
a third torso pass, target(s_tm1), to iqn's two, so its step should cost iqn's plus about one torso pass.

`--kinds fqf,iqn` times FQF (32 proposed fractions) beside iqn: FQF sends fewer rows through the embedding and fc1
(4096 against 6144 forward, 1024 against 2048 backward) but runs the fraction layer between the torso and the
embedding, where iqn's taus are drawn beforehand; which effect wins is what this measures.  The profiled pass then also
times fraction_forward_kernel and the fraction layer's optimizer launch.

The expectation this checks: munchausen applies three networks per step like double_q (online(s_tm1) with
target(s_tm1) and target(s_t) instead of online(s_t) and target(s_t)), the two target passes sharing each staged fc1
weight tile as double_q's two online passes do, so its step should cost about what double_q's does."""

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

KINDS = ('munchausen', 'double_q', 'dqn')
ALL_KINDS = KINDS + ('munchausen_iqn', 'iqn', 'fqf')


def emit(**kw):
  print(json.dumps(kw), flush=True)


def make_agent(kind, capacity=65536, seed=1):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  rep = dr.TransitionReplay(capacity, dr.Transition(None, None, None, None, None), rs)
  dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6, discount=0.99)
  common = dict(preprocessor=lambda ts: ts, sample_network_input=np.zeros((84, 84, 4), np.uint8),
                network=dl.NetworkSpec(kind, 6), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=0.02, learn_period=16, target_network_update_period=32000,
                rng_key=[0, seed])
  if kind == 'fqf':
    return ag.Fqf(exploration_epsilon=lambda t: 0.01, huber_param=1.0, **common)
  if dl.uses_iqn_network(kind):
    return ag.AGENTS[kind](exploration_epsilon=lambda t: 0.01, huber_param=1.0, tau_samples_policy=64,
                           tau_samples_s_tm1=64, tau_samples_s_t=64, **common)
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
  """Per-launch event times of `reps` eager steps (the CUDA graph is off while profiling): {tag: us per step}."""
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
  return {k: (round(v[1] * 1e3 / reps, 2), v[0] // reps, (v[2], v[3], v[4])) for k, v in prof.items()}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=2000)
  ap.add_argument('--warmup', type=int, default=200)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--kinds', default=','.join(KINDS), help='comma-separated agent kinds, alternated in this order')
  a = ap.parse_args()
  kinds = tuple(a.kinds.split(','))
  if not kinds or any(k not in ALL_KINDS for k in kinds):
    raise SystemExit('--kinds: choose from %s' % ', '.join(ALL_KINDS))
  if not torch.cuda.is_available():
    raise SystemExit('bench_munchausen.py needs a CUDA device')
  torch.cuda.set_device(0)
  emit(metric='device', **bench_train.device_info())
  agents = {k: make_agent(k) for k in kinds}
  for k, ag in agents.items():
    for _ in range(a.warmup):
      ag.learn()
  times = {k: [] for k in kinds}
  for r in range(a.rounds):
    for k in kinds:
      us = time_steps(agents[k], a.steps)
      times[k].append(us)
      emit(metric='learn_step_us', agent=k, round=r, steps=a.steps, us=round(us, 2))
  for k in kinds:
    emit(metric='learn_step_us_summary', agent=k, median=round(float(np.median(times[k])), 2),
         min=round(min(times[k]), 2), max=round(max(times[k]), 2))
  for k in kinds:
    prof = profile_step(agents[k])
    loss = {t: v for t, v in prof.items() if t.startswith('loss_')}
    emit(metric='loss_kernel_us', agent=k, kernels={t: v[0] for t, v in loss.items()})
    if k == 'fqf':   # the launches fqf adds to iqn's step
      emit(metric='fqf_kernel_us', agent=k, kernels={t: v[0] for t, v in prof.items()
                                                     if t.startswith('fraction_') or t.startswith('fqf_')})
    emit(metric='launches', agent=k, launches={t: [v[1], list(v[2])] for t, v in prof.items()})
  emit(metric='device_after', **bench_train.device_info())


if __name__ == '__main__':
  main()
