#!/usr/bin/env python
"""Random-shift augmentation (DESIGN.md §18) against the unaugmented step: the CUDA-graph `_learn()` step (sample ->
update -> priority write-back, with the step's randomness drawn beside the sampler) at pad 0 and pad 4 for dqn,
dueling double_q, rainbow and iqn, batch 32, 84x84x4, 6 actions, on a frame-deduplicated synthetic replay (uniform;
rainbow: PER at exponent 0.5).  Per kind the pad-0 and pad-4 agents run in alternated rounds in one process, so that
they share the machine's state; the median step time of the rounds is reported.  Then the shift kernel alone
(dz_test_random_shift, B = 32, 84x84x4, pad 4) timed with CUDA events over many launches, and its bytes (each
observation read once and written once) over that time.  One JSON line per result; the first and the last name the
card, its power limit and its clocks.

  python tools/bench_augment.py [--steps 1000] [--rounds 5] [--kinds dqn,double_q,rainbow,iqn]
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

KINDS = ('dqn', 'double_q', 'rainbow', 'iqn')
PAD = 4


def emit(**kw):
  print(json.dumps(kw), flush=True)


def make_agent(kind, pad, capacity, seed=1):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rs = np.random.RandomState(seed)
  structure = dr.Transition(None, None, None, None, None)
  if kind == 'rainbow':
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.5, lambda t: 0.4, 1e-3, True, rs, frame_dedup=True)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, frame_dedup=True)
  dr.bulk_fill_synthetic_stacked(rep, (84, 84, 4), seed, 6, episode_len=1000)
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6, dueling=kind == 'double_q'),
                optimizer=None, replay=rep, batch_size=32, min_replay_capacity_fraction=0.05, learn_period=16,
                target_network_update_period=40000, rng_key=[0, 7], random_shift_pad=pad)
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), transition_accumulator=dr.NStepTransitionAccumulator(3), **common)
  acc = dr.NStepTransitionAccumulator(1)
  if kind == 'iqn':
    return ag.Iqn(transition_accumulator=acc, exploration_epsilon=lambda t: 0.01, huber_param=1.0, tau_samples_policy=64,
                  tau_samples_s_tm1=64, tau_samples_s_t=64, **common)
  return ag.AGENTS[kind](transition_accumulator=acc, exploration_epsilon=lambda t: 0.01, grad_error_bound=1.0 / 32, **common)


def time_steps(agent, steps):
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  start.record()
  for _ in range(steps):
    agent.learn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) * 1e3 / steps


def shift_kernel(reps, B=32, pad=PAD):
  """(us per launch, GB/s) of the shift kernel alone over B examples' s_tm1 and s_t."""
  from dqn_zoo_b200 import _lib
  obs = 84 * 84 * 4
  rs = np.random.RandomState(0)
  src = torch.as_tensor(rs.randint(0, 256, (2 * B, obs)).astype(np.uint8), device='cuda')
  rows = src.data_ptr() + torch.arange(2 * B, dtype=torch.int64, device='cuda') * obs
  shifts = torch.as_tensor(rs.randint(0, 2 * pad + 1, (B, 4)).astype(np.int32), device='cuda')
  out = torch.empty(B * 2 * obs, dtype=torch.uint8, device='cuda')
  stream = torch.cuda.current_stream().cuda_stream
  args = (rows.data_ptr(), rows.data_ptr() + 8 * B, shifts.data_ptr(), B, 84, 84, 4, pad, out.data_ptr(), obs, stream)
  for _ in range(100):
    _lib.call('dz_test_random_shift', *args)
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  start.record()
  for _ in range(reps):
    _lib.call('dz_test_random_shift', *args)
  end.record()
  end.synchronize()
  us = start.elapsed_time(end) * 1e3 / reps
  return us, 2 * (2 * B * obs) / (us * 1e-6) / 1e9


def main():
  ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
  ap.add_argument('--steps', type=int, default=1000)
  ap.add_argument('--warmup', type=int, default=100)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--capacity', type=int, default=1 << 18)
  ap.add_argument('--kinds', default=','.join(KINDS))
  ap.add_argument('--kernel_reps', type=int, default=5000)
  a = ap.parse_args()
  kinds = tuple(a.kinds.split(','))
  if not kinds or any(k not in KINDS for k in kinds):
    raise SystemExit('--kinds: choose from %s' % ', '.join(KINDS))
  if not torch.cuda.is_available():
    raise SystemExit('bench_augment.py needs a CUDA device')
  torch.cuda.set_device(0)
  emit(metric='device', **bench_train.device_info())
  for kind in kinds:
    agents = {pad: make_agent(kind, pad, a.capacity) for pad in (0, PAD)}
    for ag in agents.values():
      for _ in range(a.warmup):
        ag.learn()
    times = {pad: [] for pad in agents}
    for _ in range(a.rounds):
      for pad, ag in agents.items():
        times[pad].append(time_steps(ag, a.steps))
    med = {pad: float(np.median(t)) for pad, t in times.items()}
    emit(metric='learn_step_us', kind=kind, dueling=kind == 'double_q', pad0=round(med[0], 2), pad4=round(med[PAD], 2),
         overhead_us=round(med[PAD] - med[0], 2), rounds_pad0=[round(t, 2) for t in times[0]],
         rounds_pad4=[round(t, 2) for t in times[PAD]])
    del agents
    torch.cuda.empty_cache()
  us, gbs = shift_kernel(a.kernel_reps)
  emit(metric='shift_kernel', batch=32, obs='84x84x4', pad=PAD, us=round(us, 3), bytes=2 * 2 * 32 * 84 * 84 * 4,
       gb_per_s=round(gbs, 1))
  emit(metric='device_after', **bench_train.device_info())


if __name__ == '__main__':
  main()
