"""K independent learners (each with its own replay shard, parameters, optimizer state, CUDA stream and CUDA graph) on
ONE GPU: aggregate learner grad-steps/s versus K.

A single batch-32 learner step is a dependent chain of ~35 short kernels, most of which cover a fraction of the 132 SMs
(the sampler is one block, the loss kernels 32, the tensor-core conv kernels 35-128 CTAs): K shards interleave on the idle
SMs.  Each shard is exactly the object bench.py times (same agent class, same fused step); nothing is shared between
shards, so per-learner results are the single-learner results (tests/test_gpu_agent.py covers those).

  python tools/bench_multi_learner.py --agent rainbow --learners 1,2,3 [--capacity 250000] [--steps 1500]
Prints one JSON line per K.  The default capacity (14.1 GB of replay per shard) lets three shards share an 80 GB H100;
K shards of 1M transitions need 56.4 GB each."""

import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402


def run(agent, k, capacity, steps, warmup):
  dev = torch.device('cuda', 0)
  torch.cuda.set_device(0)
  shards = []
  for j in range(k):
    args = argparse.Namespace(agent=agent, capacity=capacity, batch=32, seed=1 + 17 * j, no_graph=False)
    stream = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(stream):
      ag, rep = bench.build_agent(args, j, dev)
      draws = torch.as_tensor(np.stack([ag.host_draws() for _ in range(64)]), device=dev)
      for i in range(3):
        ag.learn_from_device_draws(draws[i])          # eager step + graph capture on this shard's stream
    stream.synchronize()
    shards.append((ag, rep, stream, draws))
  torch.cuda.synchronize()

  def sweep(n):
    for i in range(n):
      for ag, rep, stream, draws in shards:
        with torch.cuda.stream(stream):
          ag.learn_from_device_draws(draws[i % 64])

  sweep(warmup)
  torch.cuda.synchronize()
  e0 = [torch.cuda.Event(enable_timing=True) for _ in shards]
  e1 = [torch.cuda.Event(enable_timing=True) for _ in shards]
  for (ag, rep, stream, draws), ev in zip(shards, e0):
    ev.record(stream)
  sweep(steps)
  for (ag, rep, stream, draws), ev in zip(shards, e1):
    ev.record(stream)
  torch.cuda.synchronize()
  ms = max(a.elapsed_time(b) for a, b in zip(e0, e1))
  for ag, rep, stream, draws in shards:
    ag.check_device_flags()
  value = k * steps / (ms / 1e3)
  line = {'metric': 'learner_grad_steps_per_sec (aggregate of K learners on one GPU)', 'learners': k, 'agent': agent,
          'value': value, 'per_learner': value / k, 'ms_per_step_per_learner': ms / steps, 'steps': steps, 'warmup': warmup,
          'replay_capacity': capacity, 'replay_gb_total': k * capacity * 2 * 84 * 84 * 4 / 1e9,
          'timing': 'CUDA events on each shard stream, max over shards; one host thread submits the K graph replays round-robin'}
  print(json.dumps(line), flush=True)
  del shards
  torch.cuda.empty_cache()
  return value


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--agent', default='rainbow')
  ap.add_argument('--learners', default='1,2,3')
  ap.add_argument('--capacity', type=int, default=250000)
  ap.add_argument('--steps', type=int, default=1500)
  ap.add_argument('--warmup', type=int, default=100)
  a = ap.parse_args()
  ks = [int(x) for x in a.learners.split(',')]
  need = max(ks) * a.capacity * 2 * 84 * 84 * 4
  free, _ = torch.cuda.mem_get_info()
  if need > free:
    ap.error('%d shards of %d transitions need %.1f GB of replay, %.1f GB of HBM is free' % (max(ks), a.capacity, need / 1e9, free / 1e9))
  for k in ks:
    run(a.agent, k, a.capacity, a.steps, a.warmup)


if __name__ == '__main__':
  main()
