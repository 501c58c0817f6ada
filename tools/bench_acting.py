"""Batched acting throughput: E environment streams per tick through BatchedEpsilonGreedyActor (one network evaluation and
ONE device-to-host copy of E actions per tick) versus the single-observation path (one D2H sync per decision).
  python tools/bench_acting.py --agent dqn --streams 32 [--ticks 300]
Rainbow's two noise modes, alternated in one run (decisions/s of each round), then kernel times in a separate run:
  python tools/bench_acting.py --agent rainbow --per-stream-noise [--rounds 3]
  python tools/bench_acting.py --agent rainbow --per-stream-noise --profile OUT_DIR
The acting context against act_batch on a learner of batch E (the only single-call option without it), alternated per
stream count, then kernel times per tick in a separate run:
  python tools/bench_acting.py --agent dqn --compare-actor --streams 32,128,256,512 [--rounds 3] [--profile OUT_DIR]
Observations are device-resident frame stacks (what processors.BatchedAtariPreprocessor hands out)."""

import argparse
import collections
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
  """Name and power limit of the device the numbers were measured on."""
  out = {'gpu': torch.cuda.get_device_name()}
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader', '-i',
                        str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    out['power_limit'], out['max_sm_clock'] = [s.strip() for s in q.split(',')][:2]
  except (OSError, ValueError, subprocess.SubprocessError):
    out['power_limit'] = 'unknown'
  return out


def decisions_per_s(actor, obs, ticks):
  torch.cuda.synchronize()
  t0 = time.perf_counter()
  for _ in range(ticks):
    actor.step(obs)
  torch.cuda.synchronize()
  return obs.shape[0] * ticks / (time.perf_counter() - t0)


def noise_modes(L, E, obs, a):
  """Rainbow decisions/s with one noise apply shared by the tick's streams and with one apply per stream, alternated."""
  from dqn_zoo_b200 import agent as agent_lib
  actors = {mode: agent_lib.BatchedEpsilonGreedyActor(L, E, exploration_epsilon=0.01, rng_key=[0, 3],
                                                      per_stream_noise=mode == 'per_stream')
            for mode in ('shared', 'per_stream')}
  for actor in actors.values():
    for _ in range(20):
      actor.step(obs)
  if a.profile:
    return profile_modes(actors, obs, a)
  rates = {mode: [] for mode in actors}
  for _ in range(a.rounds):
    for mode, actor in actors.items():
      rates[mode].append(round(decisions_per_s(actor, obs, a.ticks), 1))
  print(json.dumps(dict({'metric': 'rainbow acting decisions per second by noise mode (device-resident observations)',
                         'streams': E, 'ticks_per_round': a.ticks, 'shared_noise_decisions_per_s': rates['shared'],
                         'per_stream_noise_decisions_per_s': rates['per_stream']}, **card())))


def profile_modes(actors, obs, a):
  """Kernel times per tick of each mode from torch.profiler CUDA activity (a run of its own: tracing slows the host).
  noisy1_fwd is the noisy GEMM launch with 512 / 64 = 8 column tiles, noisy2_fwd the one with ceil(A * atoms / 64)."""
  os.makedirs(a.profile, exist_ok=True)
  result = dict({'metric': 'rainbow acting kernel time per tick (us), torch.profiler', 'streams': obs.shape[0],
                 'ticks': a.ticks}, **card())
  for mode, actor in actors.items():
    path = os.path.join(a.profile, 'acting_%s.json' % mode)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
      for _ in range(a.ticks):
        actor.step(obs)
      torch.cuda.synchronize()
    prof.export_chrome_trace(path)
    per_kernel = collections.defaultdict(float)
    layers = collections.defaultdict(float)
    with open(path) as f:
      events = json.load(f)['traceEvents']
    for ev in events:
      if ev.get('cat') != 'kernel':
        continue
      name = ev['name']
      short = name.replace('(anonymous namespace)::', '').replace('void ', '').split('(')[0].split('<')[0].split('::')[-1]
      per_kernel[short] += ev['dur'] / a.ticks
      if short == 'gemm_nn_rownoise_kernel' or (short == 'gemm_nn_kernel' and 'true>' in name):
        layers['noisy1_fwd' if ev['args']['grid'][0] == 8 else 'noisy2_fwd'] += ev['dur'] / a.ticks
    result[mode] = {'noisy1_fwd_us': round(layers['noisy1_fwd'], 2), 'noisy2_fwd_us': round(layers['noisy2_fwd'], 2),
                    'kernels_us': {k: round(v, 2) for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1])}}
  print(json.dumps(result))


def kernel_times(fn, ticks, path):
  """Kernel time per tick (us) by kernel name, from torch.profiler CUDA activity written to `path`."""
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(ticks):
      fn()
    torch.cuda.synchronize()
  prof.export_chrome_trace(path)
  per_kernel = collections.defaultdict(float)
  with open(path) as f:
    for ev in json.load(f)['traceEvents']:
      if ev.get('cat') == 'kernel':
        short = ev['name'].replace('(anonymous namespace)::', '').replace('void ', '').split('(')[0].split('<')[0].split('::')[-1]
        per_kernel[short] += ev['dur'] / ticks
  return {'total_us': round(sum(per_kernel.values()), 2),
          'kernels_us': {k: round(v, 2) for k, v in sorted(per_kernel.items(), key=lambda kv: -kv[1])}}


def compare_actor(a, streams):
  """Per stream count E, alternated within each round: (a) the acting context of a batch-32 learner, (b) act_batch on
  a learner of batch E, and at E = 32 also (c) act_batch on the batch-32 learner.  A tick is one act call (greedy
  for half the streams: epsilon 0.5 with device uniforms) and the D2H of its E actions.  Rainbow: one shared noise
  apply; IQN: one tau row per stream.  Randomness is drawn once, outside the timed ticks."""
  from dqn_zoo_b200 import learner as dl
  from oracle import learner_oracle as lo
  net = dl.NetworkSpec(a.agent, 6)
  params = lo.init_params(lo.NetSpec(a.agent, 6), 2)

  def learner(batch):
    L = dl.Learner(net, batch_size=batch)
    L.set_params(params, also_target=True)
    return L

  L32 = learner(32)
  rs = np.random.RandomState(0)
  ticks = {}
  keep = []
  for E in streams:
    obs = torch.randint(0, 256, (E, 84, 84, 4), dtype=torch.uint8, device='cuda')
    explore = torch.as_tensor(rs.uniform(size=(2, E)).astype(np.float32), device='cuda')
    kw = {}
    if dl.uses_iqn_network(a.agent):
      kw['taus'] = torch.as_tensor(rs.uniform(size=(E, net.tau_samples_policy)).astype(np.float32), device='cuda')
    if a.agent == 'rainbow':
      L32.generate_randomness(1)
      kw['noise'] = L32.noise[:L32.noise_stride].clone()
    actor = L32.actor(E)
    LE = L32 if E == 32 else learner(E)
    keep += [actor, LE]

    def tick(act, obs=obs, explore=explore, kw=kw):
      actions, _ = act(obs, epsilon=0.5, explore=explore, **kw)
      actions.cpu()
    ticks[(E, 'actor_on_batch32_learner')] = lambda tick=tick, actor=actor: tick(actor.act)
    ticks[(E, 'act_batch_on_batch%d_learner' % E)] = lambda tick=tick, LE=LE: tick(LE.act_batch)
  for fn in ticks.values():
    for _ in range(20):
      fn()
  result = dict({'metric': 'acting decisions per second: acting context vs act_batch (device-resident observations)',
                 'agent': a.agent, 'ticks_per_round': a.ticks, 'rounds': a.rounds}, **card())
  if a.profile:
    os.makedirs(a.profile, exist_ok=True)
    result['metric'] = 'acting kernel time per tick (us), torch.profiler'
    result['kernel_times'] = {'E=%d %s' % k: kernel_times(fn, a.ticks, os.path.join(a.profile, 'acting_E%d_%s.json' % k))
                              for k, fn in ticks.items()}
    print(json.dumps(result))
    return
  rates = collections.defaultdict(list)
  for _ in range(a.rounds):
    for (E, mode), fn in ticks.items():
      torch.cuda.synchronize()
      t0 = time.perf_counter()
      for _ in range(a.ticks):
        fn()
      torch.cuda.synchronize()
      rates['E=%d %s' % (E, mode)].append(round(E * a.ticks / (time.perf_counter() - t0), 1))
  result['decisions_per_s'] = dict(rates)
  print(json.dumps(result))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--agent', default='dqn')
  ap.add_argument('--streams', default='32', help='streams per tick; with --compare-actor a comma-separated list')
  ap.add_argument('--ticks', type=int, default=300)
  ap.add_argument('--per-stream-noise', action='store_true',
                  help='rainbow: compare one noise apply per tick with one apply per stream, alternated')
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--compare-actor', action='store_true',
                  help='the acting context of a batch-32 learner vs act_batch on a learner of batch E, alternated')
  ap.add_argument('--profile', default=None,
                  help='with --per-stream-noise or --compare-actor: kernel times from torch.profiler, traces here')
  a = ap.parse_args()
  if a.per_stream_noise and a.agent != 'rainbow':
    ap.error('--per-stream-noise needs --agent rainbow')
  streams = [int(x) for x in str(a.streams).split(',')]
  if len(streams) > 1 and not a.compare_actor:
    ap.error('a list of stream counts needs --compare-actor')
  if not torch.cuda.is_available():
    raise SystemExit('bench_acting.py needs a CUDA device')
  if a.compare_actor:
    return compare_actor(a, streams)
  a.streams = streams[0]
  from dqn_zoo_b200 import agent as agent_lib
  from dqn_zoo_b200 import learner as dl
  from oracle import learner_oracle as lo
  L = dl.Learner(dl.NetworkSpec(a.agent, 6), batch_size=max(32, a.streams))
  L.set_params(lo.init_params(lo.NetSpec(a.agent, 6), 2), also_target=True)
  E = a.streams
  obs = torch.randint(0, 256, (E, 84, 84, 4), dtype=torch.uint8, device='cuda')
  if a.per_stream_noise:
    return noise_modes(L, E, obs, a)
  actor = agent_lib.BatchedEpsilonGreedyActor(L, E, exploration_epsilon=0.01, rng_key=[0, 3])
  for _ in range(20):
    actor.step(obs)
  batched = decisions_per_s(actor, obs, a.ticks)
  # single-observation path: q_values + D2H per decision
  noise = taus = None
  if a.agent == 'rainbow':
    noise = L.noise
  if dl.uses_iqn_network(a.agent):
    taus = L.taus[:64]
  for _ in range(20):
    L.q_values(obs[0], taus=taus, noise=noise).cpu()
  t0 = time.perf_counter()
  n = max(100, a.ticks)
  for i in range(n):
    L.q_values(obs[i % E], taus=taus, noise=noise).cpu()
  single = n / (time.perf_counter() - t0)
  print(json.dumps({'metric': 'acting decisions per second (network evaluation + action choice, device-resident observations)',
                    'agent': a.agent, 'streams': E, 'batched_decisions_per_s': batched, 'ms_per_tick': 1e3 * E / batched,
                    'single_observation_decisions_per_s': single, 'speedup': batched / single,
                    'd2h_bytes_per_tick': 4 * E, 'h2d_bytes_per_tick': 8 * E}))


if __name__ == '__main__':
  main()
