"""Per-stage timeline of CTA 0 of one TMA-fed tensor-core launch inside a learner step.

For every shared-memory stage of the launch's first CTA it prints, in SM clock cycles:
  wait  = data ready - TMA issued   (how long the stage's operands took to land after the producer issued them)
  mma   = consumed - data ready     (how long the MMA warps held the stage before releasing it to the producer)
A launch whose `mma` column dominates is bound by the MMA loop; one whose `wait` column dominates is bound by the
operand delivery (TMA / L2).

conv1_fwd stamps per 128-pixel output tile instead (csrc/dz_umma_net.cu): for every tile of CTA 0
  wait  = rows landed - row copies issued
  mma   = tile's MMAs done - rows landed     (includes the byte -> tf32 conversion, which the MMAs wait for)
  store = tile stored - tile's MMAs done    (ReLU + tf32 hi/lo epilogue)

  python tools/umma_stage_trace.py --agent rainbow --tags conv1_fwd,conv2_fwd,conv3_fwd [--graph] [--steps 8]"""

import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402

# clock-stamp slots written by CTA 0 of the traced launch (csrc/dz_umma.cuh)
ISSUED, READY, CONSUMED, EPILOGUE, STORED, EXIT, ENTRY = 0, 64, 128, 320, 321, 322, 323
# conv1_fwd's per-tile slots: row copies issued, rows landed, tile's MMAs done, tile stored (exit / entry as above)
C1_ISSUED, C1_LANDED, C1_MMA_DONE, C1_STORED = 0, 64, 192, 256


def tile_table(t):
  """Per-tile (issued, landed, MMAs done, stored) stamps of conv1_fwd relative to the kernel entry, plus the exit."""
  n = int((t[C1_ISSUED:C1_ISSUED + 64] != 0).sum())
  t0 = int(t[ENTRY])
  rows = [tuple(int(t[s + i]) - t0 for s in (C1_ISSUED, C1_LANDED, C1_MMA_DONE, C1_STORED)) for i in range(n)]
  return rows, int(t[EXIT]) - t0


def print_tiles(tag, agent, t):
  rows, exit_ = tile_table(t)
  if not rows:
    print('== %s: no stamps' % tag)
    return
  print('== %s (%s): %d tiles | exit at %d cycles' % (tag, agent, len(rows), exit_))
  print('  %5s %9s %9s %9s %9s %8s %8s %8s' % ('tile', 'issued', 'landed', 'mma_done', 'stored', 'wait', 'mma', 'store'))
  for s, (i, r, m, st) in enumerate(rows):
    print('  %5d %9d %9d %9d %9d %8d %8d %8d' % (s, i, r, m, st, r - i, m - r, st - m))
  mma = np.array([r[2] - r[1] for r in rows])
  print('  median mma %d cycles; first issue -> last store %d cycles' % (int(np.median(mma)), rows[-1][3] - rows[0][0]))


def stage_table(t):
  """Per-stage (issued, ready, consumed) stamps relative to the kernel entry, plus the summary stamps."""
  n = int((t[ISSUED:ISSUED + 64] != 0).sum())
  t0 = int(t[ENTRY])
  rows = [(int(t[ISSUED + s]) - t0, int(t[READY + s]) - t0, int(t[CONSUMED + s]) - t0) for s in range(n)]
  return rows, {'epilogue': int(t[EPILOGUE]) - t0, 'stored': int(t[STORED]) - t0, 'exit': int(t[EXIT]) - t0}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--agent', default='rainbow')
  ap.add_argument('--tags', default='conv2_fwd,conv3_fwd')
  ap.add_argument('--graph', action='store_true', help='stamp inside CUDA-graph replays (steady-state cache conditions)')
  ap.add_argument('--steps', type=int, default=8, help='learner steps run with the trace on (the last one is reported)')
  a = ap.parse_args()
  from dqn_zoo_b200 import _lib
  args = argparse.Namespace(agent=a.agent, capacity=131072, batch=32, seed=1, no_graph=not a.graph)
  torch.cuda.set_device(0)
  ag, _ = bench.build_agent(args, 0, torch.device('cuda', 0))
  for _ in range(5):
    ag.learn()
  torch.cuda.synchronize()
  for tag in a.tags.split(','):
    tr = torch.zeros(512, dtype=torch.int64, device='cuda')
    _lib.call('dz_test_learner_trace', ag.learner._h, tag.encode(), tr.data_ptr())
    if a.graph:
      ag._graph = None          # recapture with the trace pointer baked into the launch
    for _ in range(max(1, a.steps)):
      ag.learn()
    torch.cuda.synchronize()
    _lib.call('dz_test_learner_trace', ag.learner._h, b'', 0)
    if a.graph:
      ag._graph = None
    if tag == 'conv1_fwd':
      print_tiles(tag, a.agent, tr.cpu().numpy())
      continue
    rows, tail = stage_table(tr.cpu().numpy())
    if not rows:
      print('== %s: no stamps (is the tag a TMA-fed tensor-core launch of this agent?)' % tag)
      continue
    wait = np.array([r[1] - r[0] for r in rows])
    mma = np.array([r[2] - r[1] for r in rows])
    print('== %s (%s): %d stages | epilogue at %d, stores issued at %d, exit at %d cycles' %
          (tag, a.agent, len(rows), tail['epilogue'], tail['stored'], tail['exit']))
    print('  %5s %9s %9s %9s %8s %8s' % ('stage', 'issued', 'ready', 'consumed', 'wait', 'mma'))
    for s, (i, r, c) in enumerate(rows):
      print('  %5d %9d %9d %9d %8d %8d' % (s, i, r, c, r - i, c - r))
    print('  median wait %d, median mma %d cycles; mainloop %d cycles' %
          (int(np.median(wait)), int(np.median(mma)), rows[-1][2] - rows[0][0]))


if __name__ == '__main__':
  main()
