"""Debug: clock-stamp timeline of CTA 0 of one tensor-core launch inside a rainbow / dqn learner step.
  python tools/umma_trace.py --agent rainbow --tag conv2_fwd"""

import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--agent', default='rainbow')
  ap.add_argument('--graph', action='store_true', help='stamp inside CUDA-graph replays (steady-state cache / DRAM conditions)')
  ap.add_argument('--tags', default='conv2_fwd,conv3_fwd,fc1_fwd,fc1_dgrad,conv3_dgrad,conv2_dgrad,conv3_wgrad,conv2_wgrad')
  a = ap.parse_args()
  from dqn_zoo_b200 import _lib
  args = argparse.Namespace(agent=a.agent, capacity=131072, batch=32, seed=1, no_graph=not a.graph)
  torch.cuda.set_device(0)
  ag, rep = bench.build_agent(args, 0, torch.device('cuda', 0))
  for _ in range(5):
    ag.learn()
  torch.cuda.synchronize()
  for tag in a.tags.split(','):
    tr = torch.zeros(512, dtype=torch.int64, device='cuda')
    _lib.call('dz_test_learner_trace', ag.learner._h, tag.encode(), tr.data_ptr())
    if a.graph:
      ag._graph = None          # recapture with the trace pointer baked into the launch
      for _ in range(8):
        ag.learn()
    else:
      ag.learn()
    torch.cuda.synchronize()
    _lib.call('dz_test_learner_trace', ag.learner._h, b'', 0)
    t = tr.cpu().numpy()
    t0 = t[323]
    rel = lambda x: int(x - t0) if x else -1
    if tag.startswith('conv1'):
      nt = int((t[192:256] != 0).sum())
      print('== %s: tiles %d | exit %d' % (tag, nt, rel(t[322])))
      for name, o in (('rows issued', 0), ('rows landed', 64), ('tile mma done', 192), ('tile stored', 256)):
        print('  %-12s:' % name, [rel(x) for x in t[o:o + nt]])
      continue
    n = int((t[:64] != 0).sum())
    print('== %s: stages %d | setup done %d | epilogue %d stores %d exit %d' % (tag, n, rel(t[324]), rel(t[320]), rel(t[321]), rel(t[322])))
    print('  tma issued :', [rel(x) for x in t[:n]])
    print('  data ready :', [rel(x) for x in t[64:64 + n]])
    print('  consumed   :', [rel(x) for x in t[128:128 + n]])


if __name__ == '__main__':
  main()
