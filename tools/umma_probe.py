"""Bring-up probe of the TMA-fed tensor-core GEMM family: runs every operand path and prints the relative error of
each (no assertions), plus a few hints when a path is wrong.  `python tools/umma_probe.py` on an H100."""

import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tests'))


def main():
  import torch
  from test_gpu_umma import operands, rel, run_umma
  for (MI, NJ, R) in [(128, 32, 32), (128, 32, 64), (128, 64, 256), (200, 52, 100), (512, 32, 3136)]:
    Am, Bm = operands(MI, NJ, R, MI + NJ + R)
    want = Am.astype(np.float64) @ Bm.astype(np.float64).T
    for convert in (0, 1):
      for a_mn, b_mn in ((0, 0), (1, 0), (0, 1), (1, 1)):
        try:
          got, _, _ = run_umma(Am, Bm, a_mn, b_mn, convert)
          e = rel(got, want)
          hint = ''
          if not (e < 3e-6):
            nan = int(np.isnan(got).sum())
            # is it a 1xTF32 result (lo terms lost)?  a permutation of rows / columns?
            h = lambda x: (x.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32).astype(np.float64)
            e1 = rel(got, h(Am) @ h(Bm).T)
            hint = ' nan=%d rel_vs_1xtf32=%.2e |got|=%.3e |want|=%.3e got[0,:4]=%s want[0,:4]=%s' % (
                nan, e1, np.linalg.norm(np.nan_to_num(got)), np.linalg.norm(want), np.round(got[0, :4], 3), np.round(want[0, :4], 3))
          print('MI=%d NJ=%d R=%d convert=%d a_mn=%d b_mn=%d rel=%.3e%s' % (MI, NJ, R, convert, a_mn, b_mn, e, hint), flush=True)
        except Exception as ex:  # pylint: disable=broad-except
          print('MI=%d NJ=%d R=%d convert=%d a_mn=%d b_mn=%d FAILED: %s' % (MI, NJ, R, convert, a_mn, b_mn, ex), flush=True)
          torch.cuda.synchronize()


if __name__ == '__main__':
  main()
