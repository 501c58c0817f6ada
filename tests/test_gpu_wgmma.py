"""GPU: the wgmma kernel of the TMA-fed tensor-core GEMM family (csrc/dz_umma.cuh, wgmma_gemm_kernel).

Launches whose operands are both K-major tf32 hi/lo pairs (conv2 / conv3 forward and input gradient) run on
warpgroup MMAs; every other launch keeps the warp-level mma.sync kernel.  Both kernels form each k-step's three
products from zero in the same order and add them into the fp32 sums in the same order, so on the same inputs they
are expected to agree bit for bit; each is also checked against float64."""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

AUTO, MMA_SYNC, WGMMA = 0, 1, 2


def run_path(Am, Bm, path, stages=0, epi_rows=False, bias=None, relu=False, a_mn=0):
  """K-major, pre-split operands (the activation layout).  Returns (C, hi, lo) as float32 numpy."""
  from dqn_zoo_b200 import _lib
  dev = 'cuda'
  MI, R = Am.shape
  NJ = Bm.shape[0]
  dA = torch.as_tensor(np.ascontiguousarray(Am.T if a_mn else Am), device=dev)
  dB = torch.as_tensor(np.ascontiguousarray(Bm), device=dev)
  out = torch.full((MI, NJ), float('nan'), dtype=torch.float32, device=dev)
  hi = torch.full((MI, NJ), float('nan'), dtype=torch.float32, device=dev)
  lo = torch.full((MI, NJ), float('nan'), dtype=torch.float32, device=dev)
  bs = None if bias is None else torch.as_tensor(bias, device=dev).contiguous()
  _lib.call('dz_test_umma_gemm_path', dA.data_ptr(), int(a_mn), dB.data_ptr(), 0, MI, NJ, R, 0, 0, stages, int(epi_rows),
            0 if bs is None else bs.data_ptr(), int(relu), out.data_ptr(), hi.data_ptr() if epi_rows else 0,
            lo.data_ptr() if epi_rows else 0, path, torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  return out.cpu().numpy(), hi.cpu().numpy(), lo.cpu().numpy()


def rel(got, want):
  return float(np.linalg.norm(got.astype(np.float64) - want) / max(np.linalg.norm(want), 1e-30))


def operands(MI, NJ, R, seed):
  rs = np.random.RandomState(seed)
  return rs.standard_normal((MI, R)).astype(np.float32), rs.standard_normal((NJ, R)).astype(np.float32)


# valid rows per 128-row tile of the learner's launches (conv3 input gradient 45, conv2 forward 81, conv3 forward 98,
# conv2 input gradient 100) and a multi-tile case; NJ / R as in those launches
@pytest.mark.parametrize('MI', [45, 81, 98, 100, 300])
@pytest.mark.parametrize('NJ,R', [(64, 512), (32, 576), (32, 256), (64, 576)])
def test_both_paths_match_float64_and_each_other(MI, NJ, R):
  Am, Bm = operands(MI, NJ, R, MI * 7 + NJ + R)
  want = Am.astype(np.float64) @ Bm.astype(np.float64).T
  got_sync, _, _ = run_path(Am, Bm, MMA_SYNC)
  got_wg, _, _ = run_path(Am, Bm, WGMMA)
  assert rel(got_sync, want) < 3e-6, rel(got_sync, want)
  assert rel(got_wg, want) < 3e-6, rel(got_wg, want)
  np.testing.assert_array_equal(got_wg, got_sync)
  got_auto, _, _ = run_path(Am, Bm, AUTO)
  np.testing.assert_array_equal(got_auto, got_wg)


@pytest.mark.parametrize('stages', [1, 2, 4])
def test_row_epilogue_on_both_paths(stages):
  """16 reduction stages through a ring of 1, 2 or 4 slots, bias + ReLU + tf32 hi/lo outputs."""
  Am, Bm = operands(300, 64, 512, 21)
  bias = np.random.RandomState(22).standard_normal(64).astype(np.float32)
  want = np.maximum(Am.astype(np.float64) @ Bm.astype(np.float64).T + bias.astype(np.float64)[None, :], 0.0)
  res = {}
  for path in (MMA_SYNC, WGMMA):
    got, hi, lo = run_path(Am, Bm, path, stages=stages, epi_rows=True, bias=bias, relu=True)
    assert rel(got, want) < 3e-6, (path, rel(got, want))
    assert np.all((hi.view(np.uint32) & 0x1FFF) == 0)
    assert np.all((lo.view(np.uint32) & 0x1FFF) == 0)
    res[path] = (got, hi, lo)
  for a, b in zip(res[WGMMA], res[MMA_SYNC]):
    np.testing.assert_array_equal(a, b)


def test_wgmma_path_refuses_mn_major_operands():
  """tf32 wgmma reads only K-major operands from shared memory: forcing it on an MN-major problem is an error."""
  Am, Bm = operands(128, 32, 64, 5)
  with pytest.raises(ValueError):
    run_path(Am, Bm, WGMMA, a_mn=1)


@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_learner_conv_launches_run_on_wgmma(kind):
  """At 84x84x4 and batch 32 the four K-major launches take the wgmma kernel (no silent fall-back to mma.sync); the
  3136 -> 512 layer, whose weights arrive MN-major, stays on mma.sync."""
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  L = dl.Learner(dl.NetworkSpec(kind, 6), batch_size=32)
  path = ctypes.c_int32(0)
  for tag in ('conv2_fwd', 'conv3_fwd', 'conv3_dgrad', 'conv2_dgrad'):
    _lib.call('dz_test_learner_mma_path', L._h, tag.encode(), ctypes.byref(path))
    assert path.value == WGMMA, (kind, tag, path.value)
  for tag in ('conv3_wgrad', 'conv2_wgrad') + (() if kind == 'iqn' else ('fc1_fwd', 'fc1_dgrad')):
    _lib.call('dz_test_learner_mma_path', L._h, tag.encode(), ctypes.byref(path))
    assert path.value == MMA_SYNC, (kind, tag, path.value)
