"""GPU: the TMA-fed tensor-core GEMM family (csrc/dz_umma.cuh) against float64 numpy, through the C-ABI self-test hook.

Covers every operand path the learner uses: K-major and MN-major sources (the descriptor transposes), pre-split
tf32 hi/lo operands (activations) and raw fp32 tiles split in shared memory by the converter warps (weights),
reduction scaling (noisy sigma weights), ragged extents (TMA zero fill), both epilogues.  Expected accuracy: ~2^-21
relative per product (3xTF32); a plain 1xTF32 product would be ~5e-4 and fail."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def run_umma(Am, Bm, a_mn, b_mn, convert, scale=None, stages=0, epi_rows=False, bias=None, relu=False):
  """Am: logical A(i, r) [MI][R]; Bm: logical B(j, r) [NJ][R].  Returns (C, hi, lo) as float64 numpy."""
  from dqn_zoo_b200 import _lib
  dev = 'cuda'
  MI, R = Am.shape
  NJ = Bm.shape[0]
  dA = torch.as_tensor(np.ascontiguousarray(Am.T if a_mn else Am), device=dev)
  dB = torch.as_tensor(np.ascontiguousarray(Bm.T if b_mn else Bm), device=dev)
  out = torch.full((MI, NJ), float('nan'), dtype=torch.float32, device=dev)
  hi = torch.full((MI, NJ), float('nan'), dtype=torch.float32, device=dev)
  lo = torch.full((MI, NJ), float('nan'), dtype=torch.float32, device=dev)
  sc = None if scale is None else torch.as_tensor(scale, device=dev).contiguous()
  bs = None if bias is None else torch.as_tensor(bias, device=dev).contiguous()
  _lib.call('dz_test_umma_gemm', dA.data_ptr(), int(a_mn), dB.data_ptr(), int(b_mn), MI, NJ, R, int(convert),
            0 if sc is None else sc.data_ptr(), stages, int(epi_rows), 0 if bs is None else bs.data_ptr(), int(relu),
            out.data_ptr(), hi.data_ptr() if epi_rows else 0, lo.data_ptr() if epi_rows else 0,
            torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  return out.cpu().numpy().astype(np.float64), hi.cpu().numpy().astype(np.float64), lo.cpu().numpy().astype(np.float64)


def rel(got, want):
  return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


def operands(MI, NJ, R, seed):
  rs = np.random.RandomState(seed)
  return rs.standard_normal((MI, R)).astype(np.float32), rs.standard_normal((NJ, R)).astype(np.float32)


@pytest.mark.parametrize('convert', [0, 1])
@pytest.mark.parametrize('a_mn,b_mn', [(0, 0), (1, 0), (0, 1), (1, 1)])
@pytest.mark.parametrize('MI,NJ,R', [(128, 32, 64), (128, 64, 256), (200, 52, 100), (392, 64, 576), (512, 32, 3136)])
def test_operand_paths(MI, NJ, R, a_mn, b_mn, convert):
  Am, Bm = operands(MI, NJ, R, MI + NJ + R)
  want = Am.astype(np.float64) @ Bm.astype(np.float64).T
  got, _, _ = run_umma(Am, Bm, a_mn, b_mn, convert)
  assert rel(got, want) < 3e-6, rel(got, want)


@pytest.mark.parametrize('a_mn', [0, 1])
def test_reduction_scale_in_the_converter(a_mn):
  Am, Bm = operands(256, 32, 416, 7)
  s = np.random.RandomState(8).uniform(0.5, 1.5, 416).astype(np.float32)
  want = (Am.astype(np.float64) * s.astype(np.float64)[None, :]) @ Bm.astype(np.float64).T
  got, _, _ = run_umma(Am, Bm, a_mn, 0, 1, scale=s)
  assert rel(got, want) < 3e-6, rel(got, want)


@pytest.mark.parametrize('stages', [1, 2, 4])
def test_row_epilogue_bias_relu_and_split_outputs(stages):
  """16 reduction stages through a ring of 1, 2 or 4 slots: every slot is refilled after its barrier phase flips."""
  Am, Bm = operands(300, 64, 512, 11)
  bias = np.random.RandomState(12).standard_normal(64).astype(np.float32)
  want = np.maximum(Am.astype(np.float64) @ Bm.astype(np.float64).T + bias.astype(np.float64)[None, :], 0.0)
  got, hi, lo = run_umma(Am, Bm, 0, 0, 0, stages=stages, epi_rows=True, bias=bias, relu=True)
  assert rel(got, want) < 3e-6, rel(got, want)
  # hi is a tf32 number (13 low mantissa bits clear), hi + lo reproduces the fp32 output to 2^-22
  assert np.all((hi.astype(np.float32).view(np.uint32) & 0x1FFF) == 0)
  assert np.all((lo.astype(np.float32).view(np.uint32) & 0x1FFF) == 0)
  np.testing.assert_allclose(hi + lo, got, rtol=3e-7, atol=1e-30)


@pytest.mark.parametrize('kind', ['dqn', 'double_q', 'c51', 'qrdqn', 'rainbow', 'iqn'])
def test_tcgen05_path_is_active_at_the_baseline_geometry(kind):
  """The 84x84x4, batch-32 learner of BASELINE.json must run its torso (and 3136->512 layer) on the tensor-core kernels:
  a silent fall-back to the fp32-FMA kernels (geometry check, shared-memory budget) would keep every parity test green."""
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  L = dl.Learner(dl.NetworkSpec(kind, 6), batch_size=32)
  _lib.call('dz_test_learner_trace', L._h, b'', 0)   # raises ValueError when the path is not active
