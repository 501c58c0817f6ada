"""GPU: the packed-operand tensor-core GEMM (csrc/dz_tcp.cuh: tc_pack_kernel + tc_pgemm_kernel) against float64 numpy,
through the C-ABI self-test hook dz_test_tc_pgemm.

This GEMM carries IQN's embedding layer, its 3136 -> 512 layer and their backward passes.  The hook packs both operands
from plain fp32 matrices into hi/lo TF32 tile images (in caller memory, so the images are checked here too) and runs
D[i,j] = sum_r A(i,r) B(j,r) with the plain epilogue (split partials, or bias + ReLU).  Expected accuracy: ~2^-21
relative per product (3xTF32, round-to-nearest accumulation); a 1xTF32 product would be ~5e-4 and fail."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

KB = 16        # reduction elements per k-block (kPkKB)
GUARD = 64     # floats of sentinel on each side of the output
SENTINEL = np.float32(-3.0e38)


def pk_index(row, r, rg):
  """Float index of element (row, r) of a tile image with rg = rows_pad / 8 row groups (pk_index, dz_internal.cuh)."""
  return (((r // 16) * rg + row // 8) * 4 + (r % 16) // 4) * 32 + (row % 8) * 4 + r % 4


def image(flat, rows_pad, red_pad):
  """[rows_pad][red_pad] view of a tile image."""
  row, r = np.meshgrid(np.arange(rows_pad), np.arange(red_pad), indexing='ij')
  return flat[pk_index(row, r, rows_pad // 8)]


def stored(M, red_contig, odd_ld):
  """The source layout of logical M[rows][red]: red_contig 1 -> [rows][ld], 0 -> [red][ld].  ld is the contiguous
  extent, or with odd_ld the next larger value that is not a multiple of 4 (rows of a source then start off 16-byte
  alignment, which the pack kernel must read with scalar loads)."""
  X = M if red_contig else M.T
  ld = X.shape[1]
  if odd_ld:
    ld += 1
    while ld % 4 == 0:
      ld += 1
  out = np.full((X.shape[0], ld), np.nan, dtype=np.float32)
  out[:, :X.shape[1]] = X
  return out


def run_pgemm(Am, Bm, a_rc=1, b_rc=1, ones=False, splits=1, bias=None, relu=False, transposed=False, offset=0,
              odd_ld=False, images=False):
  """Am: logical A(i, r) [a_rows][red]; Bm: logical B(j, r) [b_rows][red].  Returns the output planes
  [splits][MI][NJ] as float64, and with images=True also the work images (a_hi, a_lo, b_hi, b_lo) as [rows_pad][red_pad]
  float32.  Asserts that every output element was written
  and that the guard band around the output is untouched."""
  from dqn_zoo_b200 import _lib
  a_rows, red = Am.shape
  b_rows = Bm.shape[0]
  MI, NJ = a_rows + (1 if ones else 0), b_rows
  dA = torch.as_tensor(stored(Am, a_rc, odd_ld), device='cuda')
  dB = torch.as_tensor(stored(Bm, b_rc, odd_ld), device='cuda')
  plane = MI * NJ
  n_out = splits * plane
  C = torch.full((2 * GUARD + offset + n_out,), float(SENTINEL), dtype=torch.float32, device='cuda')
  C[GUARD + offset:GUARD + offset + n_out] = float('nan')
  nwork = _lib.lib.dz_test_tc_pgemm_work(a_rows, b_rows, red)
  work = torch.full((nwork,), float('nan'), dtype=torch.float32, device='cuda')
  sc_i, sc_j = (1, MI) if transposed else (NJ, 1)
  db = None if bias is None else torch.as_tensor(bias, device='cuda')
  _lib.call('dz_test_tc_pgemm', dA.data_ptr(), a_rows, dA.shape[1], a_rc, dB.data_ptr(), b_rows, dB.shape[1], b_rc, red,
            a_rows if ones else -1, work.data_ptr(), C.data_ptr() + 4 * (GUARD + offset), sc_i, sc_j, splits, plane,
            0 if db is None else db.data_ptr(), int(relu), torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  c = C.cpu().numpy()
  guard = np.concatenate([c[:GUARD + offset], c[GUARD + offset + n_out:]])
  assert np.all(guard == SENTINEL), 'the GEMM wrote outside its output'
  out = c[GUARD + offset:GUARD + offset + n_out]
  assert not np.isnan(out).any(), '%d output elements were never written' % int(np.isnan(out).sum())
  planes = out.reshape(splits, NJ, MI).transpose(0, 2, 1) if transposed else out.reshape(splits, MI, NJ)
  if not images:
    return planes.astype(np.float64)
  ar = -(-(a_rows + 1) // 128) * 128
  br = -(-b_rows // 256) * 256
  rp = -(-red // KB) * KB
  w = work.cpu().numpy()
  parts = np.split(w, [ar * rp, 2 * ar * rp, 2 * ar * rp + br * rp])
  imgs = (image(parts[0], ar, rp), image(parts[1], ar, rp), image(parts[2], br, rp), image(parts[3], br, rp))
  return planes.astype(np.float64), imgs


def reference(Am, Bm, ones=False, bias=None, relu=False):
  A = Am.astype(np.float64)
  if ones:
    A = np.concatenate([A, np.ones((1, A.shape[1]))])
  D = A @ Bm.astype(np.float64).T
  if bias is not None:
    D = D + bias.astype(np.float64)[None, :]
  return np.maximum(D, 0.0) if relu else D


def rel(got, want):
  return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


def operands(a_rows, b_rows, red, seed):
  rs = np.random.RandomState(seed)
  return rs.standard_normal((a_rows, red)).astype(np.float32), rs.standard_normal((b_rows, red)).astype(np.float32)


ORIENTATIONS = [(1, 1), (1, 0), (0, 1), (0, 0)]


@pytest.mark.parametrize('a_rc,b_rc', ORIENTATIONS)
@pytest.mark.parametrize('a_rows,b_rows,red,odd_ld', [
    (130, 257, 100, 0),     # ragged i and j tiles: the last j tile has one column
    (257, 130, 17, 1),      # one reduction element past a k-block, ld % 4 != 0 (the pack kernel's scalar loads)
    (1, 257, 16, 0),        # one row, exactly one k-block
    (257, 1, 16, 1),        # one column
    (128, 256, 64, 0),      # exact tiles, ld % 4 == 0 (the pack kernel's 16-byte loads)
])
def test_orientations_and_ragged_extents(a_rows, b_rows, red, odd_ld, a_rc, b_rc):
  Am, Bm = operands(a_rows, b_rows, red, a_rows + 3 * b_rows + red)
  (got,) = run_pgemm(Am, Bm, a_rc, b_rc, odd_ld=odd_ld)
  want = reference(Am, Bm)
  assert rel(got, want) < 3e-6, rel(got, want)


@pytest.mark.parametrize('a_rc,b_rc', ORIENTATIONS)
def test_pack_images(a_rc, b_rc):
  """The hi/lo tile images the GEMM reads: hi is the TF32 round-to-nearest(-away) of the source, hi + lo reproduces it to
  2^-22, every padding row and reduction column is zero, the ones row is exactly 1 over the valid reduction."""
  a_rows, b_rows, red = 130, 257, 100
  Am, Bm = operands(a_rows, b_rows, red, 21)
  _, (a_hi, a_lo, b_hi, b_lo) = run_pgemm(Am, Bm, a_rc, b_rc, ones=True, odd_ld=True, images=True)
  A1 = np.concatenate([Am, np.ones((1, red), np.float32)])
  for hi, lo, src in ((a_hi, a_lo, A1), (b_hi, b_lo, Bm)):
    rows = src.shape[0]
    assert not np.isnan(hi).any() and not np.isnan(lo).any(), 'image elements left unwritten'
    for part in (hi, lo):
      assert np.all((part.view(np.uint32) & 0x1FFF) == 0), 'not a TF32 number'
    want_hi = ((src.view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)
    np.testing.assert_array_equal(hi[:rows, :red], want_hi)
    err = np.abs(hi[:rows, :red].astype(np.float64) + lo[:rows, :red] - src)
    assert np.all(err <= 2.0 ** -22 * np.abs(src.astype(np.float64))), float(err.max())
    for part in (hi, lo):
      assert np.all(part[rows:, :] == 0) and np.all(part[:, red:] == 0), 'padding is not zero'
  assert np.all(a_hi[a_rows, :red] == 1.0) and np.all(a_lo[a_rows, :red] == 0.0)


@pytest.mark.parametrize('a_rc', [1, 0])
def test_ones_row_gives_the_column_sums(a_rc):
  """a_ones_row = a_rows: the extra output row is sum_r B(j, r) (the bias gradient of a weight-gradient GEMM)."""
  Am, Bm = operands(200, 130, 300, 31)
  (got,) = run_pgemm(Am, Bm, a_rc, 0, ones=True)
  want = reference(Am, Bm, ones=True)
  assert rel(got[-1], want[-1]) < 3e-6, rel(got[-1], want[-1])
  assert rel(got, want) < 3e-6, rel(got, want)


@pytest.mark.parametrize('splits', [2, 3, 7, 9])
def test_split_partials_sum_to_the_reference(splits):
  """red 100 = 7 k-blocks: 2 and 3 splits share them unevenly, 7 gives one each, 9 leaves two splits without a k-block,
  whose planes must be written as zeros.  A bias passed with splits > 1 is not applied: the output is raw partials."""
  Am, Bm = operands(130, 257, 100, 41)
  bias = np.random.RandomState(42).standard_normal(257).astype(np.float32)
  planes = run_pgemm(Am, Bm, 1, 0, splits=splits, bias=bias, relu=True)
  want = reference(Am, Bm)
  assert rel(planes.sum(0), want) < 3e-6, rel(planes.sum(0), want)
  nkb = -(-100 // KB)
  per = -(-nkb // splits)
  for s in range(splits):
    lo_kb, hi_kb = min(s * per, nkb), min((s + 1) * per, nkb)
    part = reference(Am[:, lo_kb * KB:hi_kb * KB], Bm[:, lo_kb * KB:hi_kb * KB])
    if hi_kb == lo_kb:
      assert np.all(planes[s] == 0), 'an empty split did not write zeros'
    else:
      assert rel(planes[s], part) < 3e-6, (s, rel(planes[s], part))


@pytest.mark.parametrize('relu', [0, 1])
def test_bias_relu_epilogue(relu):
  Am, Bm = operands(257, 130, 64, 51)
  bias = np.random.RandomState(52).standard_normal(130).astype(np.float32)
  (got,) = run_pgemm(Am, Bm, 0, 1, bias=bias, relu=relu)
  want = reference(Am, Bm, bias=bias, relu=relu)
  assert rel(got, want) < 3e-6, rel(got, want)
  if relu:
    assert np.all(got[want < -1e-3] == 0)


@pytest.mark.parametrize('transposed,offset', [(0, 1), (1, 0), (1, 1)])
def test_output_placement(transposed, offset):
  """Transposed stores (sc_i = 1, sc_j = MI, as the embedding weight gradient) and a destination one float off 16-byte
  alignment (the scalar store path), with splits and the ones row; run_pgemm checks coverage and the guard band."""
  Am, Bm = operands(130, 257, 100, 61)
  planes = run_pgemm(Am, Bm, 0, 0, ones=True, splits=3, transposed=transposed, offset=offset)
  want = reference(Am, Bm, ones=True)
  assert rel(planes.sum(0), want) < 3e-6, rel(planes.sum(0), want)


def test_sign_consistent_accuracy():
  """All-positive operands over R = 3136: no cancellation hides a per-product or accumulation bias, so a 1xTF32 product
  (~5e-4) or an accumulator that truncates each of its 392 k-step adds (up to half an ulp each, all in one direction)
  misses the 3e-6 bar that 3xTF32 with round-to-nearest adds meets."""
  rs = np.random.RandomState(71)
  Am = rs.uniform(0.0, 1.0, (256, 3136)).astype(np.float32)
  Bm = rs.uniform(0.0, 1.0, (256, 3136)).astype(np.float32)
  (got,) = run_pgemm(Am, Bm, 1, 0)
  want = reference(Am, Bm)
  assert rel(got, want) < 3e-6, rel(got, want)
  assert np.abs(got / want - 1.0).max() < 1e-5


# ---- the learner's own problems (dz_learner.cu: IQN at batch 32, 64 samples per apply, 84x84 observations) --------


def test_fc1_forward_shape():
  """fc1 forward: act [2048][3136] x W [3136][512] (B read from W's columns), split partials, then bias + ReLU."""
  rs = np.random.RandomState(81)
  act = np.maximum(rs.standard_normal((2048, 3136)), 0).astype(np.float32)
  W = (rs.standard_normal((3136, 512)) / 56).astype(np.float32)
  bias = rs.standard_normal(512).astype(np.float32)
  planes = run_pgemm(act, W.T, 1, 0, splits=4)
  want = reference(act, W.T)
  assert rel(planes.sum(0), want) < 3e-6
  (got,) = run_pgemm(act, W.T, 1, 0, bias=bias, relu=True)
  want = reference(act, W.T, bias=bias, relu=True)
  assert rel(got, want) < 3e-6, rel(got, want)


def test_fc1_weight_gradient_shape():
  """fc1 weight gradient: [3136 + ones row][512] = act^T [.. | 1] x dh1 over the 2048 rows (A and B read column-wise)."""
  rs = np.random.RandomState(82)
  act = np.maximum(rs.standard_normal((2048, 3136)), 0).astype(np.float32)
  dh1 = (rs.standard_normal((2048, 512)) * 1e-3).astype(np.float32)
  planes = run_pgemm(act.T, dh1.T, 0, 0, ones=True, splits=8)
  want = reference(act.T, dh1.T, ones=True)
  got = planes.sum(0)
  assert rel(got, want) < 3e-6, rel(got, want)
  assert rel(got[-1], want[-1]) < 3e-6, 'bias-gradient row'


def test_fc1_input_gradient_shape():
  """fc1 input gradient: dh1 [2048][512] x W^T -> [2048][3136] (B = W read row-wise)."""
  rs = np.random.RandomState(83)
  dh1 = (rs.standard_normal((2048, 512)) * 1e-3).astype(np.float32)
  W = (rs.standard_normal((3136, 512)) / 56).astype(np.float32)
  (got,) = run_pgemm(dh1, W, 1, 1)
  want = reference(dh1, W)
  assert rel(got, want) < 3e-6, rel(got, want)


def test_embedding_weight_gradient_shape():
  """Embedding weight gradient: [3136][latent 64 + bias column] = dE^T x [cos | 1] over 2048 rows, stored transposed
  into [65][3136] partials (sc_i = 1, sc_j = 3136)."""
  rs = np.random.RandomState(84)
  dE = (rs.standard_normal((2048, 3136)) * 1e-3).astype(np.float32)
  cos1 = np.concatenate([np.cos(rs.uniform(0, 200, (2048, 64))), np.ones((2048, 1))], axis=1).astype(np.float32)
  planes = run_pgemm(dE.T, cos1.T, 0, 0, splits=5, transposed=True)
  want = reference(dE.T, cos1.T)
  assert rel(planes.sum(0), want) < 3e-6, rel(planes.sum(0), want)
