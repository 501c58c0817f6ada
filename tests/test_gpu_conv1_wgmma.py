"""GPU: conv1 forward on warpgroup MMAs (csrc/dz_umma_net.cu, conv1_wgmma_kernel).

The learner's conv1 forward gathers the sampled uint8 observations in place, converts them to exact tf32 values and
multiplies them with the tf32 hi/lo weight image on two consumer warpgroups.  Each k-step forms the same two products
(A*Wlo from zero, then + A*Whi) in the same order as the warp-level mma.sync kernel it replaced (conv1_umma_kernel,
kept as the reference), and the sums start from the bias and take the k-steps in the same order, so act1 hi and lo
are expected to agree bit for bit; hi + lo is also checked against a float64 convolution."""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MMA_SYNC, WGMMA = 1, 2
N_W = (256 * 32, 512 * 64, 576 * 64)   # conv1..3 weights, [kh][kw][c][n]


def conv_out(n, k, s):
  return (n - k) // s + 1


def make_inputs(B, H, W, npass, seed):
  """Two blobs [w1 | b1 | w2 | w3]; an observation pool and per-pass row tables that gather from it out of order."""
  rs = np.random.RandomState(seed)
  off_w = [0, N_W[0] + 32, N_W[0] + 32 + N_W[1]]
  size = off_w[2] + N_W[2]
  blobs = [(0.1 * rs.standard_normal(size)).astype(np.float32) for _ in range(2)]
  pool = rs.randint(0, 256, size=(npass * B + 3, H, W, 4)).astype(np.uint8)
  order = rs.permutation(pool.shape[0])[:npass * B].reshape(npass, B)
  return dict(B=B, H=H, W=W, npass=npass, blobs=blobs, off_w=off_w, off_b1=N_W[0], pool=pool, order=order)


def run(inp, path):
  """act1 hi, lo as float32 numpy [npass * B][h1][w1][32]."""
  from dqn_zoo_b200 import _lib
  dev = 'cuda'
  B, H, W, npass = inp['B'], inp['H'], inp['W'], inp['npass']
  h1, w1 = conv_out(H, 8, 4), conv_out(W, 8, 4)
  online = torch.as_tensor(inp['blobs'][0], device=dev)
  target = torch.as_tensor(inp['blobs'][1], device=dev)
  pool = torch.as_tensor(inp['pool'], device=dev)
  img = H * W * 4
  tables = [torch.as_tensor([pool.data_ptr() + int(i) * img for i in inp['order'][p]], dtype=torch.int64, device=dev)
            for p in range(npass)]
  rows = (ctypes.c_void_p * 3)(*([t.data_ptr() for t in tables] + [None] * (3 - npass)))
  off_w = (ctypes.c_int64 * 3)(*inp['off_w'])
  n = npass * B * h1 * w1 * 32
  hi = torch.full((n,), float('nan'), dtype=torch.float32, device=dev)
  lo = torch.full((n,), float('nan'), dtype=torch.float32, device=dev)
  _lib.call('dz_test_conv1_forward', B, H, W, npass, online.data_ptr(), target.data_ptr(), ctypes.addressof(off_w),
            inp['off_b1'], ctypes.addressof(rows), path, hi.data_ptr(), lo.data_ptr(), torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  shape = (npass * B, h1, w1, 32)
  return hi.cpu().numpy().reshape(shape), lo.cpu().numpy().reshape(shape)


def reference_pre(inp):
  """float64 pre-activations [npass * B][h1][w1][32] = conv(bytes / 255, W1) + b1 with the pass's blob."""
  npass = inp['npass']
  out = []
  for p in range(npass):
    blob = inp['blobs'][0 if p == 0 or (npass == 3 and p == 1) else 1].astype(np.float64)
    w = torch.as_tensor(blob[:N_W[0]].reshape(8, 8, 4, 32)).permute(3, 2, 0, 1)          # [n][c][kh][kw]
    b = torch.as_tensor(blob[inp['off_b1']:inp['off_b1'] + 32])
    x = torch.as_tensor(inp['pool'][inp['order'][p]].astype(np.float64) / 255.0).permute(0, 3, 1, 2)
    out.append(torch.nn.functional.conv2d(x, w, b, stride=4).permute(0, 2, 3, 1).numpy())
  return np.concatenate(out)


def rel(got, want):
  return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


# (B, H, W, npass): the learner's batch at 84x84 for 1, 2 and 3 passes; batch 64; 44x44 at B = 5 (last tile 116 rows);
# 36x36 at B = 1 (64 pixels: the second m64 half of the only tile is empty); 76x76 (324 pixels: tiles span two images)
PARAMS = [(32, 84, 84, 1), (32, 84, 84, 2), (32, 84, 84, 3), (64, 84, 84, 2), (5, 44, 44, 2), (1, 36, 36, 1),
          (1, 36, 36, 3), (8, 76, 76, 3)]


@pytest.mark.parametrize('B,H,W,npass', PARAMS)
def test_conv1_wgmma_matches_mma_sync_and_float64(B, H, W, npass):
  inp = make_inputs(B, H, W, npass, seed=B + H + 10 * npass)
  hi, lo = run(inp, WGMMA)
  hi_ref, lo_ref = run(inp, MMA_SYNC)
  assert not np.isnan(hi).any() and not np.isnan(lo).any()
  np.testing.assert_array_equal(hi, hi_ref)
  np.testing.assert_array_equal(lo, lo_ref)
  assert np.all((hi.view(np.uint32) & 0x1FFF) == 0)
  assert np.all((lo.view(np.uint32) & 0x1FFF) == 0)
  pre = reference_pre(inp)
  got = hi.astype(np.float64) + lo.astype(np.float64)
  # ReLU kinks: a unit whose float64 pre-activation is within float32 rounding of zero may land on the other side on
  # the device.  Every such flip must be at the kink (|pre| <= 2e-5 rms) and there may be only a handful.
  flipped = (got > 0) != (pre > 0)
  rms = float(np.sqrt(np.mean(pre * pre)))
  nflip = int(flipped.sum())
  assert nflip <= 3 + 2e-5 * pre.size, ('too many kink flips', nflip, pre.size)
  if nflip:
    assert float(np.abs(pre[flipped]).max()) <= 2e-5 * rms, ('a flipped unit is NOT at the kink', nflip)
  e = rel(got, np.maximum(pre, 0.0))
  assert e < 3e-6, e


@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_learner_conv1_forward_runs_on_wgmma(kind):
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  L = dl.Learner(dl.NetworkSpec(kind, 6), batch_size=32)
  path = ctypes.c_int32(0)
  _lib.call('dz_test_learner_mma_path', L._h, b'conv1_fwd', ctypes.byref(path))
  assert path.value == WGMMA, (kind, path.value)
