"""GPU: the fc1 / noisy1 input-gradient kernel (csrc/dz_umma.cuh, umma_fc_kernel on the K-major weight tile).

The 3136 -> 512 input gradient D[k, m] = sum_n W[k][n] g[m][n] stages mu (and sigma) K-major in n, and the MMA warps
form w = mu + sigma * eps_in[k] * eps_out[n] and its tf32 hi/lo split in registers.  Each output element sees the same
operands and the same k-steps as on umma_gemm_kernel with its converter warps, so the split partials are expected to
agree bit for bit; both are also checked against float64."""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MAX_SPLITS = 8


def conv_out(n, k, s):
  return (n - k) // s + 1


def feat_of(H, W):
  h = conv_out(conv_out(conv_out(H, 8, 4), 4, 2), 3, 1)
  w = conv_out(conv_out(conv_out(W, 8, 4), 4, 2), 3, 1)
  return h * w * 64


def noise_vec(rs, n):
  x = np.clip(rs.standard_normal(n), -2, 2)
  return (np.sign(x) * np.sqrt(np.abs(x))).astype(np.float32)


def make_inputs(B, H, W, nstream, noisy, seed):
  """The blob holds, per stream, mu [feat][512] then sigma [feat][512]; the noise holds, per stream, eps_in then eps_out."""
  feat = feat_of(H, W)
  rs = np.random.RandomState(seed)
  nw = feat * 512
  blob = (0.05 * rs.standard_normal(nstream * 2 * nw)).astype(np.float32)
  noise = noise_vec(rs, nstream * (feat + 512))
  g = (0.1 * rs.standard_normal((nstream, B, 512))).astype(np.float32)
  return dict(B=B, H=H, W=W, nstream=nstream, noisy=noisy, feat=feat, blob=blob, noise=noise, g=g,
              off_w=[s * 2 * nw for s in range(nstream)], off_sw=[s * 2 * nw + nw for s in range(nstream)],
              off_in=[s * (feat + 512) for s in range(nstream)], off_out=[s * (feat + 512) + feat for s in range(nstream)])


def run(inp, converters):
  """Split partials [nstream][S][B][feat] and S."""
  from dqn_zoo_b200 import _lib
  dev = 'cuda'
  B, nstream, feat = inp['B'], inp['nstream'], inp['feat']
  blob = torch.as_tensor(inp['blob'], device=dev)
  noise = torch.as_tensor(inp['noise'], device=dev)
  g = torch.as_tensor(inp['g'], device=dev)
  part = torch.full((nstream * MAX_SPLITS * B * feat,), float('nan'), dtype=torch.float32, device=dev)
  def i64x2(v):
    return (ctypes.c_int64 * 2)(*(list(v) + [0])[:2])
  off_w, off_sw, off_in, off_out = i64x2(inp['off_w']), i64x2(inp['off_sw']), i64x2(inp['off_in']), i64x2(inp['off_out'])
  splits = ctypes.c_int32(0)
  _lib.call('dz_test_fc_dgrad', B, inp['H'], inp['W'], nstream, int(inp['noisy']), blob.data_ptr(), ctypes.addressof(off_w),
            ctypes.addressof(off_sw), noise.data_ptr(), ctypes.addressof(off_in), ctypes.addressof(off_out), g.data_ptr(),
            int(converters), part.data_ptr(), ctypes.byref(splits), torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  S = splits.value
  return part[:nstream * S * B * feat].cpu().numpy().reshape(nstream, S, B, feat), S


def reference(inp):
  """float64 [nstream][B][feat] = g_s @ (mu + sigma * eps_in eps_out^T)^T."""
  nstream, feat = inp['nstream'], inp['feat']
  nw = feat * 512
  blob = inp['blob'].astype(np.float64)
  nz = inp['noise'].astype(np.float64)
  out = []
  for s in range(nstream):
    w = blob[inp['off_w'][s]:inp['off_w'][s] + nw].reshape(feat, 512)
    if inp['noisy']:
      ein = nz[inp['off_in'][s]:inp['off_in'][s] + feat]
      eout = nz[inp['off_out'][s]:inp['off_out'][s] + 512]
      w = w + blob[inp['off_sw'][s]:inp['off_sw'][s] + nw].reshape(feat, 512) * np.outer(ein, eout)
    out.append(inp['g'][s].astype(np.float64) @ w.T)
  return np.stack(out)


def rel(got, want):
  return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


# noisy with two streams (rainbow) and plain with one (dqn), at 84x84 (feat 3136, a half-filled last 128-row tile) and
# 76x76 (feat 2304), at the learner's batch and at one that takes the 64-column tiles
PARAMS = [(B, H, W, noisy) for B in (32, 48) for H, W in ((84, 84), (76, 76)) for noisy in (False, True)]


@pytest.mark.parametrize('B,H,W,noisy', PARAMS)
def test_fc_dgrad_matches_converter_kernel_bit_for_bit(B, H, W, noisy):
  nstream = 2 if noisy else 1
  inp = make_inputs(B, H, W, nstream, noisy, seed=B + H + int(noisy))
  new, S = run(inp, converters=False)
  old, S_old = run(inp, converters=True)
  assert S == S_old
  want = reference(inp)
  for name, got in (('umma_fc_kernel', new), ('umma_gemm_kernel', old)):
    assert not np.isnan(got).any(), name
    e = rel(got.astype(np.float64).sum(axis=1), want)
    assert e < 3e-6, (name, e)
  np.testing.assert_array_equal(new, old)
