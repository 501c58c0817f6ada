"""GPU: the fc1 / noisy1 forward kernel (csrc/dz_umma.cuh, umma_fc_kernel).

The 3136 -> 512 forward is planned per weight blob: the passes that apply the same parameters (the online net on s_tm1
and on s_t) share every staged weight tile, and the MMA warps form w = mu + sigma * eps_in * eps_out and its tf32
hi/lo split in registers.  Each output element sees the same operands and the same k-steps as on umma_gemm_kernel
with its converter warps and one CTA group per pass, so the split partials are expected to agree bit for bit; both are
also checked against float64."""

import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

MMA_SYNC = 1
MAX_SPLITS = 24


def conv_out(n, k, s):
  return (n - k) // s + 1


def feat_of(H, W):
  h = conv_out(conv_out(conv_out(H, 8, 4), 4, 2), 3, 1)
  w = conv_out(conv_out(conv_out(W, 8, 4), 4, 2), 3, 1)
  return h * w * 64


def noise_vec(rs, n):
  x = np.clip(rs.standard_normal(n), -2, 2)
  return (np.sign(x) * np.sqrt(np.abs(x))).astype(np.float32)


def make_inputs(B, H, W, npass, nstream, noisy, seed):
  """Blobs hold, per stream, mu [feat][512] then sigma [feat][512]; noise apply p holds, per stream, eps_in then eps_out."""
  feat = feat_of(H, W)
  rs = np.random.RandomState(seed)
  nw = feat * 512
  blobs = [(0.05 * rs.standard_normal(nstream * 2 * nw)).astype(np.float32) for _ in range(2)]
  stride = nstream * (feat + 512)
  noise = np.concatenate([noise_vec(rs, stride) for _ in range(3)])
  x = np.maximum(rs.standard_normal((npass * B, feat)), 0.0).astype(np.float32)
  return dict(B=B, H=H, W=W, npass=npass, nstream=nstream, noisy=noisy, feat=feat, blobs=blobs, noise=noise, x=x,
              off_w=[s * 2 * nw for s in range(nstream)], off_sw=[s * 2 * nw + nw for s in range(nstream)],
              off_in=[s * (feat + 512) for s in range(nstream)], off_out=[s * (feat + 512) + feat for s in range(nstream)],
              stride=stride)


def run(inp, per_pass):
  """Split partials [npass][nstream][S][B][512], S and the weight-tile bytes the launch staged."""
  from dqn_zoo_b200 import _lib
  dev = 'cuda'
  B, npass, nstream = inp['B'], inp['npass'], inp['nstream']
  online = torch.as_tensor(inp['blobs'][0], device=dev)
  target = torch.as_tensor(inp['blobs'][1], device=dev)
  noise = torch.as_tensor(inp['noise'], device=dev)
  x = torch.as_tensor(inp['x'], device=dev)
  part = torch.full((npass * nstream * MAX_SPLITS * B * 512,), float('nan'), dtype=torch.float32, device=dev)
  def i64x2(v):
    return (ctypes.c_int64 * 2)(*(list(v) + [0])[:2])
  off_w, off_sw, off_in, off_out = i64x2(inp['off_w']), i64x2(inp['off_sw']), i64x2(inp['off_in']), i64x2(inp['off_out'])
  splits, wbytes = ctypes.c_int32(0), ctypes.c_int64(0)
  _lib.call('dz_test_fc_forward', B, inp['H'], inp['W'], npass, nstream, int(inp['noisy']), online.data_ptr(), target.data_ptr(),
            ctypes.addressof(off_w), ctypes.addressof(off_sw), noise.data_ptr(), inp['stride'], ctypes.addressof(off_in),
            ctypes.addressof(off_out), x.data_ptr(), int(per_pass), part.data_ptr(), ctypes.byref(splits), ctypes.byref(wbytes),
            torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  S = splits.value
  return part[:npass * nstream * S * B * 512].cpu().numpy().reshape(npass, nstream, S, B, 512), S, wbytes.value


def reference(inp):
  """float64 [npass][nstream][B][512] = x_p @ (mu + sigma * eps_in eps_out^T) of the pass's blob."""
  B, npass, nstream, feat = inp['B'], inp['npass'], inp['nstream'], inp['feat']
  nw = feat * 512
  out = np.zeros((npass, nstream, B, 512))
  for p in range(npass):
    blob = inp['blobs'][0 if p == 0 or (npass == 3 and p == 1) else 1].astype(np.float64)
    xp = inp['x'][p * B:(p + 1) * B].astype(np.float64)
    for s in range(nstream):
      w = blob[inp['off_w'][s]:inp['off_w'][s] + nw].reshape(feat, 512)
      if inp['noisy']:
        nz = inp['noise'][p * inp['stride']:(p + 1) * inp['stride']].astype(np.float64)
        ein = nz[inp['off_in'][s]:inp['off_in'][s] + feat]
        eout = nz[inp['off_out'][s]:inp['off_out'][s] + 512]
        w = w + blob[inp['off_sw'][s]:inp['off_sw'][s] + nw].reshape(feat, 512) * np.outer(ein, eout)
      out[p, s] = xp @ w
  return out


def rel(got, want):
  return float(np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30))


# (B, H, W): the learner's batch at 84x84 (feat 3136) and at 76x76 (feat 2304) for 1, 2 and 3 passes, plain and noisy;
# and the rainbow layout at a batch that takes the 64-column tiles
CASES = [(32, 84, 84), (32, 76, 76)]
PARAMS = [(B, H, W, npass, noisy) for B, H, W in CASES for npass in (1, 2, 3) for noisy in (False, True)] + [(48, 84, 84, 3, True)]


@pytest.mark.parametrize('B,H,W,npass,noisy', PARAMS)
def test_fc_forward_matches_converter_kernel_bit_for_bit(B, H, W, npass, noisy):
  nstream = 2 if noisy else 1
  inp = make_inputs(B, H, W, npass, nstream, noisy, seed=B + H + 10 * npass + int(noisy))
  new, S, wb_new = run(inp, per_pass=False)
  old, S_old, wb_old = run(inp, per_pass=True)
  assert S == S_old
  want = reference(inp)
  for name, got in (('umma_fc_kernel', new), ('umma_gemm_kernel', old)):
    assert not np.isnan(got).any(), name
    e = rel(got.astype(np.float64).sum(axis=2), want)
    assert e < 3e-6, (name, e)
  np.testing.assert_array_equal(new, old)
  # each weight tile is staged once per blob: the passes that apply one blob share it
  per_blob = nstream * inp['feat'] * 512 * 4 * (2 if noisy else 1)
  blobs_used = 1 if npass == 1 else 2
  assert wb_new == blobs_used * per_blob, (wb_new, blobs_used * per_blob)
  assert wb_old == npass * per_blob, (wb_old, npass * per_blob)


@pytest.mark.parametrize('kind', ['rainbow', 'double_q', 'dqn'])
def test_learner_fc1_forward_stays_on_mma_sync(kind):
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  L = dl.Learner(dl.NetworkSpec(kind, 6), batch_size=32)
  path = ctypes.c_int32(0)
  _lib.call('dz_test_learner_mma_path', L._h, b'fc1_fwd', ctypes.byref(path))
  assert path.value == MMA_SYNC, (kind, path.value)
