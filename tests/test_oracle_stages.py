"""CPU: oracle/stage_oracle.py, the stage-local float64 references of the learner's backward, against torch.autograd in
float64 on small random convs and linear layers, at the torso's strides 4, 2 and 1, on non-square inputs and on inputs
whose last rows and columns no conv window covers."""

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import stage_oracle as so


def conv_nhwc(x, w, s):
  return F.conv2d(x.permute(0, 3, 1, 2), w.permute(3, 2, 0, 1), stride=s).permute(0, 2, 3, 1)


def autograd_conv(x, w, b, s, mask_out):
  """Gradients of sum(relu-masked conv(x) * g) by autograd; g and the output mask are random."""
  x = x.clone().requires_grad_(True)
  w = w.clone().requires_grad_(True)
  b = b.clone().requires_grad_(True)
  y = conv_nhwc(x, w, s) + b
  g = torch.randn(y.shape, dtype=torch.float64, generator=torch.Generator().manual_seed(7)) * mask_out
  (y * g).sum().backward()
  return g, x.grad, w.grad, b.grad


# (batch, H, W, C, O, kernel, stride): the torso's three geometries, shrunk, square and not, with uncovered edges
CONVS = [(2, 20, 24, 4, 5, 8, 4), (3, 23, 21, 3, 4, 8, 4), (2, 9, 11, 6, 7, 4, 2), (1, 10, 7, 5, 3, 4, 2),
         (2, 5, 7, 6, 4, 3, 1), (3, 4, 3, 2, 5, 3, 1)]


@pytest.mark.parametrize('B,H,W,C,O,k,s', CONVS)
def test_conv_gradients_match_autograd(B, H, W, C, O, k, s):
  g = torch.Generator().manual_seed(B * 1000 + H * 10 + s)
  x = torch.randn((B, H, W, C), dtype=torch.float64, generator=g)
  w = torch.randn((k, k, C, O), dtype=torch.float64, generator=g)
  b = torch.randn((O,), dtype=torch.float64, generator=g)
  oh, ow = (H - k) // s + 1, (W - k) // s + 1
  mask_out = (torch.rand((B, oh, ow, O), generator=g) < 0.7).to(torch.float64)
  dy, dx_ref, dw_ref, db_ref = autograd_conv(x, w, b, s, mask_out)
  dW, db, S_dW, S_db = so.conv_wgrad(x, dy, k, s)
  torch.testing.assert_close(dW, dw_ref, rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(db, db_ref, rtol=1e-12, atol=1e-12)
  mask_in = torch.rand((B, H, W, C), generator=g) < 0.6
  dx, S = so.conv_dgrad(dy, w, s, (H, W), mask_in)
  torch.testing.assert_close(dx, dx_ref * mask_in, rtol=1e-12, atol=1e-12)
  dx_full, S_full = so.conv_dgrad(dy, w, s, (H, W))
  torch.testing.assert_close(dx_full, dx_ref, rtol=1e-12, atol=1e-12)
  # the magnitude scale is the same contraction on |inputs|: it bounds the result and equals it on non-negative inputs
  assert (S_dW >= dW.abs() - 1e-12).all() and (S_db >= db.abs() - 1e-12).all() and (S_full >= dx_full.abs() - 1e-12).all()
  _, _, S_dW_abs, _ = so.conv_wgrad(x.abs(), dy.abs(), k, s)
  torch.testing.assert_close(so.conv_wgrad(x.abs(), dy.abs(), k, s)[0], S_dW_abs, rtol=1e-14, atol=0)
  torch.testing.assert_close(so.conv_dgrad(dy.abs(), w.abs(), s, (H, W))[0], S_full, rtol=1e-14, atol=0)
  # pixels past the last window (rows / columns the VALID conv never reads) get exactly zero
  covered_h, covered_w = (oh - 1) * s + k, (ow - 1) * s + k
  assert (dx_full[:, covered_h:] == 0).all() and (dx_full[:, :, covered_w:] == 0).all()


def test_unit_frames_are_bytes_over_255():
  u8 = np.arange(256, dtype=np.uint8).reshape(1, 4, 8, 8)
  np.testing.assert_array_equal(so.unit_frames(u8).numpy(), np.arange(256).reshape(1, 4, 8, 8) / 255.0)


def test_linear_gradients_match_autograd():
  """Two streams sharing one input, one of them a factorised-noise layer, as fc1 of a noisy dueling network."""
  g = torch.Generator().manual_seed(3)
  M, K, N = 5, 12, 7
  x = torch.randn((M, K), dtype=torch.float64, generator=g).requires_grad_(True)
  w0 = torch.randn((K, N), dtype=torch.float64, generator=g)
  mu, sigma = torch.randn((K, N), dtype=torch.float64, generator=g), torch.rand((K, N), dtype=torch.float64, generator=g)
  ei, eo = torch.randn(K, dtype=torch.float64, generator=g), torch.randn(N, dtype=torch.float64, generator=g)
  mu = mu.requires_grad_(True)
  sigma = sigma.requires_grad_(True)
  b0 = torch.zeros(N, dtype=torch.float64, requires_grad=True)
  g0, g1 = torch.randn((M, N), dtype=torch.float64, generator=g), torch.randn((M, N), dtype=torch.float64, generator=g)
  y0 = x @ w0 + b0
  y1 = x @ mu + ((x * ei) @ sigma) * eo
  ((y0 * g0).sum() + (y1 * g1).sum()).backward()
  W1, W1_abs = so.noisy_weight(mu.detach(), sigma.detach(), ei, eo)
  mask = torch.rand((M, K), generator=g) < 0.5
  dx, S = so.linear_dgrad([(g0, w0, None), (g1, W1, W1_abs)], mask)
  torch.testing.assert_close(dx, x.grad * mask, rtol=1e-12, atol=1e-12)
  assert (S >= dx.abs() - 1e-12).all()
  torch.testing.assert_close(S, (g0.abs() @ w0.abs().T + g1.abs() @ W1_abs.T) * mask, rtol=1e-14, atol=0)
  dW, db, S_dW, S_db = so.linear_wgrad(x.detach(), g0)
  torch.testing.assert_close(dW, x.detach().T @ g0, rtol=1e-14, atol=0)
  torch.testing.assert_close(db, b0.grad, rtol=1e-14, atol=1e-14)
  dmu, _, _, _ = so.linear_wgrad(x.detach(), g1)
  dsig, _, _, _ = so.linear_wgrad(x.detach() * ei, g1 * eo)
  torch.testing.assert_close(dmu, mu.grad, rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(dsig, sigma.grad, rtol=1e-12, atol=1e-12)
  assert (S_dW >= dW.abs()).all() and (S_db >= db.abs()).all()


def test_hadamard_gradient_matches_autograd():
  g = torch.Generator().manual_seed(5)
  B, N, D = 3, 4, 10
  feat = torch.rand((B, D), dtype=torch.float64, generator=g).requires_grad_(True)
  e = torch.rand((B, N, D), dtype=torch.float64, generator=g)
  dhi = torch.randn((B, N, D), dtype=torch.float64, generator=g)
  ((feat[:, None, :] * e) * dhi).sum().backward()
  mask = torch.rand((B, D), generator=g) < 0.5
  dx, S = so.hadamard_dgrad(dhi, e, mask)
  torch.testing.assert_close(dx, feat.grad * mask, rtol=1e-12, atol=1e-12)
  torch.testing.assert_close(S, (dhi.abs() * e).sum(1) * mask, rtol=1e-14, atol=0)
