"""Stage-local float64 references of the learner's backward between the head and the optimizer (TEST INFRASTRUCTURE
ONLY).

Each function restates one launch of the step on inputs the caller read back from the device after an update: the
activations, the input gradients the launch consumed and the parameters.  A stage compared this way measures only that
launch's arithmetic, and no ReLU can flip, because every mask comes from the device's own activations.

Every function returns the float64 result with its magnitude scale S: the same contraction evaluated on absolute values,
sum |a| |b|.  Any fp32 evaluation of the contraction, in any order, is within a multiple of 2^-24 S of the exact value,
so S is what the tests scale their error bars by.

Layouts are the device's: activations and their gradients NHWC [B, H, W, C], conv weights HWIO [k, k, C, O], linear
weights (in, out).  Inputs are torch tensors or numpy arrays; results are float64 torch tensors.
"""

from __future__ import annotations

import torch
import torch.nn.functional as F


def _f64(x):
  return torch.as_tensor(x).to(torch.float64)


def unit_frames(u8):
  """conv1's input: uint8 frames [B, H, W, C] / 255 in float64."""
  return _f64(u8) / 255.0


def noisy_weight(mu, sigma, eps_in, eps_out):
  """A factorised-noise layer's formed weight mu + sigma . (eps_in eps_out^T) and its magnitude |mu| + |sigma . eps_in
  eps_out^T|, the matrix whose products with |x| give S."""
  mu, sigma = _f64(mu), _f64(sigma)
  outer = torch.outer(_f64(eps_in), _f64(eps_out))
  return mu + sigma * outer, mu.abs() + (sigma * outer).abs()


def _cols(x, k, s):
  """im2col of NHWC x: [B, L, k * k * C], columns in HWIO's (kh, kw, c) order, L output positions row-major."""
  B, H, W, C = x.shape
  u = F.unfold(x.permute(0, 3, 1, 2), k, stride=s)   # [B, C * k * k, L], (c, kh, kw) order
  return u.view(B, C, k * k, -1).permute(0, 3, 2, 1).reshape(B, -1, k * k * C)


def _uncols(dcol, k, s, C, H, W):
  """col2im: the adjoint of _cols, back to NHWC [B, H, W, C]; input pixels no window covers get 0."""
  B, L, _ = dcol.shape
  u = dcol.view(B, L, k * k, C).permute(0, 3, 2, 1).reshape(B, C * k * k, L)
  return F.fold(u, (H, W), k, stride=s).permute(0, 2, 3, 1)


def conv_wgrad(x, dy, k, s):
  """Weight and bias gradient of a VALID conv, stride s, from its input x [B, H, W, C] and the gradient dy
  [B, oh, ow, O] of its (masked) output.  Returns (dW [k, k, C, O], db [O], S_dW, S_db)."""
  x, dy = _f64(x), _f64(dy)
  C, O = x.shape[3], dy.shape[3]
  cols = _cols(x, k, s).reshape(-1, k * k * C)
  g = dy.reshape(-1, O)
  assert cols.shape[0] == g.shape[0], (cols.shape, g.shape)
  dW = (cols.T @ g).view(k, k, C, O)
  S_dW = (cols.abs().T @ g.abs()).view(k, k, C, O)
  return dW, g.sum(0), S_dW, g.abs().sum(0)


def conv_dgrad(dy, w, s, in_hw, mask=None):
  """Input gradient of a VALID conv with HWIO weights w, stride s, over an input of in_hw = (H, W), from dy [B, oh, ow,
  O]: the conv transpose (dcol = dy W^T, then col2im), times mask (the device's [x > 0] of the input) when given.
  Returns (dx [B, H, W, C], S)."""
  dy, w = _f64(dy), _f64(w)
  k, C, O = w.shape[0], w.shape[2], w.shape[3]
  B = dy.shape[0]
  wf = w.reshape(k * k * C, O)
  g = dy.reshape(B, -1, O)
  dx = _uncols(g @ wf.T, k, s, C, *in_hw)
  S = _uncols(g.abs() @ wf.abs().T, k, s, C, *in_hw)
  if mask is not None:
    m = torch.as_tensor(mask).to(torch.float64)
    dx, S = dx * m, S * m
  return dx, S


def linear_dgrad(terms, mask=None):
  """Input gradient of linear layers that share one input: sum over terms (g [M, N], w [K, N], w_abs [K, N] or None)
  of g w^T, times mask [M, K] when given.  w_abs is the magnitude of a formed weight (noisy_weight); None takes |w|.
  Returns (dx [M, K], S)."""
  dx = S = 0
  for g, w, w_abs in terms:
    g, w = _f64(g), _f64(w)
    w_abs = w.abs() if w_abs is None else _f64(w_abs)
    dx = dx + g @ w.T
    S = S + g.abs() @ w_abs.T
  if mask is not None:
    m = torch.as_tensor(mask).to(torch.float64)
    dx, S = dx * m, S * m
  return dx, S


def linear_wgrad(x, g):
  """Weight and bias gradient of y = x W + b from its input x [M, K] and output gradient g [M, N].  Returns (dW [K, N],
  db [N], S_dW, S_db)."""
  x, g = _f64(x), _f64(g)
  return x.T @ g, g.sum(0), x.abs().T @ g.abs(), g.abs().sum(0)


def hadamard_dgrad(dhi, e, mask=None):
  """IQN's torso feature gradient through hi[b, n] = feat[b] . E[b, n]: sum over the N samples of dhi . E, [B, N, D]
  each, times mask [B, D] when given.  Returns (dfeat [B, D], S)."""
  dhi, e = _f64(dhi), _f64(e)
  dx, S = (dhi * e).sum(1), (dhi * e).abs().sum(1)
  if mask is not None:
    m = torch.as_tensor(mask).to(torch.float64)
    dx, S = dx * m, S * m
  return dx, S
