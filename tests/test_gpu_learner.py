"""GPU: the CUDA learner vs the float64 PyTorch-CPU oracle (oracle/learner_oracle.py).

Tolerance (BASELINE.json north_star): <= 1e-5 relative on fp32 losses and gradients.  Gradients
are compared per tensor as ||g - g_ref|| / ||g_ref|| (and the global norm), losses per example.
Parity is against the restatement of rlax/optax 0.1.2 (PARITY UNPINNED, see the oracle header).
The checks themselves are in tests/learner_parity.py; test_gpu_learner_shapes.py runs them at the shapes that switch
kernel paths.
"""

import numpy as np
import pytest
import torch

from learner_parity import (check_loss_and_gradients, check_q_values, check_three_optimizer_steps, make_batch,
                            make_case)
from oracle import learner_oracle as lo

pytestmark = pytest.mark.gpu

KINDS = list(lo.AGENT_KINDS)


@pytest.mark.parametrize('hw,B', [(84, 32), (44, 5)])
@pytest.mark.parametrize('kind', KINDS)
def test_loss_and_gradients_match_oracle(kind, hw, B):
  check_loss_and_gradients(kind, hw, B)


@pytest.mark.parametrize('kind', ['c51', 'rainbow'])
def test_largest_categorical_head_matches_oracle(kind):
  """64 actions x 128 atoms, the largest categorical head the learner accepts: the loss kernel then stages 103,696
  bytes of head outputs in shared memory, beyond the default 48 KB.  Same loss/gradient parity."""
  check_loss_and_gradients(kind, 84, 32, num_actions=64, num_atoms=128)


@pytest.mark.parametrize('kind', KINDS)
def test_three_optimizer_steps_match_oracle(kind):
  check_three_optimizer_steps(kind, 84, 32)


def test_q_values_match_oracle_forward():
  for kind in KINDS:
    check_q_values(*make_case(kind, 32, 84, seed=7))


def test_update_is_run_to_run_deterministic():
  spec, net, L, O, rs = make_case('rainbow', 32, 84, seed=9)
  arrs, batch, w, taus_o, taus_flat, noise_o, noise_flat = make_batch(spec, net, 32, rs)
  L.update(*arrs, weights=w, noise=noise_flat, apply_update=False)
  g1 = L.grads.clone()
  L.update(*arrs, weights=w, noise=noise_flat, apply_update=False)
  torch.cuda.synchronize()
  assert torch.equal(g1, L.grads)


@pytest.mark.parametrize('hw,B', [(84, 65), (40, 32)])
@pytest.mark.parametrize('kind', ['dqn', 'rainbow'])
def test_fp32_fma_fallback_matches_oracle(kind, hw, B):
  """Geometries the tensor-core torso does not cover run every contraction on the fp32-FMA kernels: batch > 64, and an
  odd conv1 output (9x9 at 40x40; at batch <= 32 this also takes the split-K FMA layers).  Same loss/gradient parity."""
  check_loss_and_gradients(kind, hw, B, fma_torso=True)


def test_uint8_to_unit_conversion_is_correctly_rounded():
  """networks.py:193 `x.astype(float32) / 255.0`: the device uses multiply + one Newton step instead of an
  IEEE division; it must give the correctly rounded quotient for every possible byte."""
  from dqn_zoo_b200 import _lib
  out = torch.zeros(256, dtype=torch.float32, device='cuda')
  _lib.call('dz_test_u8_to_unit', out.data_ptr(), torch.cuda.current_stream().cuda_stream)
  want = np.arange(256, dtype=np.float32) / np.float32(255.0)
  np.testing.assert_array_equal(out.cpu().numpy(), want)
