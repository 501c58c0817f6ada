"""GPU: the whole learner against the float64 oracle at the shapes where its kernels change path.

test_gpu_learner.py pins the learner at 84x84 / batch 32 and 44x44 / batch 5 with 6 actions.  The plans switch at
other shapes: IQN's packed-operand tensor-core GEMM (csrc/dz_tcp.cuh) turns on only at >= 1024 rows per apply, every
row count a multiple of 4 and latent <= 128, its packed embedding backward only at 64 samples for s_tm1; the
tensor-core torso covers batches 1..64 and non-square observations with an even conv1 output; the heads take different
kernels by batch (split head + finish_nn up to 32, bias in the GEMM above) and width (16-byte finish when the width is a
multiple of 4, IQN's skinny head up to 18 actions).  Each case runs the parity bars of learner_parity.py and asserts
which path ran, so that a silent fall-back cannot keep it green.
"""

import pytest

from learner_parity import check_loss_and_gradients, check_q_values, check_three_optimizer_steps, mma_path, \
    tensor_core_torso

pytestmark = pytest.mark.gpu

PACKED_LAUNCHES = ('iqn_embed_fwd', 'iqn_fc1_fwd', 'iqn_fc1_wgrad', 'iqn_fc1_dgrad')


def check(kind, hw, B, tc_torso, packed=None, embed_bwd=None, **case):
  spec, net, L, O, rs = check_loss_and_gradients(kind, hw, B, **case)
  assert tensor_core_torso(L) == tc_torso, 'torso path'
  if kind == 'iqn':
    assert {t: mma_path(L, t) for t in PACKED_LAUNCHES} == {t: 1 if packed else None for t in PACKED_LAUNCHES}
    assert mma_path(L, 'iqn_embed_wgrad') == (1 if embed_bwd else None)
  check_q_values(spec, net, L, O, rs)


# ---- IQN: the packed-operand GEMM and its branch points ---------------------------------------------------------------

@pytest.mark.parametrize('B,hw,taus,latent,packed,embed_bwd,tc_torso', [
    (16, 84, (64, 64, 64), 64, True, True, True),       # exactly 1024 rows per apply
    (32, 84, (33, 40, 36), 64, True, False, True),      # three different ragged row counts, embedding backward on FMA
    (32, 84, (64, 64, 64), 16, True, True, True),       # one k-block of latent
    (32, 84, (64, 64, 64), 128, True, True, True),      # 8 k-blocks: the embedding epilogue's limit
    (32, 84, (64, 64, 64), 144, False, False, True),    # latent > 128: fp32-FMA
    (31, 84, (33, 33, 33), 64, False, False, True),     # 1023 rows: fp32-FMA
    (64, 84, (64, 64, 64), 64, True, True, True),       # packed head on the batch-64 tensor-core torso
    (128, 44, (8, 8, 8), 64, True, False, False),       # packed head on the fp32-FMA torso (batch > 64)
])
def test_iqn_packed_gemm_branches(B, hw, taus, latent, packed, embed_bwd, tc_torso):
  check('iqn', hw, B, tc_torso, packed, embed_bwd, taus=taus, latent_dim=latent)


@pytest.mark.parametrize('num_actions', [18, 19])
def test_iqn_skinny_head_limit(num_actions):
  """18 actions: the skinny head kernels (the full Atari action set); 19: the general GEMM head."""
  check('iqn', 84, 32, True, True, True, num_actions=num_actions)


# ---- the tensor-core torso -------------------------------------------------------------------------------------------

@pytest.mark.parametrize('B', [1, 33, 64])
@pytest.mark.parametrize('kind', ['dqn', 'rainbow'])
def test_torso_batches(kind, B):
  """Batch 1, and above 32 where the torso's plans widen (64-column tiles, conv1 tiles over more images)."""
  check(kind, 84, B, True)


@pytest.mark.parametrize('kind,hw,B,tc_torso', [
    ('dqn', (36, 36), 7, True),      # feat 64, the smallest feature map
    ('rainbow', (92, 92), 32, True),  # the largest square observation
    ('dqn', (84, 92), 32, True),     # a non-square pair and its swap: a height / width mix-up fails one of them
    ('dqn', (92, 84), 32, True),
    ('rainbow', (36, 84), 32, True),
    ('rainbow', (84, 36), 32, True),
    ('dqn', (36, 44), 20, True),     # 80-pixel conv1 maps: a 128-pixel conv1 tile spans three images
    ('dqn', (84, 88), 32, False),    # odd conv1 width (21): fp32-FMA
])
def test_torso_geometries(kind, hw, B, tc_torso):
  check(kind, hw, B, tc_torso)


# ---- head widths -----------------------------------------------------------------------------------------------------
# batch 32: split head GEMM + finish_nn (16-byte path when the width is a multiple of 4); batch 48: unsplit head with
# the bias in the GEMM.  44x44 observations keep the float64 oracle cheap; the torso is on the tensor cores.

@pytest.mark.parametrize('B', [32, 48])
@pytest.mark.parametrize('kind,case', [
    ('dqn', dict(num_actions=1)), ('dqn', dict(num_actions=4)), ('dqn', dict(num_actions=18)),
    ('double_q', dict(num_actions=1)), ('double_q', dict(num_actions=4)), ('double_q', dict(num_actions=18)),
    ('prioritized', dict(num_actions=1)), ('prioritized', dict(num_actions=4)), ('prioritized', dict(num_actions=18)),
    ('c51', dict(num_atoms=2)), ('c51', dict(num_atoms=33)),
    ('rainbow', dict(num_atoms=2)), ('rainbow', dict(num_atoms=33)),
    ('qrdqn', dict(num_quantiles=1)), ('qrdqn', dict(num_quantiles=256)),
], ids=lambda x: '-'.join('%s%d' % (k.replace('num_', ''), v) for k, v in x.items()) if isinstance(x, dict) else x)
def test_head_widths(kind, case, B):
  check(kind, 44, B, True, **case)


# ---- loss hyperparameters other than the defaults ----------------------------------------------------------------------
# vmax, grad_error_bound and huber_param travel from the learner's configuration to the loss kernels; a value dropped or
# hard-coded on the way runs the default (10, 1/32, 1) and fails these bars.

@pytest.mark.parametrize('kind,case', [
    ('c51', dict(vmax=3.0)), ('c51', dict(vmax=50.0)), ('rainbow', dict(vmax=3.0)), ('rainbow', dict(vmax=50.0)),
    ('qrdqn', dict(huber_param=0.0)), ('qrdqn', dict(huber_param=3.0)),
    ('iqn', dict(huber_param=0.0)), ('iqn', dict(huber_param=3.0)),
    ('dqn', dict(grad_error_bound=1.0)), ('dqn', dict(grad_error_bound=1.0 / 1024)),
    ('prioritized', dict(grad_error_bound=1.0)), ('prioritized', dict(grad_error_bound=1.0 / 1024)),
], ids=lambda x: '-'.join('%s%g' % kv for kv in x.items()) if isinstance(x, dict) else x)
def test_non_default_loss_hyperparameters(kind, case):
  check(kind, 44, 32, True, **case)


def test_three_optimizer_steps_with_a_non_default_support():
  check_three_optimizer_steps('c51', 44, 32, vmax=3.0)


# ---- optimizer steps -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hw,B', [(84, 64), ((84, 92), 32)])
@pytest.mark.parametrize('kind', ['rainbow', 'dqn'])
def test_three_optimizer_steps_at_other_shapes(kind, hw, B):
  """rainbow (Adam) and dqn (centred RMSProp) at batch 64 and on a non-square observation."""
  check_three_optimizer_steps(kind, hw, B)
