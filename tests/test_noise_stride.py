"""CPU: `dz_learner_noise_stride`, the floats of one rainbow noise apply (the row stride of per-stream noise)."""

import ctypes

import pytest


def _cfg(kind, hw, num_actions, num_atoms):
  from dqn_zoo_b200 import _lib
  cfg = _lib.LearnerConfig()
  cfg.kind = _lib.AGENT_KINDS[kind]
  cfg.num_actions, cfg.num_atoms, cfg.num_quantiles, cfg.latent_dim = num_actions, num_atoms, 201, 64
  cfg.tau_samples_s_tm1 = cfg.tau_samples_policy = cfg.tau_samples_s_t = 64
  cfg.batch, cfg.obs_h, cfg.obs_w, cfg.obs_c = 32, hw, hw, 4
  return cfg


@pytest.mark.parametrize('hw,num_actions,num_atoms', [(84, 6, 51), (44, 6, 21), (84, 18, 51), (36, 3, 2)])
def test_noise_stride_is_one_padded_apply(hw, num_actions, num_atoms):
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  cfg = _cfg('rainbow', hw, num_actions, num_atoms)
  stride = ctypes.c_int64()
  _lib.call('dz_learner_noise_stride', ctypes.byref(cfg), ctypes.byref(stride))
  net = dl.NetworkSpec('rainbow', num_actions, num_atoms=num_atoms, obs_shape=(hw, hw, 4))
  assert stride.value == sum((n + 3) // 4 * 4 for _, n in dl.noise_vector_sizes(net))
  plan = _lib.LearnerPlan()
  _lib.call('dz_learner_plan_query', ctypes.byref(cfg), ctypes.byref(plan))
  assert plan.noise_floats == 3 * stride.value


@pytest.mark.parametrize('kind', ['dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'iqn'])
def test_noise_stride_rejects_kinds_without_noisy_layers(kind):
  from dqn_zoo_b200 import _lib
  stride = ctypes.c_int64()
  with pytest.raises(ValueError):
    _lib.call('dz_learner_noise_stride', ctypes.byref(_cfg(kind, 84, 6, 51)), ctypes.byref(stride))
