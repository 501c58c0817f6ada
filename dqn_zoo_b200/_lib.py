"""ctypes binding of include/dqn_zoo_b200.h (the C ABI).  No compute happens in Python.

The CUDA library is mandatory: importing this module raises if it is missing, and every
entry point raises on a non-zero status.  There is no CPU fallback anywhere in the package.
"""

import ctypes as C
import os

from dqn_zoo_b200 import _build

i32, i64, f32, f64, u64 = C.c_int32, C.c_int64, C.c_float, C.c_double, C.c_uint64
vp = C.c_void_p

DZ_FLAG_BAD_VALUE, DZ_FLAG_BAD_INDEX, DZ_FLAG_BAD_TARGET, DZ_FLAG_ROOT_ZERO, DZ_FLAG_NONFINITE_WEIGHT = 1, 2, 4, 8, 16
DZ_FLAG_FRAME_POOL_FULL = 32
DZ_CKPT_BAD_PLANE_ID, DZ_CKPT_UNREFERENCED_PLANE, DZ_CKPT_HASH_MISMATCH, DZ_CKPT_BAD_FREE_STACK = 1, 2, 4, 8
AGENT_KINDS = {'dqn': 0, 'double_q': 1, 'prioritized': 2, 'c51': 3, 'qrdqn': 4, 'rainbow': 5, 'iqn': 6, 'munchausen': 7,
               'munchausen_iqn': 8, 'fqf': 9}
OPTIMIZERS = {'adam': 0, 'rmsprop': 1}


class ReplayView(C.Structure):
  _fields_ = [('d_obs', vp), ('d_action', vp), ('d_reward', vp), ('d_discount', vp), ('capacity', i64),
              ('obs_bytes', i64), ('obs_stride', i64), ('d_tree', vp), ('first_leaf', i64), ('d_live', vp),
              ('d_id_at', vp), ('d_ids', vp), ('d_flags', vp),
              # frame-deduplicated layout (all NULL / 0: transition-major)
              ('d_frames', vp), ('frame_bytes', i64), ('frame_stride', i64), ('obs_channels', i64),
              ('frame_capacity', i64), ('d_planes', vp), ('d_refcount', vp), ('d_hashes', vp), ('d_table', vp),
              ('table_size', i64), ('d_free', vp), ('d_pool_counters', vp), ('d_add_staging', vp)]


class AddRecord(C.Structure):
  _fields_ = [('slot', i64), ('action', i32), ('reward', f64), ('discount', f64), ('n_patches', i32),
              ('patch_pos', i64 * 4), ('patch_val', i64 * 4), ('patch_target', i32 * 4), ('tree_index', i64),
              ('leaf_value', f64), ('evict_index', i64), ('size_after', i64), ('d_priority', vp), ('alpha', f64),
              ('release_row', i32)]


class AddBatch(C.Structure):   # struct dz_add_batch
  _fields_ = [('count', i32), ('first_slot', i64), ('d_action', vp), ('d_reward', vp), ('d_discount', vp),
              ('d_release_row', vp), ('d_tree_index', vp), ('d_evict_index', vp), ('d_leaf_value', vp),
              ('d_priority', vp), ('alpha', f64), ('n_patches', i32), ('d_patch_pos', vp), ('d_patch_val', vp),
              ('d_patch_target', vp), ('s_tm1', vp), ('s_t', vp), ('src_pitch', i64)]


class SampleInputs(C.Structure):
  _fields_ = [('d_rand_pos', vp), ('d_u_tree', vp), ('d_u_mix', vp), ('d_scalars', vp)]


class SampleOutputs(C.Structure):
  _fields_ = [('d_ids', vp), ('d_indices', vp), ('d_slots', vp), ('d_probs', vp), ('d_weights', vp)]


class LearnerConfig(C.Structure):
  _fields_ = [('kind', i32), ('num_actions', i32), ('num_atoms', i32), ('num_quantiles', i32), ('latent_dim', i32),
              ('tau_samples_s_tm1', i32), ('tau_samples_policy', i32), ('tau_samples_s_t', i32), ('batch', i32),
              ('obs_h', i32), ('obs_w', i32), ('obs_c', i32), ('vmax', f32), ('grad_error_bound', f32),
              ('huber_param', f32), ('optimizer', i32), ('learning_rate', f32), ('opt_eps', f32), ('rms_decay', f32),
              ('adam_b1', f32), ('adam_b2', f32), ('max_global_grad_norm', f32), ('munchausen_alpha', f32),
              ('entropy_temperature', f32), ('log_policy_clip', f32), ('num_fractions', i32),
              ('fraction_learning_rate', f32), ('fraction_opt_eps', f32), ('fraction_rms_decay', f32), ('dueling', i32),
              ('noisy', i32), ('random_shift_pad', i32), ('prioritized', i32), ('cql_alpha', f32)]

  def __init__(self, **fields):
    # the loss hyperparameters start at the reference's values instead of 0, which the library rejects for vmax, and
    # fqf's fraction fields at its defaults (DESIGN.md §15), which the library rejects at 0 for that kind
    super().__init__(**dict(dict(vmax=10.0, grad_error_bound=1.0 / 32, huber_param=1.0, num_fractions=32,
                                 fraction_learning_rate=2.5e-9, fraction_opt_eps=1e-5, fraction_rms_decay=0.95), **fields))


class LearnerPlan(C.Structure):
  _fields_ = [('param_count', i64), ('num_tensors', i32), ('opt_state_floats', i64), ('workspace_bytes', i64),
              ('noise_floats', i64), ('tau_floats', i64)]


class LearnerBuffers(C.Structure):
  _fields_ = [('d_online', vp), ('d_target', vp), ('d_grads', vp), ('d_opt_state', vp), ('d_workspace', vp),
              ('d_counters', vp)]


class Batch(C.Structure):
  _fields_ = [('d_s_tm1_rows', vp), ('d_s_t_rows', vp), ('d_a_tm1', vp), ('d_r_t', vp), ('d_discount_t', vp),
              ('d_weights', vp), ('d_taus', vp), ('d_noise', vp), ('d_shifts', vp)]


class UpdateOutputs(C.Structure):
  # d_regularizer last, so that positional UpdateOutputs(loss, per_example, priorities, grad_norm) leaves it NULL
  _fields_ = [('d_loss', vp), ('d_per_example', vp), ('d_priorities', vp), ('d_grad_norm', vp), ('d_regularizer', vp)]


class ResampleAxis(C.Structure):   # struct dz_resample_axis
  _fields_ = [('d_bounds', C.c_void_p), ('d_kk', C.c_void_p), ('ksize', C.c_int32), ('in_size', C.c_int32),
              ('out_size', C.c_int32)]


class LearnIO(C.Structure):
  _fields_ = [('sample_in', SampleInputs), ('sample_out', SampleOutputs), ('d_taus', vp), ('d_noise', vp),
              ('update_out', UpdateOutputs), ('d_max_seen_priority', vp), ('priority_exponent', f64), ('d_shifts', vp)]


class GameConfig(C.Structure):   # struct dz_game_config: dz_catch_config, dz_breakout_config, dz_pong_config
  _fields_ = [('num_streams', i32), ('num_actions', i32), ('min_noop_steps', i32), ('max_noop_steps', i32),
              ('seed', C.c_uint32), ('stream_offset', C.c_uint32)]


CatchConfig = BreakoutConfig = PongConfig = GameConfig

CATCH_STATE_FIELDS = ('paddle_x', 'ball_x', 'ball_y', 'ball_dx', 'lives', 'balls_left', 'counter', 'noops', 'over')
CATCH_MAX_STREAMS = 4096
CATCH_MAX_NOOP_STEPS = 89


BREAKOUT_STATE_FIELDS = ('paddle_x', 'ball_x', 'ball_y', 'ball_dx', 'ball_dy', 'in_play', 'serve_timer', 'lives',
                         'row0', 'row1', 'row2', 'row3', 'row4', 'row5', 'counter', 'noops', 'over')
BREAKOUT_MAX_STREAMS = 4096
BREAKOUT_MAX_NOOP_STEPS = 63


PONG_STATE_FIELDS = ('paddle_y', 'opponent_y', 'ball_x', 'ball_y', 'ball_dx', 'ball_dy', 'in_play', 'serve_timer',
                     'agent_score', 'opponent_score', 'counter', 'noops', 'over')
PONG_MAX_STREAMS = 4096
PONG_MAX_NOOP_STEPS = 63


class DzError(RuntimeError):
  pass


_ERRORS = {-1: ValueError, -2: DzError, -3: IndexError, -4: DzError}

_SIGNATURES = {
    'dz_last_error': (C.c_char_p, []),
    'dz_build_info': (C.c_char_p, []),
    'dz_launch_count': (i64, []),
    'dz_profile_begin': (i32, []),
    'dz_profile_end': (i32, [C.c_char_p, i64]),
    'dz_sumtree_rebuild': (i32, [vp, i64, i64, vp]),
    'dz_sumtree_set': (i32, [vp, i64, i64, vp, vp, i64, vp, vp]),
    'dz_sumtree_query': (i32, [vp, i64, vp, i64, vp, vp, vp]),
    'dz_sumtree_get': (i32, [vp, i64, i64, vp, i64, vp, vp, vp]),
    'dz_replay_add': (i32, [C.POINTER(ReplayView), C.POINTER(AddRecord), vp, vp, vp]),
    'dz_replay_add_batch_workspace': (i32, [C.POINTER(ReplayView), C.POINTER(i32), C.POINTER(i64)]),
    'dz_replay_add_batch': (i32, [C.POINTER(ReplayView), C.POINTER(AddBatch), vp, i64, vp]),
    'dz_replay_fill_synthetic': (i32, [C.POINTER(ReplayView), i64, i64, u64, i32, f64, vp]),
    'dz_replay_fill_synthetic_stacked': (i32, [C.POINTER(ReplayView), i64, u64, i64, i32, f64, vp]),
    'dz_replay_frame_pool_reset': (i32, [C.POINTER(ReplayView), vp]),
    'dz_replay_frames_in_use': (i32, [C.POINTER(ReplayView), C.POINTER(i64), vp]),
    'dz_replay_sample': (i32, [C.POINTER(ReplayView), i32, C.POINTER(SampleInputs), C.POINTER(SampleOutputs), i32, vp]),
    'dz_replay_gather': (i32, [C.POINTER(ReplayView), vp, i32, vp, vp, vp, vp, vp, vp]),
    'dz_replay_update_priorities': (i32, [C.POINTER(ReplayView), vp, vp, i32, f64, i64, vp]),
    'dz_ckpt_digest': (i32, [vp, i64, vp, vp]),
    'dz_ckpt_digest_host': (i32, [vp, i64, C.POINTER(u64)]),
    'dz_ckpt_pool_live': (i32, [C.POINTER(ReplayView), vp, vp, vp, vp]),
    'dz_ckpt_snapshot': (i32, [C.POINTER(ReplayView), vp, i64, vp, i64, vp, vp]),
    'dz_ckpt_pool_scatter': (i32, [C.POINTER(ReplayView), vp, i64, vp, vp, vp]),
    'dz_ckpt_pool_rebuild': (i32, [C.POINTER(ReplayView), vp, i64, vp, vp, i64, i64, vp, vp]),
    'dz_ckpt_rows': (i32, [C.POINTER(ReplayView), i64, i64, vp, i32, vp]),
    'dz_learner_plan_query': (i32, [C.POINTER(LearnerConfig), C.POINTER(LearnerPlan)]),
    'dz_learner_tensor_info': (i32, [C.POINTER(LearnerConfig), i32, C.c_char_p, C.POINTER(i64), C.POINTER(i32),
                                     C.POINTER(i64)]),
    'dz_learner_create': (i32, [C.POINTER(LearnerConfig), C.POINTER(LearnerBuffers), C.POINTER(vp)]),
    'dz_learner_destroy': (None, [vp]),
    'dz_learner_update': (i32, [vp, C.POINTER(Batch), C.POINTER(UpdateOutputs), i32, vp]),
    'dz_learner_learn': (i32, [vp, C.POINTER(ReplayView), i32, C.POINTER(LearnIO), vp]),
    'dz_learner_generate_randomness': (i32, [vp, u64, vp, vp, vp]),
    'dz_learner_generate_randomness_async': (i32, [vp, u64, vp, vp, vp]),
    'dz_learner_generate_shifts': (i32, [vp, u64, vp, vp]),
    'dz_learner_act_batch': (i32, [vp, vp, i32, vp, vp, i64, vp, f32, vp, vp, vp]),
    'dz_learner_noise_stride': (i32, [C.POINTER(LearnerConfig), C.POINTER(i64)]),
    'dz_learner_generate_stream_noise': (i32, [vp, u64, i32, vp, vp]),
    'dz_actor_plan_query': (i32, [C.POINTER(LearnerConfig), i32, C.POINTER(i64)]),
    'dz_actor_create': (i32, [vp, i32, vp, C.POINTER(vp)]),
    'dz_actor_destroy': (None, [vp]),
    'dz_actor_act': (i32, [vp, vp, vp, vp, i64, vp, f32, vp, vp, vp]),
    'dz_actor_generate_randomness': (i32, [vp, u64, i32, vp, vp]),
    'dz_actor_frozen_plan_query': (i32, [C.POINTER(LearnerConfig), i32, C.POINTER(i64)]),
    'dz_actor_create_frozen': (i32, [vp, i32, vp, C.POINTER(vp)]),
    'dz_actor_load_params': (i32, [vp, vp, vp]),
    'dz_actor_get_params': (i32, [vp, vp, vp]),
    'dz_actor_get_counter': (i32, [vp, C.POINTER(i64), vp]),
    'dz_actor_set_counter': (i32, [vp, i64, vp]),
    'dz_test_actor_mma_path': (i32, [vp, C.c_char_p, C.POINTER(i32)]),
    'dz_test_actor_buffer': (i32, [vp, C.c_char_p, vp, vp]),
    'dz_learner_sync_target': (i32, [vp, vp]),
    'dz_test_u8_to_unit': (i32, [vp, vp]),
    'dz_atari_preprocess': (i32, [vp, vp, i32, vp, vp, vp, vp, i32, vp, i32, vp]),
    'dz_atari_preprocess_band_rows': (i32, []),
    'dz_jax_uniform': (i32, [vp, vp, i32, vp, vp]),
    'dz_test_threefry2x32': (i32, [C.c_uint32, C.c_uint32, C.c_uint32, C.c_uint32, vp]),
    'dz_catch_step': (i32, [C.POINTER(CatchConfig), vp, vp, vp, vp, vp, vp, vp]),
    'dz_catch_render': (i32, [C.POINTER(CatchConfig), vp, vp, vp]),
    'dz_test_catch_step': (i32, [C.POINTER(CatchConfig), vp, i32, i32, vp, vp]),
    'dz_breakout_step': (i32, [C.POINTER(BreakoutConfig), vp, vp, vp, vp, vp, vp, vp]),
    'dz_breakout_render': (i32, [C.POINTER(BreakoutConfig), vp, vp, vp]),
    'dz_test_breakout_step': (i32, [C.POINTER(BreakoutConfig), vp, i32, i32, vp, vp]),
    'dz_pong_step': (i32, [C.POINTER(PongConfig), vp, vp, vp, vp, vp, vp, vp]),
    'dz_pong_render': (i32, [C.POINTER(PongConfig), vp, vp, vp]),
    'dz_test_pong_step': (i32, [C.POINTER(PongConfig), vp, i32, i32, vp, vp]),
    'dz_test_learner_buffer': (i32, [vp, C.c_char_p, vp, vp]),
    'dz_test_munchausen_example': (i32, [vp, vp, vp, i32, i32, f32, f32, f32, f32, f32, vp]),
    'dz_test_munchausen_iqn_example': (i32, [vp, vp, i32, i32, i32, i32, f32, f32, f32, f32, f32, vp]),
    'dz_test_fqf_example': (i32, [vp, vp, vp, i32, f32, vp]),
    'dz_test_dueling_example': (i32, [vp, f32, vp, i32, vp]),
    'dz_test_cql_example': (i32, [vp, i32, i32, f32, vp]),
    'dz_test_loss': (i32, [C.POINTER(LearnerConfig), i32, C.POINTER(vp), C.POINTER(vp), vp, vp, vp, vp, vp, vp, vp, vp, vp,
                           vp, vp, vp, vp]),
    'dz_test_loss_fqf': (i32, [C.POINTER(LearnerConfig), i32, C.POINTER(vp), vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp,
                               vp]),
    'dz_test_q_values': (i32, [C.POINTER(LearnerConfig), i32, vp, vp, vp, f32, vp, vp, vp]),
    'dz_test_q_values_fqf': (i32, [C.POINTER(LearnerConfig), i32, vp, vp, vp, f32, vp, vp, vp]),
    'dz_test_fraction_forward': (i32, [vp, i32, i32, C.POINTER(vp), vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                       C.POINTER(vp), vp, vp, vp]),
    'dz_test_dueling_head_fwd': (i32, [vp, i32, i32, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), i64, C.POINTER(vp), vp]),
    'dz_test_dueling_head_bwd': (i32, [vp, i32, vp, vp, C.POINTER(vp), vp, vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                       vp]),
    'dz_test_noisy_head_fwd': (i32, [vp, i32, i32, C.POINTER(vp), C.POINTER(vp), vp, C.POINTER(vp), vp]),
    'dz_test_noisy_head_bwd': (i32, [vp, i32, C.POINTER(vp), vp, vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(vp),
                                     C.POINTER(vp), vp]),
    'dz_test_iqn_cos': (i32, [vp, i64, i32, vp, vp]),
    'dz_test_iqn_head_fwd': (i32, [vp, i32, C.POINTER(i32), C.POINTER(vp), C.POINTER(vp), C.POINTER(vp), vp]),
    'dz_test_iqn_head_dgrad': (i32, [vp, i32, vp, vp, vp, vp, vp]),
    'dz_test_iqn_hadamard_bwd': (i32, [i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, i32, vp]),
    'dz_test_copy': (i32, [vp, vp, i64, vp]),
    'dz_test_random_shift': (i32, [vp, vp, vp, i32, i32, i32, i32, i32, vp, i64, vp]),
    'dz_test_learner_trace': (i32, [vp, C.c_char_p, vp]),
    'dz_test_learner_mma_path': (i32, [vp, C.c_char_p, C.POINTER(i32)]),
    'dz_debug_timeline': (i32, [vp]),
    'dz_test_tc_pgemm_work': (i64, [i32, i32, i32]),
    'dz_test_tc_pgemm': (i32, [vp, i32, i32, i32, vp, i32, i32, i32, i32, i32, vp, vp, i64, i64, i32, i64, vp, i32, vp]),
    'dz_test_iqn_embed_packed': (i32, [vp, i32, i32, vp, i32, vp, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp]),
    'dz_test_umma_gemm': (i32, [vp, i32, vp, i32, i32, i32, i32, i32, vp, i32, i32, vp, i32, vp, vp, vp, vp]),
    'dz_test_umma_gemm_path': (i32, [vp, i32, vp, i32, i32, i32, i32, i32, vp, i32, i32, vp, i32, vp, vp, vp, i32, vp]),
    'dz_test_fc_forward': (i32, [i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, i64, vp, vp, vp, i32, vp, C.POINTER(i32),
                                 C.POINTER(i64), vp]),
    'dz_test_fc_dgrad': (i32, [i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, i32, vp, C.POINTER(i32), vp]),
    'dz_test_conv1_forward': (i32, [i32, i32, i32, i32, vp, vp, vp, i64, vp, i32, vp, vp, vp]),
}

EXPORTS = tuple(_SIGNATURES)


def library_path():
  return _build.LIB_PATH


def _load():
  path = library_path()
  if not os.path.exists(path):
    raise ImportError('dqn_zoo_b200: %s is missing — run `python -c "import __graft_entry__ as g; g.build()"` '
                      '(there is no CPU fallback)' % path)
  lib = C.CDLL(path)
  for name, (res, args) in _SIGNATURES.items():
    fn = getattr(lib, name)
    fn.restype, fn.argtypes = res, args
  return lib


lib = _load()


def check(status):
  if status != 0:
    raise _ERRORS.get(status, DzError)(lib.dz_last_error().decode())


def call(name, *args):
  check(getattr(lib, name)(*args))
