"""CPU: host-side logic that needs no GPU — parts.run_loop call tape, LinearSchedule values, the C-ABI
library's exported symbols, and the multi-rank target broadcast / throughput aggregation on gloo."""

import ctypes
import os
import re
import subprocess
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_linear_schedule_values():
  """parts_test.py:29-75."""
  from dqn_zoo_b200 import parts
  s = parts.LinearSchedule(begin_t=5, decay_steps=7, begin_value=1.0, end_value=0.3)
  for t in range(20):
    want = 1.0 if t <= 5 else (0.3 if t >= 12 else (1.0 - (t - 5) / 7 * 0.7))
    assert abs(s(t) - want) < 1e-12
  s2 = parts.LinearSchedule(begin_t=5, end_t=12, begin_value=1.0, end_value=0.3)
  assert all(abs(s(t) - s2(t)) < 1e-15 for t in range(20))
  with pytest.raises(ValueError):
    parts.LinearSchedule(begin_value=0.0, end_value=1.0, begin_t=0)
  with pytest.raises(ValueError):
    parts.LinearSchedule(begin_value=0.0, end_value=1.0, begin_t=0, end_t=5, decay_steps=5)


class _TapeAgent:
  def __init__(self, tape):
    self.tape = tape

  def reset(self):
    self.tape.append('agent.reset')

  def step(self, ts):
    self.tape.append('agent.step(%s)' % ts.observation)
    return 7


class _TapeEnv:
  def __init__(self, tape, episode_len):
    self.tape, self.n, self.t = tape, episode_len, 0

  def reset(self):
    from dqn_zoo_b200 import parts
    self.tape.append('env.reset')
    self.t = 0
    return parts.TimeStep(parts.StepType.FIRST, None, None, 0)

  def step(self, action):
    from dqn_zoo_b200 import parts
    self.t += 1
    self.tape.append('env.step(%d)' % action)
    st = parts.StepType.LAST if self.t >= self.n else parts.StepType.MID
    return parts.TimeStep(st, 0.0, 1.0, self.t)


def test_run_loop_call_tape_and_truncation():
  """parts_test.py:110-166: exact alternation, extra agent step on LAST, max_steps truncation,
  yield_before_reset."""
  from dqn_zoo_b200 import parts
  tape = []
  loop = parts.run_loop(_TapeAgent(tape), _TapeEnv(tape, 3))
  out = [next(loop) for _ in range(5)]
  assert tape == ['agent.reset', 'env.reset', 'agent.step(0)', 'env.step(7)', 'agent.step(1)', 'env.step(7)',
                  'agent.step(2)', 'env.step(7)', 'agent.step(3)', 'agent.reset', 'env.reset', 'agent.step(0)']
  assert [o[3] for o in out] == [7, 7, 7, None, 7]
  assert out[3][1].last()
  tape = []
  loop = parts.run_loop(_TapeAgent(tape), _TapeEnv(tape, 100), max_steps_per_episode=2)
  out = [next(loop) for _ in range(3)]
  assert out[2][1].last() and out[2][3] is None          # truncated to LAST after 2 steps
  tape = []
  loop = parts.run_loop(_TapeAgent(tape), _TapeEnv(tape, 2), yield_before_reset=True)
  first = next(loop)
  assert first[1] is None and first[3] is None and tape == []


def test_c_abi_library_exports_every_declared_symbol():
  """include/dqn_zoo_b200.h <-> the built shared library <-> the ctypes binding (no compute calls)."""
  from dqn_zoo_b200 import _build
  header = open(os.path.join(ROOT, 'include', 'dqn_zoo_b200.h')).read()
  declared = set(re.findall(r'\b(dz_[a-z0-9_]+)\s*\(', header))
  declared -= {'dz_agent_kind', 'dz_optimizer_kind'}
  assert len(declared) >= 20
  path = _build.build()
  lib = ctypes.CDLL(path)
  for name in sorted(declared):
    assert hasattr(lib, name), 'library does not export %s' % name
  from dqn_zoo_b200 import _lib
  assert set(_lib.EXPORTS) == declared, set(_lib.EXPORTS) ^ declared
  assert b'sm_90a' in _lib.lib.dz_build_info()
  # argument validation happens before any CUDA call
  cfg = _lib.LearnerConfig()
  cfg.kind = 99
  plan = _lib.LearnerPlan()
  with pytest.raises(ValueError):
    _lib.call('dz_learner_plan_query', ctypes.byref(cfg), ctypes.byref(plan))


def test_loss_hyperparameters_are_validated_for_every_kind():
  """vmax, grad_error_bound and huber_param reach the loss kernels as given: non-finite values, vmax <= 0 and a
  negative bound or Huber width are refused by validate() (here through dz_learner_plan_query, which does no device
  work), for every kind; the defaults and the boundary values 0 of the bound and the width pass."""
  from dqn_zoo_b200 import _lib
  plan = _lib.LearnerPlan()

  def cfg(kind, **fields):
    c = _lib.LearnerConfig(**fields)
    c.kind = _lib.AGENT_KINDS[kind]
    c.num_actions, c.num_atoms, c.num_quantiles, c.latent_dim = 6, 51, 201, 64
    c.tau_samples_s_tm1 = c.tau_samples_policy = c.tau_samples_s_t = 64
    c.batch, c.obs_h, c.obs_w, c.obs_c = 32, 84, 84, 4
    c.munchausen_alpha, c.entropy_temperature, c.log_policy_clip = 0.9, 0.03, -1.0
    return c

  nan, inf = float('nan'), float('inf')
  bad = [('vmax', 0.0), ('vmax', -1.0), ('vmax', nan), ('vmax', inf), ('huber_param', -1e-3), ('huber_param', nan),
         ('huber_param', inf), ('grad_error_bound', -1.0 / 32), ('grad_error_bound', nan), ('grad_error_bound', -inf)]
  for kind in _lib.AGENT_KINDS:
    _lib.call('dz_learner_plan_query', ctypes.byref(cfg(kind)), ctypes.byref(plan))
    _lib.call('dz_learner_plan_query', ctypes.byref(cfg(kind, grad_error_bound=0.0, huber_param=0.0, vmax=1e-3)),
              ctypes.byref(plan))
    for field, value in bad:
      with pytest.raises(ValueError, match=field):
        _lib.call('dz_learner_plan_query', ctypes.byref(cfg(kind, **{field: value})), ctypes.byref(plan))


def test_parameter_layout_matches_the_oracle_shapes():
  from dqn_zoo_b200 import _lib
  from oracle import learner_oracle as lo
  for kind in lo.AGENT_KINDS:
    cfg = _lib.LearnerConfig()
    cfg.kind = _lib.AGENT_KINDS[kind]
    cfg.num_actions, cfg.num_atoms, cfg.num_quantiles, cfg.latent_dim = 6, 51, 201, 64
    cfg.tau_samples_s_tm1 = cfg.tau_samples_policy = cfg.tau_samples_s_t = 64
    cfg.batch, cfg.obs_h, cfg.obs_w, cfg.obs_c = 32, 84, 84, 4
    plan = _lib.LearnerPlan()
    _lib.call('dz_learner_plan_query', ctypes.byref(cfg), ctypes.byref(plan))
    want = lo.param_shapes(lo.NetSpec(kind, 6))
    assert plan.num_tensors == len(want)
    name = ctypes.create_string_buffer(64)
    shape = (ctypes.c_int64 * 4)()
    ndim, off = ctypes.c_int32(), ctypes.c_int64()
    total = 0
    for i, (wname, wshape) in enumerate(want.items()):
      _lib.call('dz_learner_tensor_info', ctypes.byref(cfg), i, name, shape, ctypes.byref(ndim), ctypes.byref(off))
      assert name.value.decode() == wname
      assert tuple(shape[k] for k in range(ndim.value)) == tuple(wshape)
      assert off.value % 4 == 0 and off.value >= total
      total = off.value + int(np.prod(wshape))
    # SURVEY §8(a): P = 1,687,206 (dqn) ... 6,868,485 (rainbow), up to 4-float alignment padding per tensor
    exact = sum(int(np.prod(s)) for s in want.values())
    assert exact <= plan.param_count <= exact + 4 * len(want)


_WORKER = r'''
import os, sys
sys.path.insert(0, %(root)r)
import torch, torch.distributed as dist
from dqn_zoo_b200 import distributed as dd
dist.init_process_group('gloo', init_method='tcp://127.0.0.1:%(port)d', rank=int(sys.argv[1]), world_size=2)
rank = dist.get_rank()
online = torch.full((1000,), float(rank + 1))
target = torch.zeros(1000)
dd.broadcast_target(online, target, dist, src=0)
assert torch.equal(target, torch.full((1000,), 1.0)), target[:3]     # every shard bootstraps from rank 0's online net
assert torch.equal(online, torch.full((1000,), float(rank + 1)))    # online nets stay per-shard
ms = torch.tensor([10.0 + 5 * rank], dtype=torch.float64)
dist.all_reduce(ms, op=dist.ReduceOp.MAX)
assert abs(dd.aggregate_throughput(100, 2, float(ms)) - 2 * 100 / 0.015) < 1e-9
assert dd.shard_seed(1, rank) == 1 + rank
dist.barrier()
dist.destroy_process_group()
print('ok', rank)
'''


def test_two_rank_target_broadcast_and_aggregation_on_gloo(tmp_path):
  port = 29000 + os.getpid() % 2000
  script = tmp_path / 'worker.py'
  script.write_text(_WORKER % {'root': ROOT, 'port': port})
  procs = [subprocess.Popen([sys.executable, str(script), str(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                            text=True) for r in range(2)]
  outs = [p.communicate(timeout=240)[0] for p in procs]
  for r, (p, o) in enumerate(zip(procs, outs)):
    assert p.returncode == 0, o
    assert 'ok %d' % r in o


def test_bilinear_axis_tables_match_oracle():
  """Host half of the device preprocessing: Pillow's window/coefficient tables (processors.py:381-386 -> PIL)."""
  from dqn_zoo_b200 import processors
  from oracle import processors_oracle as po
  for in_size, out_size in [(160, 84), (210, 84), (100, 42), (96, 50), (84, 84), (50, 84), (7, 5)]:
    b, k, ks = processors.bilinear_axis(in_size, out_size)
    ob, ok, oks = po.resample_coeffs(in_size, out_size)
    assert ks == oks and np.array_equal(b, ob) and np.array_equal(k, ok)
  assert processors.LUMA == po.LUMA


def test_codec_pair_is_validated_on_the_host():
  """replay.py:148,155: the reference stores encoder(item) and hands out decoder(stored).  The device replay takes the
  pair and applies the round trip at insert; giving only one of the two is an error (checked before any CUDA call)."""
  from dqn_zoo_b200 import replay
  assert replay._check_codec(None, None) is None
  rt = replay._check_codec(lambda t: t._replace(r_t=t.r_t * 2), lambda t: t._replace(r_t=t.r_t / 2))
  item = replay.Transition(s_tm1=1, a_tm1=2, r_t=3.0, discount_t=0.5, s_t=4)
  assert rt(item) == item
  import pytest
  with pytest.raises(ValueError):
    replay._check_codec(lambda t: t, None)


def test_cpu_reference_arm_thread_calibration():
  """The `--impl reference` arm calibrates its OpenMP thread count (64 threads were 3-4x slower than 8-16 on the GPU box's
  host): pick_threads keeps the fastest candidate within the CPUs the process may use and leaves torch set to it."""
  import time
  import torch
  from oracle import cpu_reference as cr
  limit = cr.cgroup_cpu_limit()
  assert isinstance(limit, int) and limit >= 1

  class FakeLearner:
    calls = []

    def update(self, *inputs):
      t = torch.get_num_threads()
      self.calls.append(t)
      time.sleep(0.002 if t == 8 else 0.02)   # 8 threads is the optimum of this fake

  before = torch.get_num_threads()
  try:
    fake = FakeLearner()
    best = cr.pick_threads(fake, lambda: (), 64)
    assert best == 8 and torch.get_num_threads() == 8
    assert set(fake.calls) <= {4, 8, 16, 32, 64}
    # a limit below the smallest candidate falls back to the limit itself
    assert cr.pick_threads(FakeLearner(), lambda: (), 2) == 2
  finally:
    torch.set_num_threads(before)
