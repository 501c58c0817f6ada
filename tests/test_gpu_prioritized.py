"""GPU: prioritized replay for every agent kind (DESIGN.md §19).  The weighted update of a prioritized learner of each
kind and network option against its float64 oracle, priorities by oracle/prioritized_oracle.py; weights of 1 against
the uniform update bit for bit; DoubleQ on a prioritized replay against PrioritizedDqn bit for bit; the fused step's
ids, sum tree and max-seen priority against oracle/replay_oracle.py; uniform steps untouched (launches, unwritten
priorities, a refused prioritized learn); agents through run_loop, state, checkpoints and the vectorised trainer; and
qrdqn and c51 on PER learning Catch."""

import copy
import os
import pickle

import numpy as np
import pytest
import torch

import learner_parity as lp
import test_gpu_dueling as tdu
import test_gpu_fqf as tfq
import test_gpu_munchausen as tmu
import test_gpu_munchausen_iqn as tmi
import test_gpu_noisy as tno
import test_gpu_vector_trainer as tvt
from oracle import learner_oracle as lo
from oracle import prioritized_oracle as po
from oracle import replay_oracle as ro

pytestmark = pytest.mark.gpu

KINDS = ('dqn', 'double_q', 'prioritized', 'c51', 'qrdqn', 'rainbow', 'iqn', 'munchausen', 'munchausen_iqn', 'fqf')
OTHER_KINDS = tuple(k for k in KINDS if k not in ('prioritized', 'rainbow'))

def _twin(L, prioritized=True):
  """A learner with L's configuration, parameters, optimizer state and counters; prioritized or not."""
  from dqn_zoo_b200 import learner as dl
  c = L.cfg
  T = dl.Learner(L.net, batch_size=L.batch_size, optimizer=L.opt, grad_error_bound=c.grad_error_bound,
                 huber_param=c.huber_param, munchausen_alpha=c.munchausen_alpha, entropy_temperature=c.entropy_temperature,
                 log_policy_clip=c.log_policy_clip, fraction_learning_rate=c.fraction_learning_rate,
                 fraction_opt_eps=c.fraction_opt_eps, fraction_rms_decay=c.fraction_rms_decay,
                 random_shift_pad=L.random_shift_pad, prioritized=prioritized)
  for name in ('online', 'target', 'opt_state', 'counters'):
    getattr(T, name).copy_(getattr(L, name))
  return T


def _weights(B, rs):
  """Importance weights in [0, 1] that include 0 and values below 1e-3."""
  w = rs.uniform(0.0, 1.0, B)
  w[0] = 0.0
  w[1 % B] = 5e-4
  if B > 2:
    w[2] = 3e-7
  return w


# ---- 1. parity with weights ----------------------------------------------------------------------------------------------

def _case(kind, net, hw, B):
  """(L, device update, oracle grads(tap), ReLU table) of one weighted update of a prioritized learner."""
  wrs = np.random.RandomState(100 + B)
  if net.get('noisy'):
    spec, nspec, L, O, rs = tno.make_case(kind, bool(net.get('dueling')), B, hw, 3)
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, nspec, B, rs)
    noise_o, noise_flat = tno._noise(spec, nspec, bool(net.get('dueling')), rs)
    w = _weights(B, wrs)
    L = _twin(L)
    return (L, lambda: L.update(*arrs, weights=w, noise=noise_flat, apply_update=False),
            lambda tap: O.grads(batch, torch.tensor(w), noise=noise_o, tap=tap), tno._table(bool(net.get('dueling'))))
  if net.get('dueling'):
    spec, nspec, L, O, rs = tdu.make_case(kind, B, hw, 3)
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, nspec, B, rs)
    w = _weights(B, wrs)
    L = _twin(L)
    return (L, lambda: L.update(*arrs, weights=w, apply_update=False),
            lambda tap: O.grads(batch, torch.tensor(w), tap=tap), 'rainbow')
  if kind == 'munchausen':
    spec, nspec, L, O, rs = tmu.make_case(B, hw, 3)
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, nspec, B, rs)
    w = _weights(B, wrs)
    L = _twin(L)
    return (L, lambda: L.update(*arrs, weights=w, apply_update=False),
            lambda tap: O.grads(batch, torch.tensor(w), tap=tap), 'dqn')
  if kind == 'munchausen_iqn':
    full = lp._hw(hw) == (84, 84)
    spec, nspec, L, O, rs = tmi.make_case(B, hw, 3, taus=(64, 64, 64) if full else (8, 5, 7))
    arrs, batch, taus_o, taus_flat = tmi.make_batch(nspec, B, rs)
    w = _weights(B, wrs)
    L = _twin(L)
    return (L, lambda: L.update(*arrs, weights=w, taus=taus_flat, apply_update=False),
            lambda tap: O.grads(batch, torch.tensor(w), taus=taus_o, tap=tap), 'iqn')
  if kind == 'fqf':
    spec, nspec, L, O, rs = tfq.make_case(B, hw, 3)
    arrs, batch = tfq.make_batch(nspec, B, rs)
    w = _weights(B, wrs)
    L = _twin(L)
    return (L, lambda: L.update(*arrs, weights=w, apply_update=False),
            lambda tap: O.grads(batch, torch.tensor(w), device_fractions=tfq.device_fractions(L), tap=tap), 'iqn')
  spec, nspec, L, O, rs = lp.make_case(kind, B, hw, seed=3)
  arrs, batch, _, taus_o, taus_flat, noise_o, noise_flat = lp.make_batch(spec, nspec, B, rs)
  w = _weights(B, wrs)
  L = _twin(L)
  return (L, lambda: L.update(*arrs, weights=w, taus=taus_flat, noise=noise_flat, apply_update=False),
          lambda tap: O.grads(batch, torch.tensor(w), taus_o, noise_o, tap=tap), kind)


PARITY = ([(k, {}) for k in KINDS] +
          [(k, n) for k in ('dqn', 'double_q', 'munchausen')
           for n in ({'dueling': True}, {'noisy': True}, {'dueling': True, 'noisy': True})])
PARITY_IDS = ['%s%s' % (k, ''.join('-' + o for o in sorted(n))) for k, n in PARITY]


def _check_parity(kind, net, hw, B):
  L, update, oracle_grads, table = _case(kind, net, hw, B)
  update()
  torch.cuda.synchronize()
  tap = lo.ReluTap()
  loss, aux, grads = oracle_grads(tap)
  assert abs(float(L.loss.item()) - float(loss)) <= lp.REL * abs(float(loss)), (float(L.loss.item()), float(loss))
  masks, flips = lp.relu_kink_flips(table, L, tap)
  lp.assert_flips_at_the_kink(flips)
  if flips:
    loss, aux, grads = oracle_grads(lo.ReluTap(masks))
  td_per_example = kind in ('dqn', 'double_q', 'prioritized')
  want_pe = aux['td_errors'] if td_per_example else aux['losses']
  assert lp.rel_err(L.per_example.cpu().numpy(), want_pe.numpy()) <= lp.REL
  if kind == 'fqf':
    gn = tfq.main_norm(grads)
  else:
    gn = float(torch.sqrt(sum((g * g).sum() for g in grads.values())))
  assert abs(float(L.grad_norm.item()) - gn) <= lp.REL * gn
  bad = {}
  for name in L.tensors:
    got, want = L.view(L.grads, name).cpu().numpy(), grads[name].numpy()
    if np.linalg.norm(want) < 1e-12 * max(gn, 1e-30):
      assert np.abs(got).max() <= 1e-9 * max(gn, 1.0), name
      continue
    if lp.rel_err(got, want) > lp.REL:
      bad[name] = lp.rel_err(got, want)
  assert not bad, bad
  pri = L.priorities.cpu()
  assert lp.rel_err(pri.numpy(), po.priorities(kind, aux).numpy()) <= lp.REL
  if kind in po.LOSS_KINDS:
    assert torch.equal(pri, L.per_example.cpu().abs().clamp(0.0, 100.0))
  return L


@pytest.mark.parametrize('hw,B', [(84, 32), (44, 5)], ids=['84x84-B32', '44x44-B5'])
@pytest.mark.parametrize('kind,net', PARITY, ids=PARITY_IDS)
def test_weighted_update_and_priorities_match_the_oracle(kind, net, hw, B):
  _check_parity(kind, net, hw, B)


@pytest.mark.parametrize('kind', ['dqn', 'c51', 'qrdqn', 'iqn', 'munchausen', 'fqf'])
def test_weighted_update_on_the_fp32_fma_torso(kind):
  L = _check_parity(kind, {}, (84, 88), 32)
  assert not lp.tensor_core_torso(L)


# ---- 2. weights of 1 -----------------------------------------------------------------------------------------------------

def _learner(kind, B=32, hw=(84, 84), prioritized=False, pad=0, **net):
  from dqn_zoo_b200 import learner as dl
  return dl.Learner(dl.NetworkSpec(kind, 6, obs_shape=(hw[0], hw[1], 4), **net), batch_size=B, prioritized=prioritized,
                    random_shift_pad=pad)


def _inputs(L, rs):
  from dqn_zoo_b200 import learner as dl
  B = L.batch_size
  H, W, Cc = L.net.obs_shape
  kw = dict(s_tm1=rs.randint(0, 256, (B, H, W, Cc)).astype(np.uint8), s_t=rs.randint(0, 256, (B, H, W, Cc)).astype(np.uint8),
            a_tm1=rs.randint(0, L.net.num_actions, B), r_t=rs.choice([-1.0, 0.0, 1.0, 0.37], size=B),
            discount_t=rs.choice([0.0, 0.99], size=B))
  if dl.draws_taus(L.kind):
    kw['taus'] = rs.uniform(size=L.plan.tau_floats).astype(np.float32)
  if dl.noisy_layers(L.net):
    kw['noise'] = rs.uniform(-1.4, 1.4, size=L.plan.noise_floats).astype(np.float32)
  return kw


@pytest.mark.parametrize('kind', OTHER_KINDS)
def test_weights_of_one_give_the_uniform_update_bit_for_bit(kind):
  uni = _learner(kind)
  uni.init_params(4)
  per = _twin(uni)
  rs = np.random.RandomState(9)
  for step in range(3):
    kw = _inputs(uni, rs)
    uni.update(**kw)
    per.update(weights=np.ones(uni.batch_size), **kw)
    torch.cuda.synchronize()
    for name in ('loss', 'per_example', 'grad_norm', 'grads', 'online', 'opt_state'):
      assert torch.equal(getattr(uni, name), getattr(per, name)), (step, name)


# ---- agents on replays ---------------------------------------------------------------------------------------------------

def _agent(kind, prioritized, capacity=512, seed=3, graph=True, dedup=False, pad=0, optimizer=None, min_fill=None,
           epsilon=0.1, n_step=1, preprocessor=None, **net):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  structure = dr.Transition(None, None, None, None, None)
  extra = dict(frame_dedup=True, frame_capacity=8 * (capacity + 1) + 1) if dedup else {}
  rs = np.random.RandomState(seed)
  if prioritized:
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.5, lambda t: 0.4, 1e-3, True, rs, **extra)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, **extra)
  common = dict(preprocessor=preprocessor, sample_network_input=None, optimizer=optimizer,
                network=dl.NetworkSpec(kind, 6, **net), transition_accumulator=dr.NStepTransitionAccumulator(n_step),
                replay=rep, batch_size=32, min_replay_capacity_fraction=(min_fill or capacity) / capacity, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=graph, random_shift_pad=pad)
  eps = lambda t: epsilon
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common), rep
  if kind == 'c51':
    return ag.C51(support=np.linspace(-10, 10, 51), exploration_epsilon=eps, **common), rep
  if kind == 'qrdqn':
    return ag.QrDqn(quantiles=(np.arange(201) + 0.5) / 201, exploration_epsilon=eps, huber_param=1.0, **common), rep
  if kind == 'fqf':
    return ag.Fqf(exploration_epsilon=eps, huber_param=1.0, **common), rep
  if dl.uses_iqn_network(kind):
    return ag.AGENTS[kind](exploration_epsilon=eps, huber_param=1.0, tau_samples_policy=64, tau_samples_s_tm1=64,
                           tau_samples_s_t=64, **common), rep
  return ag.AGENTS[kind](exploration_epsilon=eps, grad_error_bound=1.0 / 32, **common), rep


def _fill(rep, dedup, seed=3):
  from dqn_zoo_b200 import replay as dr
  if dedup:
    dr.bulk_fill_synthetic_stacked(rep, (84, 84, 4), seed, 6, episode_len=37)
  else:
    dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6)


def _tree(rep):
  return rep.get_state()['distribution']['sum_tree']['storage']


def test_the_replay_classes_say_whether_they_are_prioritized():
  from dqn_zoo_b200 import replay as dr
  assert dr.TransitionReplay.prioritized is False and dr.PrioritizedTransitionReplay.prioritized is True
  for kind in KINDS:
    uni, _ = _agent(kind, False, capacity=64)
    per, _ = _agent(kind, True, capacity=64)
    assert uni.PRIORITIZED == (kind in ('prioritized', 'rainbow')) and per.PRIORITIZED, kind
    assert per.max_seen_priority == 1.0 and per.importance_sampling_exponent == 0.4
    assert 'max_seen_priority' in per.get_state()
    if not uni.PRIORITIZED:
      assert not hasattr(uni, 'max_seen_priority') and not hasattr(uni, 'importance_sampling_exponent')
      assert 'max_seen_priority' not in uni.get_state()


# ---- 3. DoubleQ on PER is PrioritizedDqn -----------------------------------------------------------------------------------

@pytest.mark.parametrize('dedup', [False, True], ids=['dense', 'dedup'])
@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graph'])
def test_double_q_on_per_is_prioritized_dqn_bit_for_bit(graph, dedup):
  from dqn_zoo_b200 import learner as dl
  opt = dl.default_optimizer('prioritized')
  dq, rep_dq = _agent('double_q', True, graph=graph, dedup=dedup, optimizer=opt)
  pr, rep_pr = _agent('prioritized', True, graph=graph, dedup=dedup, optimizer=opt)
  _fill(rep_dq, dedup)
  _fill(rep_pr, dedup)
  assert torch.equal(dq.learner.online, pr.learner.online)
  for step in range(24):
    dq.learn()
    pr.learn()
    torch.cuda.synchronize()
    a, b = dq.learner, pr.learner
    assert torch.equal(a.sampled_ids, b.sampled_ids), step
    assert torch.equal(a.sampled_weights, b.sampled_weights), step
    assert np.array_equal(_tree(rep_dq), _tree(rep_pr)), step
    assert dq.max_seen_priority == pr.max_seen_priority, step
    for name in ('online', 'opt_state', 'priorities', 'loss'):
      assert torch.equal(getattr(a, name), getattr(b, name)), (step, name)


# ---- 4. the fused step against the replay oracle -------------------------------------------------------------------------

def _oracle_replay(cap, seed):
  orep = ro.PrioritizedTransitionReplay(cap, ro.Transition(None, None, None, None, None), 0.5, lambda t: 0.4, 1e-3, True,
                                        np.random.RandomState(seed))
  z = np.zeros(1, np.uint8)
  for _ in range(cap):   # the tree does not depend on the observations
    orep.add(ro.Transition(z, 0, 0.0, 0.0, z), 1.0)
  return orep


@pytest.mark.parametrize('kind,dedup,pad', [('c51', False, 0), ('qrdqn', True, 0), ('iqn', False, 0),
                                            ('munchausen', True, 0), ('fqf', False, 0), ('qrdqn', False, 4)],
                         ids=['c51-dense', 'qrdqn-dedup', 'iqn-dense', 'munchausen-dedup', 'fqf-dense', 'qrdqn-shift4'])
def test_fused_step_matches_the_replay_oracle_and_graph_is_eager(kind, dedup, pad):
  cap, seed = 512, 3
  graphed, rep_g = _agent(kind, True, graph=True, dedup=dedup, pad=pad, seed=seed)
  eager, rep_e = _agent(kind, True, graph=False, dedup=dedup, pad=pad, seed=seed)
  _fill(rep_g, dedup)
  _fill(rep_e, dedup)
  orep = _oracle_replay(cap, seed)
  assert np.array_equal(_tree(rep_g), _tree(orep))
  max_seen = 1.0
  L = graphed.learner
  for step in range(8):
    graphed.learn()
    eager.learn()
    torch.cuda.synchronize()
    ids, _, w = orep.sample_ids(32)
    assert np.array_equal(L.sampled_ids.cpu().numpy(), ids), step
    np.testing.assert_allclose(L.sampled_weights.cpu().numpy(), w, rtol=1e-14)
    pri = L.priorities.cpu().numpy()
    assert np.isfinite(pri).all() and (pri >= 0).all()
    if kind in po.LOSS_KINDS:
      assert np.array_equal(pri, np.clip(np.abs(L.per_example.cpu().numpy()), 0, 100))
    orep.update_priorities(ids, pri)
    assert np.array_equal(_tree(rep_g), _tree(orep)), step
    max_seen = max(max_seen, float(pri.max()))
    assert graphed.max_seen_priority == max_seen, step
    for name in ('online', 'opt_state', 'priorities', 'loss', 'max_seen_priority'):
      assert torch.equal(getattr(L, name), getattr(eager.learner, name)), (step, name)
    assert np.array_equal(_tree(rep_g), _tree(rep_e)), step
  graphed.check_device_flags()


# ---- 5. uniform steps are untouched -----------------------------------------------------------------------------------------

def _launches_per_step(agent):
  from dqn_zoo_b200 import _lib
  agent.learn()
  torch.cuda.synchronize()
  c0 = _lib.lib.dz_launch_count()
  agent.learn()
  torch.cuda.synchronize()
  return int(_lib.lib.dz_launch_count() - c0)


def test_per_adds_the_launches_it_adds_for_double_q():
  counts = {}
  for kind in OTHER_KINDS:
    for per in (False, True):
      agent, rep = _agent(kind, per, graph=False)
      _fill(rep, False)
      counts[kind, per] = _launches_per_step(agent)
  extra = counts['double_q', True] - counts['double_q', False]
  assert extra > 0
  for kind in OTHER_KINDS:
    assert counts[kind, True] - counts[kind, False] == extra, (kind, counts)
  print('launches per step (uniform, per):', {k: (counts[k, False], counts[k, True]) for k in OTHER_KINDS})


@pytest.mark.parametrize('kind', OTHER_KINDS)
def test_a_uniform_learner_writes_no_priorities_and_refuses_a_prioritized_learn(kind):
  agent, rep = _agent(kind, False, graph=False)
  _fill(rep, False)
  L = agent.learner
  L.priorities.fill_(-7.0)
  L.max_seen_priority.fill_(3.25)
  for _ in range(2):
    agent.learn()
  torch.cuda.synchronize()
  assert (L.priorities == -7.0).all() and float(L.max_seen_priority.item()) == 3.25
  # a prioritized learn on a learner that writes no priorities would write stale priorities into a tree: refused
  per_rep = _agent(kind, True, graph=False)[1]
  _fill(per_rep, False)
  before = _tree(per_rep).copy()
  with pytest.raises(ValueError, match='writes priorities'):
    L.learn(per_rep.device_view(), True, agent._io)
  torch.cuda.synchronize()
  assert np.array_equal(_tree(per_rep), before)
  assert (L.priorities == -7.0).all()


def test_the_config_field_is_validated():
  import ctypes as C
  from dqn_zoo_b200 import _lib
  cfg = _lib.LearnerConfig.from_buffer_copy(_learner('c51').cfg)
  cfg.prioritized = 2
  with pytest.raises(ValueError, match='prioritized'):
    _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(_lib.LearnerPlan()))
  cfg.prioritized = 1
  _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(_lib.LearnerPlan()))


# ---- 6. agents ---------------------------------------------------------------------------------------------------------

class _Env:
  """Deterministic dummy environment: random uint8 frames, episodes of 9..17 steps."""

  def __init__(self, seed):
    self.rs = np.random.RandomState(seed)
    self.left = 0

  def _obs(self):
    return self.rs.randint(0, 256, (84, 84, 4)).astype(np.uint8)

  def reset(self):
    from dqn_zoo_b200 import parts
    self.left = int(self.rs.randint(9, 18))
    return parts.TimeStep(parts.StepType.FIRST, None, None, self._obs())

  def step(self, action):
    from dqn_zoo_b200 import parts
    self.left -= 1
    last = self.left <= 0
    return parts.TimeStep(parts.StepType.LAST if last else parts.StepType.MID, float(self.rs.randint(-1, 2)),
                          0.0 if last else 0.99, self._obs())


def _run(agent, frames, seed=3):
  from dqn_zoo_b200 import parts
  n = 0
  for _ in parts.run_loop(agent, _Env(seed), max_steps_per_episode=15):
    n += 1
    if n >= frames:
      break
  torch.cuda.synchronize()


def _continue(agent, steps, seed=77):
  from dqn_zoo_b200 import parts
  rs = np.random.RandomState(seed)
  acts = []
  for _ in range(steps):
    ts = parts.TimeStep(parts.StepType.MID, float(rs.randint(-1, 2)), 0.99, rs.randint(0, 256, (84, 84, 4)).astype(np.uint8))
    acts.append(agent.step(ts))
  torch.cuda.synchronize()
  return acts


def _continuation(agent, run_state):
  """The next 24 steps of `agent` from the run state outside the agent's state (last action, accumulator, the replay's
  RandomState): actions, then the learner's blobs and the sum tree."""
  action, acc, rs_state = run_state
  agent._action = action
  agent._transition_accumulator = copy.deepcopy(acc)
  agent._replay._random_state.set_state(rs_state)
  acts = _continue(agent, 24)
  L = agent.learner
  return acts, [getattr(L, n).clone() for n in ('online', 'target', 'opt_state', 'counters', 'max_seen_priority')], \
      _tree(agent._replay).copy()


@pytest.mark.parametrize('kind', OTHER_KINDS)
def test_agents_run_loop_state_and_checkpoint_on_per(kind, tmp_path):
  a, _ = _agent(kind, True, capacity=96, min_fill=40, preprocessor=lambda ts: ts, seed=1)
  _run(a, 200)
  assert a._learn_steps > 10 and a._replay.size == 96
  ok, msg = a._replay.check_valid()
  assert ok, msg
  a.check_device_flags()
  st = copy.deepcopy(a.get_state())
  assert st['max_seen_priority'] == a.max_seen_priority > 0
  a.save_checkpoint(str(tmp_path / 'ckpt'))
  run_state = (a._action, copy.deepcopy(a._transition_accumulator), a._replay._random_state.get_state())
  b, _ = _agent(kind, True, capacity=96, min_fill=40, preprocessor=lambda ts: ts, seed=2)
  b.set_state(st)
  c, _ = _agent(kind, True, capacity=96, min_fill=40, preprocessor=lambda ts: ts, seed=2)
  c.load_checkpoint(str(tmp_path / 'ckpt'))
  want = _continuation(a, run_state)
  for restored in (b, c):
    got = _continuation(restored, run_state)
    assert got[0] == want[0]
    for x, y in zip(got[1], want[1]):
      assert torch.equal(x, y)
    assert np.array_equal(got[2], want[2])


def test_mismatched_checkpoints_raise_naming_prioritized(tmp_path):
  per, _ = _agent('qrdqn', True, capacity=600)
  uni, _ = _agent('qrdqn', False, capacity=600)
  per.save_checkpoint(str(tmp_path / 'per'))
  uni.save_checkpoint(str(tmp_path / 'uni'))
  with pytest.raises(ValueError, match='prioritized'):
    uni.load_checkpoint(str(tmp_path / 'per'))
  with pytest.raises(ValueError, match='prioritized'):
    per.load_checkpoint(str(tmp_path / 'uni'))
  # checkpoints written before the key existed: the kind's old default (prioritized only for prioritized and rainbow)
  for kind, want in (('qrdqn', False), ('rainbow', True)):
    agent, _ = _agent(kind, want, capacity=600)
    path = str(tmp_path / ('old-' + kind))
    agent.save_checkpoint(path)
    with open(os.path.join(path, 'agent.pkl'), 'rb') as f:
      state = pickle.load(f)
    assert state['prioritized'] is want
    del state['prioritized']
    with open(os.path.join(path, 'agent.pkl'), 'wb') as f:
      pickle.dump(state, f)
    agent.load_checkpoint(path)
  with pytest.raises(ValueError, match='prioritized'):
    per.load_checkpoint(str(tmp_path / 'old-qrdqn'))


@pytest.mark.parametrize('kind', ['c51', 'qrdqn', 'munchausen'])
def test_vector_trainer_tick_is_the_hand_composition(kind):
  E = 48
  script = tvt._script(E, tvt._ticks(E), seed=3)
  frames = tvt._frames(E, 2)
  a, _ = _agent(kind, True, min_fill=tvt._min_fill(E), seed=5)
  b, _ = _agent(kind, True, min_fill=tvt._min_fill(E), seed=5)
  tr = tvt._trainer(a, E)
  got = tvt._drive(tr, frames, script, 0, len(script))
  want = tvt._Hand(b, E).drive(frames, script)
  assert tr.learn_steps > 0
  np.testing.assert_array_equal(np.stack(got), np.stack(want))
  tvt._assert_same(a._replay.get_state(), b._replay.get_state())
  tvt._assert_same_learner(a, b)
  assert torch.equal(a.learner.max_seen_priority, b.learner.max_seen_priority)


# ---- 7. learning ---------------------------------------------------------------------------------------------------------
LEARNING_FRAMES = 1_500_000
LEARNING_THRESHOLD = 9.8          # the bar of the other Catch learning tests at this budget


def _learning_run(kind, n_step):
  import importlib
  import sys
  here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools')
  if here not in sys.path:
    sys.path.insert(0, here)
  bench_env = importlib.import_module('bench_env')
  return bench_env.learning_run(LEARNING_FRAMES, seed=0, kind=kind, prioritized=True, n_step=n_step)


@pytest.mark.parametrize('kind,n_step', [('qrdqn', 3), ('c51', 1)])
def test_learns_catch_on_per(kind, n_step):
  """bench_env's Catch schedule on rainbow's prioritized replay: 32 streams for LEARNING_FRAMES frames, then >= 50
  evaluation episodes at epsilon 0.01, held to the bar of the uniform agents' Catch learning tests."""
  curve = _learning_run(kind, n_step)
  frames, ret, episodes, _ = curve[-1]
  print('%s on PER (n=%d) catch curve' % (kind, n_step), curve)
  assert frames >= LEARNING_FRAMES and episodes >= 50
  assert ret >= LEARNING_THRESHOLD, curve
