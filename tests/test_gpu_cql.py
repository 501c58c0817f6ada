"""GPU: conservative Q-learning, CQL(H), in every agent kind's loss (DESIGN.md §20), and offline training.

- one update per kind and network option at cql_alpha 1 against the float64 oracles plus oracle/cql_oracle.py: loss,
  every gradient tensor and `.regularizer`, with non-unit importance weights including 0, on the tensor-core and
  fp32-FMA paths, ReLU kink flips counted as learner_parity does;
- the loss kernels on their own (dz_test_loss) at alpha > 0, with argmax ties and saturated softmaxes: the change of
  dout / dadv / dval and loss_terms from alpha 0 against the oracle's CQL term in float64, per_example and priorities
  unchanged bit for bit;
- what alpha leaves alone: per_example and priorities of a learner update bit-identical to alpha 0; alpha 0 is the
  parent (bit-identical to a learner built without the field); launches per fused step equal at every alpha;
- composition: a fused PER step against replay_oracle, graph and eager, both layouts; a pad-4 random-shift update
  against the pad-0 update on the oracle's shifted batch;
- OfflineTrainer: n steps are n hand `learn()` calls with target syncs at the cadence, graph equal to eager; acting
  state, frame_t and replay contents untouched; state and checkpoint round trips; an empty replay refused; the
  'cql_alpha' checkpoint key;
- learning: on a 3-action random Catch dataset a 6-action CQL agent keeps its greedy actions inside the data's actions
  and learns offline.
"""

import copy
import os
import pickle
import sys

import numpy as np
import pytest
import torch

import learner_parity as lp
import test_gpu_dueling as tdu
import test_gpu_fqf as tfq
import test_gpu_loss_kernels as tlk
import test_gpu_munchausen as tmu
import test_gpu_munchausen_iqn as tmi
import test_gpu_noisy as tno
import test_gpu_prioritized as tpr
from oracle import augment_oracle as ao
from oracle import cql_oracle as co
from oracle import learner_oracle as lo
from oracle import prioritized_oracle as po

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if os.path.join(ROOT, 'tools') not in sys.path:
  sys.path.insert(0, os.path.join(ROOT, 'tools'))

KINDS = co.KINDS
ALPHA = 1.0


def _twin(L, alpha, prioritized=None, pad=None):
  """A learner with L's configuration, parameters, optimizer state and counters, at cql_alpha `alpha`."""
  from dqn_zoo_b200 import learner as dl
  c = L.cfg
  T = dl.Learner(L.net, batch_size=L.batch_size, optimizer=L.opt, grad_error_bound=c.grad_error_bound,
                 huber_param=c.huber_param, munchausen_alpha=c.munchausen_alpha, entropy_temperature=c.entropy_temperature,
                 log_policy_clip=c.log_policy_clip, fraction_learning_rate=c.fraction_learning_rate,
                 fraction_opt_eps=c.fraction_opt_eps, fraction_rms_decay=c.fraction_rms_decay,
                 random_shift_pad=L.random_shift_pad if pad is None else pad,
                 prioritized=bool(c.prioritized) if prioritized is None else prioritized, cql_alpha=alpha)
  for name in ('online', 'target', 'opt_state', 'counters'):
    getattr(T, name).copy_(getattr(L, name))
  return T


# ---- 1. parity ---------------------------------------------------------------------------------------------------------

def _case(kind, net, hw, B):
  """(L at ALPHA, device update, oracle grads(tap) with the CQL term, ReLU table, weights)."""
  wrs = np.random.RandomState(200 + B)
  w = tpr._weights(B, wrs)
  if net.get('noisy'):
    dueling = bool(net.get('dueling'))
    spec, nspec, L, O, rs = tno.make_case(kind, dueling, B, hw, 3)
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, nspec, B, rs)
    noise_o, noise_flat = tno._noise(spec, nspec, dueling, rs)
    L = _twin(L, ALPHA)
    return (L, lambda: L.update(*arrs, weights=w, noise=noise_flat, apply_update=False),
            lambda tap: co.grads(O, batch, ALPHA, O.grads(batch, torch.tensor(w), noise=noise_o, tap=tap), torch.tensor(w),
                                 noise=noise_o, tap=tap), tno._table(dueling))
  if net.get('dueling'):
    spec, nspec, L, O, rs = tdu.make_case(kind, B, hw, 3)
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, nspec, B, rs)
    L = _twin(L, ALPHA)
    return (L, lambda: L.update(*arrs, weights=w, apply_update=False),
            lambda tap: co.grads(O, batch, ALPHA, O.grads(batch, torch.tensor(w), tap=tap), torch.tensor(w), tap=tap),
            'rainbow')
  if kind == 'munchausen':
    spec, nspec, L, O, rs = tmu.make_case(B, hw, 3)
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, nspec, B, rs)
    L = _twin(L, ALPHA)
    return (L, lambda: L.update(*arrs, weights=w, apply_update=False),
            lambda tap: co.grads(O, batch, ALPHA, O.grads(batch, torch.tensor(w), tap=tap), torch.tensor(w), tap=tap), 'dqn')
  if kind == 'munchausen_iqn':
    full = lp._hw(hw) == (84, 84)
    spec, nspec, L, O, rs = tmi.make_case(B, hw, 3, taus=(64, 64, 64) if full else (8, 5, 7))
    arrs, batch, taus_o, taus_flat = tmi.make_batch(nspec, B, rs)
    L = _twin(L, ALPHA)
    return (L, lambda: L.update(*arrs, weights=w, taus=taus_flat, apply_update=False),
            lambda tap: co.grads(O, batch, ALPHA, O.grads(batch, torch.tensor(w), taus=taus_o, tap=tap), torch.tensor(w),
                                 taus=taus_o, tap=tap), 'iqn')
  if kind == 'fqf':
    spec, nspec, L, O, rs = tfq.make_case(B, hw, 3)
    arrs, batch = tfq.make_batch(nspec, B, rs)
    L = _twin(L, ALPHA)

    def oracle(tap):
      fr = tfq.device_fractions(L)
      return co.grads(O, batch, ALPHA, O.grads(batch, torch.tensor(w), device_fractions=fr, tap=tap), torch.tensor(w),
                      device_fractions=fr, tap=tap)
    return L, lambda: L.update(*arrs, weights=w, apply_update=False), oracle, 'iqn'
  spec, nspec, L, O, rs = lp.make_case(kind, B, hw, seed=3)
  arrs, batch, _, taus_o, taus_flat, noise_o, noise_flat = lp.make_batch(spec, nspec, B, rs)
  L = _twin(L, ALPHA)
  return (L, lambda: L.update(*arrs, weights=w, taus=taus_flat, noise=noise_flat, apply_update=False),
          lambda tap: co.grads(O, batch, ALPHA, O.grads(batch, torch.tensor(w), taus_o, noise_o, tap=tap), torch.tensor(w),
                               taus=taus_o, noise=noise_o, tap=tap), kind)


PARITY = ([(k, {}) for k in KINDS] +
          [(k, n) for k in ('dqn', 'double_q') for n in ({'dueling': True}, {'noisy': True}, {'dueling': True, 'noisy': True})])
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
    print('relu kink flips %s %s B=%d: %s' % (kind, lp._hw(hw), B, {k: v[:2] for k, v in flips.items()}))
    loss, aux, grads = oracle_grads(lo.ReluTap(masks))
  R = aux['regularizer'].numpy()
  assert (R >= 0).all()
  assert lp.rel_err(L.regularizer.cpu().numpy(), R) <= lp.REL
  want_pe = aux['td_errors'] if kind in ('dqn', 'double_q', 'prioritized') else aux['losses']
  assert lp.rel_err(L.per_example.cpu().numpy(), want_pe.numpy()) <= lp.REL
  gn = tfq.main_norm(grads) if kind == 'fqf' else float(torch.sqrt(sum((g * g).sum() for g in grads.values())))
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
  return L


@pytest.mark.parametrize('hw,B', [(84, 32), (44, 5)], ids=['84x84-B32', '44x44-B5'])
@pytest.mark.parametrize('kind,net', PARITY, ids=PARITY_IDS)
def test_cql_update_matches_the_oracle(kind, net, hw, B):
  _check_parity(kind, net, hw, B)


@pytest.mark.parametrize('kind', KINDS)
def test_cql_update_on_the_fp32_fma_torso(kind):
  L = _check_parity(kind, {}, (84, 88), 32)
  assert not lp.tensor_core_torso(L)


# ---- 2. the loss kernels on their own ----------------------------------------------------------------------------------

def _with_alpha(case, alpha):
  config = tlk.Case.config.__get__(case)

  def cfg():
    c = config()
    c.cql_alpha = alpha
    return c
  case.config = cfg
  return case


def _kernel_cases(kind, rs):
  A = 6
  wide = 18 if kind.startswith('munchausen') else 64    # munchausen's kernels hold one action per lane
  out = [tlk.random_case(kind, 32, A, rs), tlk.random_case(kind, 5, 18, rs, scale=30.0, name='saturated'),
         tlk.random_case(kind, 3, 1, rs, name='one action'), tlk.random_case(kind, 4, wide, rs, name='wide')]
  tie = tlk.random_case(kind, 8, A, rs, name='ties')   # actions 1 and 3 of pass 0 equal: tied Q, a_tm1 on the tie
  h0 = tie.heads[0][0] if kind == 'rainbow' else tie.heads[0]
  if kind in ('qrdqn', 'iqn', 'munchausen_iqn'):
    h0[:, :, 3] = h0[:, :, 1]
  else:
    h0[:, 3] = h0[:, 1]
  tie.a[:] = 1
  out.append(tie)
  for c in out:
    if c.w is None:
      c.w = tlk.f32(rs.uniform(0.0, 1.0, c.B))
      c.w[0] = 0.0
  return out


def _cql_head_grad(case, alpha):
  rb = case.kind == 'rainbow'
  h = case.heads[0]
  head = (tlk.t64(h[0]), tlk.t64(h[1])) if rb else tlk.t64(h)
  R, g = co.head_grad(case.kind, head, torch.tensor(case.a.astype(np.int64)), alpha, tlk.t64(case.w), vmax=case.vmax)
  return R.numpy(), (tuple(x.numpy() for x in g) if rb else g.numpy())


@pytest.mark.parametrize('kind', [k for k in KINDS if k != 'fqf'])
def test_loss_kernels_add_the_cql_term(kind):
  rs = np.random.RandomState(5)
  for case in _kernel_cases(kind, rs):
    alpha = 0.75
    base = tlk.run_device(case)
    got = tlk.run_device(_with_alpha(copy.copy(case), alpha))
    # what alpha leaves alone, bit for bit
    assert np.array_equal(got['per_example'], base['per_example']), case.name
    if case.kind in ('prioritized', 'rainbow'):
      assert np.array_equal(got['priorities'], base['priorities']), case.name
    R, g = _cql_head_grad(case, alpha)
    w = case.w.astype(np.float64)
    # loss_terms = w (loss + alpha R): the change is w alpha R, up to the rounding of the sum
    scale = np.abs(base['loss_terms']) + w * alpha * R + 1e-30
    assert np.all(np.abs((got['loss_terms'] - base['loss_terms']) - w * alpha * R) <= 8 * tlk.U * scale + 1e-12), case.name
    pairs = [('dout', g[0] if case.kind == 'rainbow' else g)] + ([('dval', g[1])] if case.kind == 'rainbow' else [])
    for name, want in pairs:
      diff = got[name] - base[name]
      tol = 2e-5 * np.abs(want).max() + 8 * tlk.U * np.abs(base[name]).max() + 1e-12
      assert np.abs(diff - want).max() <= tol, (case.name, name, np.abs(diff - want).max(), tol)
      assert np.all(got[name][w == 0] == base[name][w == 0]), (case.name, name)


# ---- 3. what alpha leaves alone -----------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind', KINDS)
def test_alpha_leaves_per_example_and_priorities_and_zero_is_the_parent(kind):
  from dqn_zoo_b200 import learner as dl
  plain = tpr._learner(kind, prioritized=True)
  plain.init_params(4)
  zero = _twin(plain, 0.0)
  cql = _twin(plain, 2.0)
  assert plain.cql_alpha == 0.0 and plain.cfg.cql_alpha == 0.0
  rs = np.random.RandomState(9)
  for step in range(3):
    kw = tpr._inputs(plain, rs)
    w = rs.uniform(0.0, 1.0, plain.batch_size)
    plain.update(weights=w, **kw)
    zero.update(weights=w, **kw)
    torch.cuda.synchronize()
    for name in ('loss', 'per_example', 'priorities', 'grad_norm', 'grads', 'online', 'opt_state'):
      assert torch.equal(getattr(plain, name), getattr(zero, name)), (step, name)
    # the alpha > 0 twin on the same parameters and batch
    for name in ('online', 'target', 'opt_state', 'counters'):
      getattr(cql, name).copy_(getattr(plain, name))
    cql.update(weights=w, apply_update=False, **kw)
    ref = _twin(plain, 0.0)
    ref.update(weights=w, apply_update=False, **kw)
    torch.cuda.synchronize()
    assert torch.equal(cql.per_example, ref.per_example) and torch.equal(cql.priorities, ref.priorities), step
    assert (cql.regularizer >= 0).all() and float(cql.loss) > float(ref.loss)
  assert dl.Learner(plain.net, cql_alpha=0).cql_alpha == 0.0


def _agent(kind, alpha, prioritized=False, graph=True, dedup=False, seed=3, capacity=512):
  """bench_offline's agent of `kind` at `alpha` on a fresh replay (prioritized for prioritized and rainbow, which learn
  from nothing else), learn period 4, target period 16."""
  import bench_offline
  from dqn_zoo_b200 import replay as dr
  structure = dr.Transition(None, None, None, None, None)
  extra = dict(frame_dedup=True, frame_capacity=8 * (capacity + 1) + 1) if dedup else {}
  rs = np.random.RandomState(seed)
  if prioritized or kind in ('prioritized', 'rainbow'):
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.5, lambda t: 0.4, 1e-3, True, rs, **extra)
  else:
    rep = dr.TransitionReplay(capacity, structure, rs, **extra)
  return bench_offline.make_agent(kind, rep, alpha, seed=seed, graph=graph, learn_period=4, target_period=16), rep


def test_launches_per_step_do_not_depend_on_alpha():
  counts = {}
  for kind in KINDS:
    for alpha in (0.0, 1.0):
      agent, rep = _agent(kind, alpha, graph=False)
      tpr._fill(rep, False)
      counts[kind, alpha] = tpr._launches_per_step(agent)
    assert counts[kind, 0.0] == counts[kind, 1.0], (kind, counts)
  print('launches per step:', {k: counts[k, 0.0] for k in KINDS})


# ---- 4. composition ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,dedup', [('c51', False), ('qrdqn', True), ('dqn', False), ('fqf', True)],
                         ids=['c51-dense', 'qrdqn-dedup', 'dqn-dense', 'fqf-dedup'])
def test_fused_per_step_matches_the_replay_oracle_and_graph_is_eager(kind, dedup):
  cap, seed = 512, 3
  graphed, rep_g = _agent(kind, ALPHA, prioritized=True, graph=True, dedup=dedup, seed=seed)
  eager, rep_e = _agent(kind, ALPHA, prioritized=True, graph=False, dedup=dedup, seed=seed)
  tpr._fill(rep_g, dedup)
  tpr._fill(rep_e, dedup)
  orep = tpr._oracle_replay(cap, seed)
  L = graphed.learner
  for step in range(6):
    graphed.learn()
    eager.learn()
    torch.cuda.synchronize()
    ids, _, w = orep.sample_ids(32)
    assert np.array_equal(L.sampled_ids.cpu().numpy(), ids), step
    pri = L.priorities.cpu().numpy()
    if kind in po.LOSS_KINDS:
      assert np.array_equal(pri, np.clip(np.abs(L.per_example.cpu().numpy()), 0, 100))
    orep.update_priorities(ids, pri)
    assert np.array_equal(tpr._tree(rep_g), tpr._tree(orep)), step
    for name in ('online', 'opt_state', 'priorities', 'loss', 'regularizer', 'max_seen_priority'):
      assert torch.equal(getattr(L, name), getattr(eager.learner, name)), (step, name)
  assert (L.regularizer > 0).any()
  graphed.check_device_flags()


@pytest.mark.parametrize('kind', ['dqn', 'c51', 'iqn', 'fqf'])
def test_a_shifted_cql_update_is_the_update_on_the_oracles_shift(kind):
  from dqn_zoo_b200 import learner as dl
  p = 4
  off = dl.Learner(dl.NetworkSpec(kind, 6), cql_alpha=ALPHA)
  off.init_params(1)
  on = _twin(off, ALPHA, pad=p)
  rs = np.random.RandomState(11)
  for step in range(3):
    s_tm1, s_t, kw = tpr_inputs(on, rs)
    S = rs.randint(0, 2 * p + 1, size=(on.batch_size, 4))
    on.update(s_tm1=s_tm1, s_t=s_t, shifts=S, **kw)
    x_tm1, x_t = ao.shift_batch(s_tm1, s_t, S, p)
    off.update(s_tm1=x_tm1, s_t=x_t, **kw)
    torch.cuda.synchronize()
    for name in ('loss', 'per_example', 'regularizer', 'grads', 'online', 'opt_state'):
      assert torch.equal(getattr(on, name), getattr(off, name)), (step, name)


def tpr_inputs(L, rs):
  kw = tpr._inputs(L, rs)
  return kw.pop('s_tm1'), kw.pop('s_t'), kw


# ---- 5. OfflineTrainer ------------------------------------------------------------------------------------------------

def _blobs(agent):
  L = agent.learner
  return [getattr(L, n).clone() for n in ('online', 'target', 'opt_state', 'counters', 'loss', 'regularizer')]


@pytest.mark.parametrize('kind,prioritized', [('dqn', False), ('qrdqn', True), ('iqn', False), ('rainbow', True)])
def test_offline_steps_are_hand_learn_calls_with_target_syncs(kind, prioritized):
  from dqn_zoo_b200 import agent as ag
  a, rep_a = _agent(kind, ALPHA, prioritized=prioritized, graph=True)
  b, rep_b = _agent(kind, ALPHA, prioritized=prioritized, graph=False)
  tpr._fill(rep_a, False)
  tpr._fill(rep_b, False)
  a._frame_t = b._frame_t = 123
  host = a._host_rng.get_state()
  rows = list(range(0, rep_a.size, 8))
  before, tree = rep_a.get(rows), (tpr._tree(rep_a).copy() if prioritized else None)
  tr = ag.OfflineTrainer(a)
  assert tr.target_update_period == 4     # 16 // 4
  tr.step(3)
  tr.step(7)
  for u in range(1, 11):
    b.learn()
    if u % 4 == 0:
      b.learner.sync_target()
  torch.cuda.synchronize()
  assert tr.updates == 10
  for x, y in zip(_blobs(a), _blobs(b)):
    assert torch.equal(x, y)
  assert a._frame_t == 123 and a._action is None
  np.testing.assert_equal(a._host_rng.get_state(), host)
  for x, y in zip(rep_a.get(rows), before):
    for f, g in zip(x, y):
      np.testing.assert_array_equal(f, g)
  if prioritized:   # priorities are written back offline
    assert not np.array_equal(tpr._tree(rep_a), tree)


def test_offline_state_and_checkpoint_round_trips(tmp_path):
  from dqn_zoo_b200 import agent as ag
  a, rep = _agent('c51', ALPHA, prioritized=True)
  tpr._fill(rep, False)
  tr = ag.OfflineTrainer(a, target_update_period=3)
  tr.step(5)
  st = copy.deepcopy(tr.get_state())
  tr.save_checkpoint(str(tmp_path / 'off'))
  tr.step(7)
  torch.cuda.synchronize()
  want = _blobs(a) + [torch.tensor(tpr._tree(rep))]
  for restore in ('state', 'checkpoint'):
    b, rep_b = _agent('c51', ALPHA, prioritized=True, seed=9)
    tpr._fill(rep_b, False)
    tb = ag.OfflineTrainer(b, target_update_period=3)
    if restore == 'state':
      tb.set_state(st)
    else:
      tb.load_checkpoint(str(tmp_path / 'off'))
    assert tb.updates == 5
    tb.step(7)
    torch.cuda.synchronize()
    got = _blobs(b) + [torch.tensor(tpr._tree(rep_b))]
    for x, y in zip(got, want):
      assert torch.equal(x, y), restore
  other = ag.OfflineTrainer(_agent('c51', ALPHA, prioritized=True)[0], target_update_period=5)
  with pytest.raises(ValueError, match='target_update_period'):
    other.load_checkpoint(str(tmp_path / 'off'))


def test_offline_refuses_an_empty_replay_and_bad_periods():
  from dqn_zoo_b200 import agent as ag
  a, _ = _agent('dqn', ALPHA)
  with pytest.raises(ValueError, match='empty'):
    ag.OfflineTrainer(a).step(1)
  for bad in (0, -1, 2.5):
    with pytest.raises(ValueError):
      ag.OfflineTrainer(a, target_update_period=bad)
  with pytest.raises(TypeError):
    ag.OfflineTrainer(object())


def test_the_cql_alpha_checkpoint_key(tmp_path):
  cql, rep = _agent('qrdqn', ALPHA, capacity=600)
  plain, _ = _agent('qrdqn', 0.0, capacity=600)
  cql.save_checkpoint(str(tmp_path / 'cql'))
  plain.save_checkpoint(str(tmp_path / 'plain'))
  with pytest.raises(ValueError, match='cql_alpha'):
    plain.load_checkpoint(str(tmp_path / 'cql'))
  with pytest.raises(ValueError, match='cql_alpha'):
    cql.load_checkpoint(str(tmp_path / 'plain'))
  path = str(tmp_path / 'plain')
  with open(os.path.join(path, 'agent.pkl'), 'rb') as f:
    state = pickle.load(f)
  assert state['cql_alpha'] == 0.0
  del state['cql_alpha']            # a checkpoint written before the key existed
  with open(os.path.join(path, 'agent.pkl'), 'wb') as f:
    pickle.dump(state, f)
  plain.load_checkpoint(path)
  with pytest.raises(ValueError, match='cql_alpha'):
    cql.load_checkpoint(path)


# ---- 6. learning -------------------------------------------------------------------------------------------------------
OFFLINE_UPDATES = 30000
DATASET = 1 << 17
# CQL qrdqn's evaluation return at OFFLINE_UPDATES in the measured run of tools/bench_offline.py (DESIGN.md §20, same
# dataset, seeds and schedule); a run must reach more than half of it.
MEASURED_RETURN = 18.906


@pytest.fixture(scope='module')
def catch_dataset():
  import bench_offline
  rep, behaviour = bench_offline.record_dataset(DATASET)
  rep = bench_offline.load_dataset(rep)
  return rep, behaviour, bench_offline.dataset_states(rep)


def test_cql_is_conservative_and_learns_catch_offline(catch_dataset):
  """qrdqn with a 6-action network trained offline on 2^17 transitions of 3-action random Catch: at alpha 1 the greedy
  action stays inside the data's actions on >= 99 % of 4096 dataset states, the out-of-data gap is negative, and the
  evaluation return beats the behaviour policy clearly and reaches half of the measured run.  alpha 0's numbers are
  printed beside it, not asserted."""
  import bench_offline
  rep, behaviour, states = catch_dataset
  assert rep.size == DATASET and behaviour < -1.5
  curves = {}
  for alpha in (0.0, 1.0):
    curves[alpha] = bench_offline.offline_run(rep, 'qrdqn', alpha, OFFLINE_UPDATES, OFFLINE_UPDATES // 3, states=states)
    print('offline qrdqn alpha=%g (updates, return, episodes, out-of-data greedy share, gap):' % alpha, curves[alpha])
  _, ret, n, share, gap = curves[1.0][-1]
  assert n >= 50
  assert share <= 0.01, curves[1.0]
  assert gap < 0.0, curves[1.0]
  assert ret > behaviour + 4.0, (ret, behaviour)
  assert ret > 0.5 * MEASURED_RETURN, (ret, MEASURED_RETURN)
