"""GPU: random-shift augmentation of the learner step (DrQ; DESIGN.md §18).  The shift kernel bit for bit against
oracle/augment_oracle.py; the shift draws against the Philox restatement and their statistics; a pad-p update on a batch
X with shifts S against a pad-0 update on the oracle's shift of X, bit for bit, for every kind and network option on the
tensor-core and fp32-FMA paths; the fused `_learn()` against sample -> oracle shift -> update, eager and in a CUDA graph,
on uniform, prioritized and frame-deduplicated replays; the launches it adds; acting, which never sees a shift; trainer
and checkpoint round trips; and a dueling double_q with random shifts learning Catch."""

import copy
import ctypes as C
import os
import pickle

import numpy as np
import pytest
import scipy.stats
import torch

from oracle import augment_oracle as ao
from oracle import replay_oracle as ro

pytestmark = pytest.mark.gpu

LAST = 2


def _stream():
  return torch.cuda.current_stream().cuda_stream


# ---- the shift kernel --------------------------------------------------------------------------------------------------

def _run_kernel(s_tm1, s_t, shifts, pad, stride_extra=32, guard=256):
  """dz_test_random_shift over dense [B, H, W, C] uint8 batches into a 0xFF-filled buffer with a guard band on both
  sides.  Returns (rows [B, 2, stride] as numpy, the two guard bands)."""
  from dqn_zoo_b200 import _lib
  B, H, W, Cc = s_tm1.shape
  obs = H * W * Cc
  stride = obs + stride_extra
  src = [torch.as_tensor(x, device='cuda').reshape(B, obs).contiguous() for x in (s_tm1, s_t)]
  tables = [x.data_ptr() + torch.arange(B, dtype=torch.int64, device='cuda') * obs for x in src]
  sh = torch.as_tensor(shifts, dtype=torch.int32, device='cuda').contiguous()
  buf = torch.full((guard + B * 2 * stride + guard,), 0xFF, dtype=torch.uint8, device='cuda')
  _lib.call('dz_test_random_shift', tables[0].data_ptr(), tables[1].data_ptr(), sh.data_ptr(), B, H, W, Cc, pad,
            buf.data_ptr() + guard, stride, _stream())
  host = buf.cpu().numpy()
  return host[guard:guard + B * 2 * stride].reshape(B, 2, stride), host[:guard], host[guard + B * 2 * stride:]


def _extreme_shifts(B, p, rs):
  """Random shifts in [0, 2p] whose first examples take every extreme pair of (dy, dx) on both observations."""
  s = rs.randint(0, 2 * p + 1, size=(B, 4)).astype(np.int32)
  ext = [(a, b) for a in (0, p, 2 * p) for b in (0, p, 2 * p)]
  for b in range(min(B, len(ext))):
    s[b, 0:2] = ext[b]
    s[b, 2:4] = ext[-1 - b]
  return s


@pytest.mark.parametrize('hw', [(84, 84), (44, 44), (84, 92), (84, 88)], ids=lambda v: '%dx%d' % v)
@pytest.mark.parametrize('B', [1, 32, 33, 128])
@pytest.mark.parametrize('p', [1, 4, 16])
def test_kernel_is_the_oracle_bit_for_bit(hw, B, p):
  H, W = hw
  rs = np.random.RandomState(B * 131 + p * 7 + H + W)
  s_tm1 = rs.randint(0, 256, size=(B, H, W, 4)).astype(np.uint8)
  s_t = rs.randint(0, 256, size=(B, H, W, 4)).astype(np.uint8)
  shifts = _extreme_shifts(B, p, rs)
  out, lo, hi = _run_kernel(s_tm1, s_t, shifts, p)
  obs = H * W * 4
  want_tm1, want_t = ao.shift_batch(s_tm1, s_t, shifts, p)
  assert np.array_equal(out[:, 0, :obs].reshape(B, H, W, 4), want_tm1)
  assert np.array_equal(out[:, 1, :obs].reshape(B, H, W, 4), want_t)
  assert not out[:, :, obs:].any(), 'the stride padding must be zero'
  assert (lo == 0xFF).all() and (hi == 0xFF).all(), 'the kernel wrote outside its rows'


def test_kernel_with_eight_channels_and_a_band_loop():
  """C = 8 (two 32-bit words per pixel) and rows wide enough that a band holds fewer rows than the observation."""
  rs = np.random.RandomState(3)
  B, H, W, Cc, p = 3, 70, 1024, 8, 16      # 8 KB rows: 4 rows per band
  s_tm1 = rs.randint(0, 256, size=(B, H, W, Cc)).astype(np.uint8)
  s_t = rs.randint(0, 256, size=(B, H, W, Cc)).astype(np.uint8)
  shifts = _extreme_shifts(B, p, rs)
  out, lo, hi = _run_kernel(s_tm1, s_t, shifts, p, stride_extra=0)
  want_tm1, want_t = ao.shift_batch(s_tm1, s_t, shifts, p)
  assert np.array_equal(out[:, 0].reshape(B, H, W, Cc), want_tm1)
  assert np.array_equal(out[:, 1].reshape(B, H, W, Cc), want_t)
  assert (lo == 0xFF).all() and (hi == 0xFF).all()


def test_kernel_rejects_bad_arguments():
  from dqn_zoo_b200 import _lib
  x = torch.zeros(84 * 84 * 4, dtype=torch.uint8, device='cuda')
  tab = torch.tensor([x.data_ptr()], dtype=torch.int64, device='cuda')
  sh = torch.zeros(4, dtype=torch.int32, device='cuda')
  out = torch.zeros(2 * 84 * 84 * 4 + 16, dtype=torch.uint8, device='cuda')
  ok = (tab.data_ptr(), tab.data_ptr(), sh.data_ptr(), 1, 84, 84, 4, 4, out.data_ptr(), 84 * 84 * 4, _stream())
  _lib.call('dz_test_random_shift', *ok)
  for i, bad in [(7, 17), (7, 84), (7, -1), (6, 2), (5, 83), (9, 84 * 84 * 4 - 16), (9, 84 * 84 * 4 + 8)]:
    args = list(ok)
    args[i] = bad
    with pytest.raises(ValueError):
      _lib.call('dz_test_random_shift', *args)
  with pytest.raises(ValueError):
    _lib.call('dz_test_random_shift', *(ok[:8] + (out.data_ptr() + 8,) + ok[9:]))


# ---- the draws ---------------------------------------------------------------------------------------------------------

def _learner(kind='dqn', pad=4, B=32, hw=(84, 84), **net):
  from dqn_zoo_b200 import learner as dl
  return dl.Learner(dl.NetworkSpec(kind, 6, obs_shape=(hw[0], hw[1], 4), **net), batch_size=B, random_shift_pad=pad)


@pytest.mark.parametrize('p', [1, 4, 16])
def test_draws_are_the_oracles_and_the_counter_steps_once(p):
  L = _learner(pad=p, B=33)
  for seed, ctr in [(0, 0), (7, 1), (2 ** 32 + 9, 2 ** 32 - 1), (2 ** 63 + 5, 2 ** 32 + 3), (12345, 2 ** 40)]:
    L.counters[1] = ctr
    L.generate_randomness(seed)
    torch.cuda.synchronize()
    assert np.array_equal(L.shifts.cpu().numpy(), ao.draws(33, seed, ctr, p)), (seed, ctr)
    assert int(L.counters[1].item()) == ctr + 1
  # beside the sampler: the same draws, the same counter step
  L.counters[1] = 77
  L.generate_randomness(5, beside_sampler=True)
  torch.cuda.synchronize()
  assert np.array_equal(L.shifts.cpu().numpy(), ao.draws(33, 5, 77, p))
  assert int(L.counters[1].item()) == 78


def test_generate_shifts_does_not_advance_the_counter():
  from dqn_zoo_b200 import _lib
  L = _learner()
  L.counters[1] = 41
  _lib.call('dz_learner_generate_shifts', L._h, 3, L.shifts.data_ptr(), _stream())
  torch.cuda.synchronize()
  assert int(L.counters[1].item()) == 41
  assert np.array_equal(L.shifts.cpu().numpy(), ao.draws(32, 3, 41, 4))
  off = _learner(pad=0)
  with pytest.raises(ValueError):
    _lib.call('dz_learner_generate_shifts', off._h, 3, off.shifts.data_ptr(), _stream())


@pytest.mark.parametrize('kind,net', [('iqn', {}), ('munchausen_iqn', {}), ('rainbow', {}), ('dqn', {'noisy': True})])
def test_taus_and_noise_do_not_depend_on_the_pad(kind, net):
  a, b = _learner(kind, pad=0, **net), _learner(kind, pad=4, **net)
  for L in (a, b):
    L.counters[1] = 2 ** 32 - 2
    for _ in range(3):
      L.generate_randomness(99)
  torch.cuda.synchronize()
  assert torch.equal(a.taus, b.taus) and torch.equal(a.noise, b.noise) and torch.equal(a.counters, b.counters)


def test_draws_are_uniform_over_the_cells_and_uncorrelated():
  p, B, calls = 4, 1024, 32
  L = _learner(pad=p, B=B)
  got = []
  for _ in range(calls):
    L.generate_randomness(2024)
    got.append(L.shifts.clone())
  s = torch.cat(got).cpu().numpy().astype(np.int64)            # [calls * B, 4]
  assert s.min() >= 0 and s.max() <= 2 * p
  n = 2 * p + 1
  cells = np.concatenate([s[:, 0] * n + s[:, 1], s[:, 2] * n + s[:, 3]])    # 2^16 (dy, dx) pairs
  counts = np.bincount(cells, minlength=n * n)
  chi2 = ((counts - cells.size / n ** 2) ** 2 / (cells.size / n ** 2)).sum()
  assert scipy.stats.chi2.sf(chi2, n * n - 1) > 1e-4, chi2
  bar = 5.0 / np.sqrt(s.shape[0])
  for i, j in [(0, 2), (1, 3), (0, 1), (2, 3), (0, 3), (1, 2)]:      # within an example, s_tm1 against s_t
    assert abs(np.corrcoef(s[:, i], s[:, j])[0, 1]) < bar, (i, j)
  for i in range(4):                                                # neighbouring examples
    assert abs(np.corrcoef(s[:-1, i], s[1:, i])[0, 1]) < bar, i


# ---- learner equivalence -----------------------------------------------------------------------------------------------

CASES = [('dqn', {}), ('double_q', {}), ('prioritized', {}), ('c51', {}), ('qrdqn', {}), ('rainbow', {}), ('iqn', {}),
         ('munchausen', {}), ('munchausen_iqn', {}), ('fqf', {}), ('dqn', {'dueling': True}), ('dqn', {'noisy': True}),
         ('dqn', {'dueling': True, 'noisy': True})]
CASE_IDS = ['%s%s' % (k, ''.join('-' + o for o in sorted(n))) for k, n in CASES]
OUTPUTS = ('loss', 'per_example', 'priorities', 'grad_norm', 'grads')


def _pair(kind, net, hw, pad, B=32):
  """A pad-0 and a pad-p learner with the same online, target and optimizer state."""
  a, b = _learner(kind, 0, B, hw, **net), _learner(kind, pad, B, hw, **net)
  a.init_params(2)
  target = a.get_params()
  a.init_params(1)
  a.set_params(target, blob='target')
  b.set_params(a.get_params())
  b.set_params(target, blob='target')
  return a, b


def _inputs(L, rs):
  from dqn_zoo_b200 import learner as dl
  B = L.batch_size
  H, W, Cc = L.net.obs_shape
  s_tm1 = rs.randint(0, 256, (B, H, W, Cc)).astype(np.uint8)
  s_t = rs.randint(0, 256, (B, H, W, Cc)).astype(np.uint8)
  kw = dict(a_tm1=rs.randint(0, L.net.num_actions, B), r_t=rs.choice([-1.0, 0.0, 1.0, 0.37], size=B),
            discount_t=rs.choice([0.0, 0.99], size=B))
  if L.kind in ('prioritized', 'rainbow'):
    kw['weights'] = rs.uniform(0.1, 1.0, B)
  if dl.draws_taus(L.kind):
    kw['taus'] = rs.uniform(size=L.plan.tau_floats).astype(np.float32)
  if dl.noisy_layers(L.net):
    kw['noise'] = rs.uniform(-1.4, 1.4, size=L.plan.noise_floats).astype(np.float32)
  return s_tm1, s_t, kw


@pytest.mark.parametrize('hw', [(84, 84), (84, 88)], ids=['tensor_core', 'fp32_fma'])
@pytest.mark.parametrize('kind,net', CASES, ids=CASE_IDS)
def test_a_shifted_update_is_the_update_on_the_oracles_shift(kind, net, hw):
  """Three steps with random shifts, then one with every shift at (p, p): the pad-4 learner on (X, S) and the pad-0
  learner on oracle.shift(X, S) give the same outputs, parameters and optimizer state, bit for bit."""
  p = 4
  off, on = _pair(kind, net, hw, p)
  rs = np.random.RandomState(11)
  for step in range(4):
    s_tm1, s_t, kw = _inputs(on, rs)
    S = rs.randint(0, 2 * p + 1, size=(on.batch_size, 4)) if step < 3 else np.full((on.batch_size, 4), p)
    on.update(s_tm1=s_tm1, s_t=s_t, shifts=S, **kw)
    x_tm1, x_t = ao.shift_batch(s_tm1, s_t, S, p)
    off.update(s_tm1=x_tm1, s_t=x_t, **kw)
    torch.cuda.synchronize()
    for name in OUTPUTS:
      assert torch.equal(getattr(on, name), getattr(off, name)), (step, name)
  for name in ('online', 'target', 'opt_state', 'counters'):
    assert torch.equal(getattr(on, name), getattr(off, name)), name


def test_update_needs_shifts_and_rejects_bad_pads():
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import learner as dl
  for bad in (-1, 17, 1.5, True):
    with pytest.raises(ValueError):
      dl.Learner(dl.NetworkSpec('dqn', 6), random_shift_pad=bad)
  with pytest.raises(ValueError):
    dl.Learner(dl.NetworkSpec('dqn', 6, obs_shape=(36, 36, 4)), random_shift_pad=36)
  cfg = _lib.LearnerConfig(kind=0, num_actions=6, batch=32, obs_h=84, obs_w=84, obs_c=4, optimizer=1,
                           learning_rate=1e-4, opt_eps=1e-4, rms_decay=0.95, random_shift_pad=17)
  with pytest.raises(ValueError):
    _lib.call('dz_learner_plan_query', C.byref(cfg), C.byref(_lib.LearnerPlan()))
  L = _learner()
  rs = np.random.RandomState(0)
  s_tm1, s_t, kw = _inputs(L, rs)
  dev = lambda x: torch.as_tensor(x, device='cuda')
  keep = [dev(s_tm1).reshape(32, -1), dev(s_t).reshape(32, -1), dev(kw['a_tm1']).to(torch.int32),
          dev(kw['r_t']).float(), dev(kw['discount_t']).float()]
  tabs = [L._row_table(keep[0]), L._row_table(keep[1])]
  batch = _lib.Batch(tabs[0].data_ptr(), tabs[1].data_ptr(), keep[2].data_ptr(), keep[3].data_ptr(), keep[4].data_ptr(),
                     0, 0, 0, 0)
  out = _lib.UpdateOutputs(L.loss.data_ptr(), L.per_example.data_ptr(), L.priorities.data_ptr(), L.grad_norm.data_ptr())
  with pytest.raises(ValueError, match='d_shifts'):
    _lib.call('dz_learner_update', L._h, C.byref(batch), C.byref(out), 1, _stream())
  with pytest.raises(ValueError):
    _learner(pad=0).update(s_tm1, kw['a_tm1'], kw['r_t'], kw['discount_t'], s_t, shifts=np.zeros((32, 4)))


# ---- the fused step ----------------------------------------------------------------------------------------------------

def _agent(kind, pad=4, capacity=512, seed=3, graph=True, min_fill=None, dueling=False, noisy=False, epsilon=0.1,
           frame_dedup=False):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  structure = dr.Transition(None, None, None, None, None)
  extra = dict(frame_dedup=True, frame_capacity=8 * (capacity + 1) + 1) if frame_dedup else {}
  if kind in ('prioritized', 'rainbow'):
    rep = dr.PrioritizedTransitionReplay(capacity, structure, 0.6, lambda t: 0.4, 1e-3, True, np.random.RandomState(seed),
                                         **extra)
  else:
    rep = dr.TransitionReplay(capacity, structure, np.random.RandomState(seed), **extra)
  common = dict(preprocessor=None, sample_network_input=None, optimizer=None,
                network=dl.NetworkSpec(kind, 6, dueling=dueling, noisy=noisy),
                transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=(min_fill or capacity) / capacity, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=graph, random_shift_pad=pad)
  if kind == 'rainbow':
    return ag.Rainbow(support=np.linspace(-10, 10, 51), **common), rep
  if dl.uses_iqn_network(kind):
    return ag.AGENTS[kind](exploration_epsilon=lambda t: epsilon, huber_param=1.0, tau_samples_policy=64,
                           tau_samples_s_tm1=64, tau_samples_s_t=64, **common), rep
  return ag.AGENTS[kind](exploration_epsilon=lambda t: epsilon, grad_error_bound=1.0 / 32, **common), rep


@pytest.mark.parametrize('graph', [False, True], ids=['eager', 'graph'])
@pytest.mark.parametrize('kind', ['dqn', 'prioritized', 'rainbow', 'iqn'])
def test_fused_learn_is_sample_then_oracle_shift_then_update(kind, graph):
  """Each fused step equals a pad-0 update on the sampled rows shifted by the oracle with the step's shifts, taus and
  noise: outputs, parameters and (prioritized) the sum tree after the priority write-back, bit for bit."""
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  cap, seed, p = 512, 3, 4
  agent, rep = _agent(kind, graph=graph, seed=seed)
  dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6)
  twin = None
  if agent.PRIORITIZED:
    _, twin = _agent(kind, seed=seed)
    dr.bulk_fill_synthetic(twin, (84, 84, 4), seed, 6)
  obs, a, r, d = ro.synthetic_rows(seed, np.arange(cap), 84 * 84 * 4, 6)
  L = agent.learner
  R = dl.Learner(L.net, batch_size=32, optimizer=L.opt)
  for name in ('online', 'target', 'opt_state', 'counters', 'max_seen_priority'):
    getattr(R, name).copy_(getattr(L, name))
  for step in range(4):
    agent.learn()
    torch.cuda.synchronize()
    ids = L.sampled_ids.cpu().numpy()
    S = L.shifts.cpu().numpy()
    s_tm1, s_t = ao.shift_batch(obs[ids, 0].reshape(-1, 84, 84, 4), obs[ids, 1].reshape(-1, 84, 84, 4), S, p)
    w = L.sampled_weights.cpu().numpy() if agent.PRIORITIZED else None
    R.update(s_tm1, a[ids], r[ids], d[ids], s_t, weights=w, taus=L.taus if dl.draws_taus(kind) else None,
             noise=L.noise if dl.noisy_layers(L.net) else None)
    torch.cuda.synchronize()
    for name in ('loss', 'per_example', 'priorities', 'grad_norm', 'online', 'opt_state'):
      assert torch.equal(getattr(L, name), getattr(R, name)), (step, name)
    if twin is not None:
      twin.update_priorities(ids, R.priorities.cpu().numpy())
      assert np.array_equal(rep.get_state()['distribution']['sum_tree']['storage'],
                            twin.get_state()['distribution']['sum_tree']['storage']), step


@pytest.mark.parametrize('kind', ['double_q', 'rainbow'])
def test_layouts_graph_and_eager_are_bit_identical_and_deterministic(kind):
  from dqn_zoo_b200 import replay as dr
  runs = []
  for dedup, graph in ((False, True), (True, True), (True, False), (False, True)):
    agent, rep = _agent(kind, graph=graph, dueling=kind == 'double_q', frame_dedup=dedup)
    dr.bulk_fill_synthetic_stacked(rep, (84, 84, 4), 5, 6, episode_len=37)
    for _ in range(5):
      agent.learn()
    torch.cuda.synchronize()
    runs.append({n: getattr(agent.learner, n).clone() for n in ('online', 'target', 'opt_state', 'counters', 'loss',
                                                                 'per_example', 'priorities', 'shifts')})
    runs[-1]['ids'] = agent.learner.sampled_ids.clone()
  for other in runs[1:]:
    for name, t in runs[0].items():
      assert torch.equal(t, other[name]), name


@pytest.mark.parametrize('kind', ['dqn', 'rainbow', 'iqn'])
def test_the_pad_adds_only_the_draw_and_the_shift_launches(kind):
  from dqn_zoo_b200 import _lib
  from dqn_zoo_b200 import replay as dr
  counts = {}
  for pad in (0, 4):
    agent, rep = _agent(kind, pad=pad, graph=False)
    dr.bulk_fill_synthetic(rep, (84, 84, 4), 3, 6)
    agent.learn()
    torch.cuda.synchronize()
    c0 = _lib.lib.dz_launch_count()
    agent.learn()
    torch.cuda.synchronize()
    counts[pad] = int(_lib.lib.dz_launch_count() - c0)
  # a kind that draws nothing at pad 0 also gains generate_randomness's counter step
  draws = kind != 'dqn'
  assert counts[4] == counts[0] + (2 if draws else 3), counts


# ---- acting ------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind,net', [('dqn', {}), ('iqn', {}), ('rainbow', {}), ('fqf', {})])
def test_acting_never_sees_a_shift(kind, net):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  off, on = _pair(kind, net, (84, 84), 4, B=64)
  rs = np.random.RandomState(4)
  E = 17
  obs = torch.as_tensor(rs.randint(0, 256, (E, 84, 84, 4)).astype(np.uint8), device='cuda')
  explore = torch.as_tensor(rs.uniform(size=(2, E)).astype(np.float32), device='cuda')
  kw = {}
  if kind == 'iqn':
    kw['taus'] = torch.as_tensor(rs.uniform(size=(E, 64)).astype(np.float32), device='cuda')
  if kind == 'rainbow':
    kw['noise'] = torch.as_tensor(rs.uniform(-1, 1, size=off.noise_stride).astype(np.float32), device='cuda')
  got = []
  for L in (off, on):
    a, q = L.act_batch(obs, epsilon=0.1, explore=explore, **kw)
    row = [a.clone(), q.clone()]
    for frozen in (False, True):
      x = L.actor(E, frozen=frozen)
      if frozen:
        x.load_params(L)
      a, q = x.act(obs, epsilon=0.1, explore=explore, **kw)
      row += [a.clone(), q.clone()]
    ev = ag.VectorEvaluator(L, 8, 0.05, [0, 3])
    ev.network_params = L
    env = environments.VectorCatch(8, 7)
    _, acts = _drive(ev, env, env.reset(), 30)
    row.append(torch.as_tensor(acts))
    torch.cuda.synchronize()
    got.append(row)
  for x, y in zip(*got):
    assert torch.equal(x.cpu(), y.cpu())


# ---- trainer, checkpoints ------------------------------------------------------------------------------------------------

def _drive(trainer, env, out, ticks):
  actions = []
  for _ in range(ticks):
    frames, st, rw, dc, lv = out
    a = trainer.step(frames, st, rw, dc, lv)
    actions.append(np.array(a))
    last = st == LAST
    if last.any():
      trainer.reset(np.nonzero(last)[0])
    out = env.step(a, reset=last)
  torch.cuda.synchronize()
  return out, np.array(actions)


def _trainer(seed=5, pad=4):
  from dqn_zoo_b200 import agent as ag
  agent, _ = _agent('double_q', pad=pad, capacity=2000, min_fill=40, seed=seed, dueling=True, epsilon=0.05)
  return agent, ag.VectorTrainer(agent, num_streams=8, rng_key=[0, 11])


def test_vector_trainer_state_and_checkpoint_round_trips(tmp_path):
  from dqn_zoo_b200 import environments
  E = 8
  agent, tr = _trainer()
  env = environments.VectorCatch(E, 21)
  out = env.reset()
  out, _ = _drive(tr, env, out, 60)
  assert tr.learn_steps > 0
  state, env_state, record = copy.deepcopy(tr.get_state()), env.get_state(), out[1:]
  tr.save_checkpoint(str(tmp_path / 'ckpt'))
  _, rest = _drive(tr, env, out, 60)
  params, shifts = agent.learner.online.clone(), agent.learner.shifts.clone()
  for restore in ('state', 'checkpoint'):
    agent2, tr2 = _trainer()
    if restore == 'state':
      tr2.set_state(state)
    else:
      tr2.load_checkpoint(str(tmp_path / 'ckpt'))
    env2 = environments.VectorCatch(E, 21)
    env2.set_state(env_state)
    _, again = _drive(tr2, env2, (env2.frames,) + record, 60)
    np.testing.assert_array_equal(rest, again)
    assert torch.equal(agent2.learner.online, params), restore
    assert torch.equal(agent2.learner.shifts, shifts), restore


def test_mismatched_checkpoints_raise_naming_the_pad(tmp_path):
  shifted, _ = _agent('double_q', pad=4, capacity=600)
  plain, _ = _agent('double_q', pad=0, capacity=600)
  shifted.save_checkpoint(str(tmp_path / 'shifted'))
  plain.save_checkpoint(str(tmp_path / 'plain'))
  with pytest.raises(ValueError, match='random_shift_pad'):
    plain.load_checkpoint(str(tmp_path / 'shifted'))
  with pytest.raises(ValueError, match='random_shift_pad'):
    shifted.load_checkpoint(str(tmp_path / 'plain'))
  # a checkpoint written before the field existed loads as pad 0
  path = os.path.join(str(tmp_path / 'plain'), 'agent.pkl')
  with open(path, 'rb') as f:
    state = pickle.load(f)
  del state['random_shift_pad']
  with open(path, 'wb') as f:
    pickle.dump(state, f)
  plain.load_checkpoint(str(tmp_path / 'plain'))
  with pytest.raises(ValueError, match='random_shift_pad'):
    shifted.load_checkpoint(str(tmp_path / 'plain'))


# ---- learning ----------------------------------------------------------------------------------------------------------
LEARNING_FRAMES = 1_500_000
LEARNING_THRESHOLD = 9.8          # test_dueling_double_q_learns_catch's bar, at its frame budget


def test_dueling_double_q_with_random_shifts_learns_catch():
  """Dueling double_q with random shifts at pad 1 on bench_env's Catch schedule: 32 streams for LEARNING_FRAMES frames,
  then >= 50 evaluation episodes at epsilon 0.01.  At this budget larger pads learn Catch more slowly (DESIGN.md §18)."""
  import importlib
  import sys
  here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools')
  if here not in sys.path:
    sys.path.insert(0, here)
  bench_env = importlib.import_module('bench_env')
  curve = bench_env.learning_run(LEARNING_FRAMES, seed=0, kind='double_q', dueling=True, random_shift_pad=1)
  frames, ret, episodes, _ = curve[-1]
  print('random-shift dueling double_q catch curve', curve)
  assert frames >= LEARNING_FRAMES and episodes >= 50
  assert ret >= LEARNING_THRESHOLD, curve
