"""GPU: FQF (DESIGN.md §15).  The learner against the float64 oracle (oracle/fqf_oracle.py) at the bars of
learner_parity.py: the loss, the per-example losses, every gradient tensor (the fraction layer's included) and the
proposed fractions, on the packed and unpacked IQN GEMMs and both torsos, then three optimizer steps; the limit where
every fraction is uniform against an iqn learner given the same taus; the fused `_learn()` and its CUDA graph; acting;
the vectorised trainer and evaluator on Catch with state and checkpoint round trips; and a learning curve on Catch.

The oracle evaluates the quantile network at the float32 taus the device proposed (read back through
dz_test_learner_buffer), so both sides feed the cosine embedding the same inputs; the proposals themselves are compared
with the oracle's float64 ones at the same 1e-5 bar."""

import copy
import os

import numpy as np
import pytest
import torch

import learner_parity as lp
from oracle import fqf_oracle as fo
from oracle import learner_oracle as lo

pytestmark = pytest.mark.gpu

FIRST, MID, LAST = 0, 1, 2
KIND = 'fqf'


def make_case(B, hw, seed, num_actions=6, N=32, frac_scale=100.0, fraction_lr=2.5e-9, zero_fractions=False):
  """The learner and the oracle on the same online / target parameters.  `frac_scale` multiplies the initial fraction
  layer (its default init proposes fractions uniform to within about 1e-2; x100 spreads them)."""
  from dqn_zoo_b200 import learner as dl
  H, W = lp._hw(hw)
  spec = lo.NetSpec(KIND, num_actions, obs_hw=H, obs_w=W)
  net = dl.NetworkSpec(KIND, num_actions, obs_shape=(H, W, 4), num_fractions=N)
  online = fo.init_params(spec, seed, N)
  target = fo.init_params(spec, seed + 1, N)
  online['fraction/w'] = (online['fraction/w'] * frac_scale).astype(np.float32)
  online['fraction/b'] = np.linspace(-0.5, 0.5, N).astype(np.float32)
  if zero_fractions:
    online['fraction/w'][:] = 0
    online['fraction/b'][:] = 0
  L = dl.Learner(net, batch_size=B, fraction_learning_rate=fraction_lr)
  L.set_params(online)
  L.set_params(target, blob='target')
  O = fo.Learner(spec, online, hyper=fo.Hyper(N, float(np.float32(fraction_lr))))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  return spec, net, L, O, np.random.RandomState(seed)


def make_batch(net, B, rs):
  H, W = net.obs_shape[:2]
  s_tm1 = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
  s_t = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
  a = rs.randint(0, net.num_actions, B)
  r = rs.choice([-1.0, 0.0, 1.0, 0.37], size=B)
  d = rs.choice([0.0, 0.99, 0.99 ** 3], size=B)
  return (s_tm1, a, r, d, s_t), lo.batch_from_numpy(s_tm1, a, r, d, s_t)


def device_fractions(L):
  """(tau_tm1 [B, N+1], tau_hat_tm1 [B, N], tau_t, tau_hat_t) of the last step, as the device proposed them."""
  B, N = L.batch_size, L.net.num_fractions
  tau = lp.device_buffer(L, 'fqf_tau').numpy().reshape(2, B, N + 1)
  hat = lp.device_buffer(L, 'fqf_tau_hat').numpy().reshape(2, B, N)
  return tau[0], hat[0], tau[1], hat[1]


def check_fractions(fr, aux):
  for got, want in ((fr[0], aux['prop_tm1']['tau']), (fr[1], aux['prop_tm1']['tau_hat']), (fr[2], aux['prop_t']['tau']),
                    (fr[3], aux['prop_t']['tau_hat'])):
    assert lp.rel_err(got, want.numpy()) <= lp.REL, lp.rel_err(got, want.numpy())
    assert np.all(np.diff(got, axis=1) >= 0)


def main_norm(grads):
  return float(torch.sqrt(sum((g * g).sum() for k, g in grads.items() if k not in fo.FRACTION_TENSORS)))


def check_loss_and_gradients(B, hw, **case):
  spec, net, L, O, rs = make_case(B, hw, 3, **case)
  arrs, batch = make_batch(net, B, rs)
  L.update(*arrs, apply_update=False)
  torch.cuda.synchronize()
  fr = device_fractions(L)
  tap = lo.ReluTap()
  loss, aux, grads = O.grads(batch, device_fractions=fr, tap=tap)
  check_fractions(fr, aux)
  assert abs(float(L.loss.item()) - float(loss)) <= lp.REL * abs(float(loss)), (float(L.loss.item()), float(loss))
  masks, flips = lp.relu_kink_flips('iqn', L, tap)
  lp.assert_flips_at_the_kink(flips)
  if flips:
    print('relu kink flips %s B=%d: %s' % (hw, B, {k: v[:2] for k, v in flips.items()}))
    loss2, aux, grads = O.grads(batch, device_fractions=fr, tap=lo.ReluTap(masks))
    assert abs(float(loss2) - float(loss)) <= 1e-5 * abs(float(loss))
  assert lp.rel_err(L.per_example.cpu().numpy(), aux['losses'].numpy()) <= lp.REL
  gn = main_norm(grads)
  assert abs(float(L.grad_norm.item()) - gn) <= lp.REL * gn
  errs, bad = {}, {}
  for name in L.tensors:
    got, want = L.view(L.grads, name).cpu().numpy(), grads[name].numpy()
    if np.linalg.norm(want) < 1e-12 * max(gn, 1e-30):
      assert np.abs(got).max() <= 1e-9 * max(gn, 1.0), name
      continue
    errs[name] = lp.rel_err(got, want)
    if errs[name] > lp.REL:
      bad[name] = errs[name]
  print('fqf %s B=%d: fraction/w %.2e fraction/b %.2e' % (hw, B, errs.get('fraction/w', 0), errs.get('fraction/b', 0)))
  assert not bad, bad
  return spec, net, L, O, aux, batch, grads


def check_three_optimizer_steps(B, hw, **case):
  """Three full steps: Adam over the quantile network (iqn's moment bar) and centred RMSProp over the fraction layer."""
  spec, net, L, O, rs = make_case(B, hw, 5, **case)
  p0 = {k: v.numpy().copy() for k, v in O.online.items()}
  for step in range(3):
    arrs, batch = make_batch(net, B, rs)
    L.update(*arrs, apply_update=True)
    torch.cuda.synchronize()
    fr = device_fractions(L)
    tap = lo.ReluTap()
    O.grads(batch, device_fractions=fr, tap=tap)
    masks, flips = lp.relu_kink_flips('iqn', L, tap)
    lp.assert_flips_at_the_kink(flips, step)
    aux = O.update(batch, device_fractions=fr, tap=lo.ReluTap(masks) if flips else None)
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 2 * lp.REL * abs(float(aux['loss'])) + 1e-7
  got = L.get_params()
  moved_norm = {}
  for name, want in O.online.items():
    lr = O.frac_opt.learning_rate if name in fo.FRACTION_TENSORS else L.opt.learning_rate
    moved_ref = want.numpy() - p0[name]
    moved_got = got[name].astype(np.float64) - p0[name]
    moved_norm[name] = float(np.abs(moved_got).max())
    if name in fo.FRACTION_TENSORS and lr < 1e-6:
      # at the default 2.5e-9 a step is below half a float32 spacing of most weights, so the device's float32
      # parameters keep their bits where the float64 oracle moves: the bar is the step plus one spacing
      spacing = np.spacing(np.abs(p0[name]).astype(np.float32)).astype(np.float64)
      assert np.all(np.abs(moved_got - moved_ref) <= 3 * lr + spacing), name
      continue
    assert lp.rel_err(moved_got, moved_ref) <= 1e-2, (name, lp.rel_err(moved_got, moved_ref))
    assert np.abs(moved_got - moved_ref).max() <= 0.5 * lr + 1e-7, name
  st = L.get_opt_state()
  for name in L.tensors:
    assert lp.rel_err(st['mu'][name], O.state['mu'][name].numpy()) <= 1e-2 or np.abs(st['mu'][name]).max() < 1e-12, name
  return moved_norm


# ---- parity ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hw,B,A,N,tc_torso,packed', [
    (84, 32, 6, 32, True, True),          # the stock shape: 1024 / 1024 / 2048 rows on the packed GEMM
    (44, 5, 6, 32, True, False),
    (84, 1, 6, 32, True, False),
    (84, 33, 6, 32, True, True),
    (84, 64, 6, 32, True, True),
    ((84, 88), 32, 6, 32, False, True),   # odd conv1 width: the fp32-FMA torso
    (84, 32, 1, 32, True, True),
    (84, 32, 18, 32, True, True),
    (84, 32, 6, 2, True, False),
    (84, 32, 6, 128, True, True),
], ids=lambda x: 'x'.join(map(str, x)) if isinstance(x, tuple) else str(x))
def test_parity_with_the_oracle(hw, B, A, N, tc_torso, packed):
  L = check_loss_and_gradients(B, hw, num_actions=A, N=N)[2]
  assert lp.tensor_core_torso(L) == tc_torso
  assert (lp.mma_path(L, 'iqn_fc1_fwd') == 1) == packed
  check_three_optimizer_steps(B, hw, num_actions=A, N=N)


def test_the_fraction_optimizer_moves_the_fraction_layer():
  """At a fraction learning rate of 1e-3 the RMSProp tail visibly moves, and still matches the oracle's step."""
  moved = check_three_optimizer_steps(32, 84, fraction_lr=1e-3)
  assert moved['fraction/w'] > 1e-5 and moved['fraction/b'] > 1e-5, moved


# ---- the iqn limit ---------------------------------------------------------------------------------------------------

def test_uniform_fractions_match_iqn_at_the_same_taus():
  """fraction/w = fraction/b = 0: every tau is exactly i / 32 in float32, and the quantile part of the step is iqn's
  with tau_hat in all three tau blocks (the selector's mean over 32 samples is the interval-weighted sum)."""
  from dqn_zoo_b200 import learner as dl
  B, N = 32, 32
  spec, net, L, O, rs = make_case(B, 84, 3, zero_fractions=True)
  arrs, batch = make_batch(net, B, rs)
  L.update(*arrs, apply_update=False)
  torch.cuda.synchronize()
  fr = device_fractions(L)
  exact = np.arange(N + 1, dtype=np.float32) / N
  for tau in (fr[0], fr[2]):
    assert np.array_equal(tau, np.broadcast_to(exact, tau.shape))
  hat = ((np.arange(N) + 0.5) / N).astype(np.float32)
  iq = dl.Learner(dl.NetworkSpec('iqn', 6, tau_samples_s_tm1=N, tau_samples_policy=N, tau_samples_s_t=N), batch_size=B)
  params = L.get_params()
  iq.set_params({k: v for k, v in params.items() if k not in fo.FRACTION_TENSORS})
  iq.set_params({k: v for k, v in L.get_params('target').items() if k not in fo.FRACTION_TENSORS}, blob='target')
  iq.update(*arrs, taus=np.tile(hat, 3 * B), apply_update=False)
  torch.cuda.synchronize()
  assert abs(float(iq.loss.item()) - float(L.loss.item())) <= lp.REL * abs(float(L.loss.item()))
  assert lp.rel_err(L.per_example.cpu().numpy(), iq.per_example.cpu().numpy()) <= lp.REL
  for name in iq.tensors:
    assert lp.rel_err(L.view(L.grads, name).cpu().numpy(), iq.view(iq.grads, name).cpu().numpy()) <= lp.REL, name
  _, aux, grads = O.grads(batch, device_fractions=fr)
  for name in fo.FRACTION_TENSORS:
    assert lp.rel_err(L.view(L.grads, name).cpu().numpy(), grads[name].numpy()) <= lp.REL, name


# ---- the fused step and its CUDA graph ------------------------------------------------------------------------------

def _agent(kind=KIND, capacity=512, seed=3, graph=True, min_fill=None, **extra):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rep = dr.TransitionReplay(capacity, dr.Transition(None, None, None, None, None), np.random.RandomState(seed))
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=(min_fill or capacity) / capacity, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=graph, huber_param=1.0)
  if kind != KIND:
    common.update(tau_samples_policy=64, tau_samples_s_tm1=64, tau_samples_s_t=64)
  return ag.AGENTS[kind](exploration_epsilon=lambda t: 0.1, **common, **extra), rep


def test_fused_learn_matches_the_oracle_step_by_step_and_graph_is_bit_identical():
  from dqn_zoo_b200 import replay as dr
  from oracle import replay_oracle as ro
  cap, seed, steps = 512, 3, 4
  agent, rep = _agent(graph=False, seed=seed)
  dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6)
  ora = ro.TransitionReplay(cap, ro.Transition(None, None, None, None, None), np.random.RandomState(seed))
  obs, a, r, d = ro.synthetic_rows(seed, np.arange(cap), 84 * 84 * 4, 6)
  for i in range(cap):
    ora.add(ro.Transition(obs[i, 0].reshape(84, 84, 4), int(a[i]), float(r[i]), float(d[i]),
                          obs[i, 1].reshape(84, 84, 4)))
  L = agent.learner
  O = fo.Learner(lo.NetSpec(KIND, 6), L.get_params('online'))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params('target').items()}
  for step in range(steps):
    agent.learn()
    torch.cuda.synchronize()
    ids = L.sampled_ids.cpu().numpy()
    batch = lo.batch_from_numpy(*ro._stack_fields(ora._structure, ora.get(ids.tolist())))
    aux = O.update(batch, device_fractions=device_fractions(L))
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 1e-4 * abs(float(aux['loss'])), step
    np.testing.assert_allclose(L.per_example.cpu().numpy(), aux['losses'].numpy(), rtol=1e-3, atol=1e-7)
  graphed, grep = _agent(graph=True, seed=seed)
  dr.bulk_fill_synthetic(grep, (84, 84, 4), seed, 6)
  eager, erep = _agent(graph=False, seed=seed)
  dr.bulk_fill_synthetic(erep, (84, 84, 4), seed, 6)
  for _ in range(6):
    graphed.learn()
    eager.learn()
  torch.cuda.synchronize()
  for name in ('online', 'target', 'opt_state', 'counters', 'loss', 'per_example', 'grad_norm'):
    assert torch.equal(getattr(graphed.learner, name), getattr(eager.learner, name)), name
  assert torch.equal(lp.device_buffer(graphed.learner, 'fqf_tau'), lp.device_buffer(eager.learner, 'fqf_tau'))


# ---- acting ----------------------------------------------------------------------------------------------------------

def test_acting_q_values_and_actors():
  """act_batch's q-values are sum_i w_i Z at the proposed fractions (the oracle's float64 proposal: the float32 taus
  differ from it by rounding, hence a 1e-4 bar); live and frozen actors give row e the same bits at every E and
  act_batch's greedy actions; no taus are passed anywhere."""
  from dqn_zoo_b200 import learner as dl
  rs = np.random.RandomState(8)
  spec = lo.NetSpec(KIND, 6)
  params = fo.init_params(spec, 4)
  params['fraction/w'] = (params['fraction/w'] * 100).astype(np.float32)
  L = dl.Learner(dl.NetworkSpec(KIND, 6), batch_size=32)
  L.set_params(params, also_target=True)
  assert L.taus.numel() == 1 and L.plan.tau_floats == 0
  obs = torch.as_tensor(rs.randint(0, 256, (256, 84, 84, 4)).astype(np.uint8), device='cuda')
  _, q = L.act_batch(obs[:32])
  torch.cuda.synchronize()
  p64 = {k: torch.tensor(v, dtype=torch.float64) for k, v in params.items()}
  o = torch.as_tensor(obs[:32].cpu().numpy())
  prop = fo.fractions(p64, lo.torso(p64, o, torch.float64))
  z = fo.quantiles(spec, p64, o, torch.float64, prop['tau_hat'])
  want = (prop['w'][:, :, None] * z).sum(1).numpy()
  np.testing.assert_allclose(q.cpu().numpy(), want, rtol=1e-4, atol=1e-5)
  greedy, q32 = [x.clone() for x in L.act_batch(obs[:32])]
  q1 = L.q_values(obs[0]).clone()
  torch.cuda.synchronize()
  np.testing.assert_allclose(q1.cpu().numpy(), want[0], rtol=1e-4, atol=1e-5)
  rows = {}
  for E in (1, 33, 256):
    for frozen in (False, True):
      x = L.actor(E, frozen=frozen)
      if frozen:
        x.load_params(L)
      assert x.taus is None
      a, qa = x.act(obs[:E])
      torch.cuda.synchronize()
      rows.setdefault(frozen, []).append(qa.cpu().numpy().copy())
      n = min(E, 32)
      assert torch.equal(a[:n], greedy[:n]), (E, frozen)
      np.testing.assert_allclose(qa[:n].cpu().numpy(), q32[:n].cpu().numpy(), rtol=1e-5, atol=1e-6)
      with pytest.raises(ValueError):
        x.generate_randomness(5)
  for frozen, qs in rows.items():
    for qa in qs[1:]:
      assert np.array_equal(qa[:1], qs[0][:1]), frozen
    assert np.array_equal(qs[1], qs[2][:33]), frozen
  assert np.array_equal(rows[False][2], rows[True][2])


# ---- learning --------------------------------------------------------------------------------------------------------
LEARNING_FRAMES = 1_000_000       # the measured curve: 1.24 at 0.5M frames, 19.72 at 1M (DESIGN.md §15)
LEARNING_THRESHOLD = 9.86         # half the measured 19.72 at 1M frames


def _tools(name):
  import importlib
  import sys
  here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools')
  if here not in sys.path:
    sys.path.insert(0, here)
  return importlib.import_module(name)


def test_fqf_learns_catch():
  """32 Catch streams for LEARNING_FRAMES frames, then >= 50 evaluation episodes at epsilon 0.01: the mean return
  reaches at least half of the measured one (DESIGN.md §15)."""
  bench_env = _tools('bench_env')
  curve = bench_env.learning_run(LEARNING_FRAMES, seed=0, kind=KIND)
  frames, ret, episodes, _ = curve[-1]
  print('fqf catch curve', curve)
  assert frames >= LEARNING_FRAMES and episodes >= 50
  assert ret >= LEARNING_THRESHOLD, curve


def test_acting_row_limit():
  """E * num_fractions <= 16384: 512 streams of 32 fractions act, 513 are refused by the batched actor and the trainer."""
  from dqn_zoo_b200 import agent as ag
  agent, _ = _agent(capacity=600)
  obs = torch.randint(0, 256, (512, 84, 84, 4), dtype=torch.uint8, device='cuda')
  actor = ag.BatchedEpsilonGreedyActor(agent.learner, 512, exploration_epsilon=0.01, rng_key=[0, 3])
  actions = np.array(actor.step(obs))
  assert actions.shape == (512,) and actions.min() >= 0 and actions.max() < 6
  with pytest.raises(ValueError, match='16384'):
    ag.BatchedEpsilonGreedyActor(agent.learner, 513, exploration_epsilon=0.01, rng_key=[0, 3])
  with pytest.raises(ValueError, match='16384'):
    ag.VectorTrainer(agent, num_streams=513, rng_key=[0, 11])


# ---- the vectorised trainer and evaluator on Catch -------------------------------------------------------------------

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


def _trainer(seed=5):
  from dqn_zoo_b200 import agent as ag
  agent, _ = _agent(capacity=2000, min_fill=40, seed=seed)
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
  params = agent.learner.online.clone()
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
  iqn_agent, _ = _agent('iqn', capacity=2000, min_fill=40)
  iqn_agent.save_checkpoint(str(tmp_path / 'iqn'))
  with pytest.raises(ValueError):
    agent.load_checkpoint(str(tmp_path / 'iqn'))


def test_vector_evaluator_state_round_trip():
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  E, cut, ticks = 16, 40, 90
  agent, _ = _agent(capacity=600)
  agent.learner.init_params(9)

  def run(ev, env, out, n):
    acts = []
    for _ in range(n):
      frames, st, rw, dc, lv = out
      a = ev.step(frames, st, rw, dc, lv)
      acts.append(np.array(a))
      last = st == LAST
      if last.any():
        ev.reset(np.nonzero(last)[0])
      out = env.step(a, reset=last)
    torch.cuda.synchronize()
    return out, np.array(acts)

  ev = ag.VectorEvaluator(agent.learner, E, 0.05, [0, 3])
  ev.network_params = agent.learner
  env = environments.VectorCatch(E, 7)
  out = env.reset()
  out, _ = run(ev, env, out, cut)
  state, env_state, record = copy.deepcopy(ev.get_state()), env.get_state(), out[1:]
  _, rest = run(ev, env, out, ticks - cut)
  fresh = ag.VectorEvaluator(agent.learner, E, 0.05, [0, 3])
  fresh.set_state(state)
  env2 = environments.VectorCatch(E, 7)
  env2.set_state(env_state)
  _, again = run(fresh, env2, (env2.frames,) + record, ticks - cut)
  np.testing.assert_array_equal(rest, again)
  np.testing.assert_array_equal(ev.episode_return, fresh.episode_return)
