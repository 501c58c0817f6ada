"""GPU: Munchausen-IQN (DESIGN.md §14).  The learner against the float64 oracle (oracle/munchausen_iqn_oracle.py) with
the bars of learner_parity.py on the packed and unpacked IQN GEMMs, the tensor-core and fp32-FMA torsos, at
non-default hyperparameters, through the fused `_learn()` and its CUDA graph; acting bit-identical to iqn's on the same
parameters and taus; the vectorised trainer and evaluator on Catch with state and checkpoint round trips; and a
learning curve on Catch."""

import copy
import os

import numpy as np
import pytest
import torch

import learner_parity as lp
from oracle import learner_oracle as lo
from oracle import munchausen_iqn_oracle as mo

pytestmark = pytest.mark.gpu

FIRST, MID, LAST = 0, 1, 2
KIND = 'munchausen_iqn'


def _f32(hyper):
  return mo.Hyper(*(float(np.float32(x)) for x in hyper))


def make_case(B, hw, seed, num_actions=6, taus=(64, 64, 64), hyper=mo.Hyper(), target_scale=1.0):
  """The learner and the oracle on the same online / target parameters.  `target_scale` multiplies the target head so
  that the target network's policy is sharp enough for tau log pi to fall below l0."""
  from dqn_zoo_b200 import learner as dl
  H, W = lp._hw(hw)
  spec = lo.NetSpec(KIND, num_actions, obs_hw=H, obs_w=W)
  net = dl.NetworkSpec(KIND, num_actions, obs_shape=(H, W, 4), tau_samples_s_tm1=taus[0], tau_samples_policy=taus[1],
                       tau_samples_s_t=taus[2])
  online = mo.init_params(spec, seed)
  target = mo.init_params(spec, seed + 1)
  for name in ('head/w', 'head/b'):
    target[name] = (target[name] * target_scale).astype(np.float32)
  L = dl.Learner(net, batch_size=B, munchausen_alpha=hyper.alpha, entropy_temperature=hyper.tau,
                 log_policy_clip=hyper.l0)
  L.set_params(online)
  L.set_params(target, blob='target')
  O = mo.Learner(spec, online, hyper=_f32(hyper))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  return spec, net, L, O, np.random.RandomState(seed)


def make_batch(net, B, rs):
  """learner_parity.make_batch for this kind: the batch and the three tau blocks [B][N] | [B][K] | [B][N']."""
  H, W = net.obs_shape[:2]
  s_tm1 = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
  s_t = rs.randint(0, 256, (B, H, W, 4)).astype(np.uint8)
  a = rs.randint(0, net.num_actions, B)
  r = rs.choice([-1.0, 0.0, 1.0, 0.37], size=B)
  d = rs.choice([0.0, 0.99, 0.99 ** 3], size=B)
  taus = [rs.uniform(size=(B, k)).astype(np.float32)
          for k in (net.tau_samples_s_tm1, net.tau_samples_policy, net.tau_samples_s_t)]
  return (s_tm1, a, r, d, s_t), lo.batch_from_numpy(s_tm1, a, r, d, s_t), [torch.tensor(t) for t in taus], \
      np.concatenate([t.reshape(-1) for t in taus])


def check_loss_and_gradients(B, hw, **case):
  """learner_parity.check_loss_and_gradients for this agent: loss, per-example losses, global norm and every gradient
  tensor within 1e-5 of the oracle, on the device's ReLU pattern when a unit sits at a kink."""
  spec, net, L, O, rs = make_case(B, hw, 3, **case)
  arrs, batch, taus_o, taus_flat = make_batch(net, B, rs)
  tap = lo.ReluTap()
  loss, aux, grads = O.grads(batch, taus=taus_o, tap=tap)
  L.update(*arrs, taus=taus_flat, apply_update=False)
  torch.cuda.synchronize()
  assert abs(float(L.loss.item()) - float(loss)) <= lp.REL * abs(float(loss)), (float(L.loss.item()), float(loss))
  masks, flips = lp.relu_kink_flips('iqn', L, tap)
  lp.assert_flips_at_the_kink(flips)
  if flips:
    print('relu kink flips %s B=%d: %s' % (hw, B, {k: v[:2] for k, v in flips.items()}))
    loss2, aux, grads = O.grads(batch, taus=taus_o, tap=lo.ReluTap(masks))
    assert abs(float(loss2) - float(loss)) <= 1e-5 * abs(float(loss))
  assert lp.rel_err(L.per_example.cpu().numpy(), aux['losses'].numpy()) <= lp.REL
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
  return spec, net, L, O, aux, batch


def check_three_optimizer_steps(B, hw, **case):
  """learner_parity.check_three_optimizer_steps for this agent (iqn's Adam without a norm clip, iqn's moment bar)."""
  spec, net, L, O, rs = make_case(B, hw, 5, **case)
  lr = L.opt.learning_rate
  p0 = {k: v.numpy().copy() for k, v in O.online.items()}
  for step in range(3):
    arrs, batch, taus_o, taus_flat = make_batch(net, B, rs)
    tap = lo.ReluTap()
    O.grads(batch, taus=taus_o, tap=tap)
    L.update(*arrs, taus=taus_flat, apply_update=True)
    torch.cuda.synchronize()
    masks, flips = lp.relu_kink_flips('iqn', L, tap)
    lp.assert_flips_at_the_kink(flips, step)
    aux = O.update(batch, taus=taus_o, tap=lo.ReluTap(masks) if flips else None)
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 2 * lp.REL * abs(float(aux['loss'])) + 1e-7
  got = L.get_params()
  for name, want in O.online.items():
    moved_ref = want.numpy() - p0[name]
    moved_got = got[name].astype(np.float64) - p0[name]
    assert lp.rel_err(moved_got, moved_ref) <= 1e-2, (name, lp.rel_err(moved_got, moved_ref))
    assert np.abs(moved_got - moved_ref).max() <= 0.5 * lr + 1e-7, name
  st = L.get_opt_state()
  for name in L.tensors:
    assert lp.rel_err(st['mu'][name], O.state['mu'][name].numpy()) <= 1e-2 or np.abs(st['mu'][name]).max() < 1e-12, name


# ---- parity ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('hw,B,A,taus,tc_torso,packed', [
    (84, 32, 6, (64, 64, 64), True, True),       # the stock shape
    (84, 16, 6, (64, 64, 64), True, True),       # exactly 1024 rows per apply
    (84, 8, 6, (33, 40, 36), True, False),       # ragged sample counts
    (44, 5, 6, (8, 5, 7), True, False),
    (84, 64, 6, (64, 64, 64), True, True),
    ((84, 88), 16, 6, (64, 64, 64), False, True),   # odd conv1 width: the fp32-FMA torso
    (84, 32, 1, (64, 64, 64), True, True),       # one action: bonus 0, y_j = r + discount zbar_j
    (84, 32, 18, (64, 64, 64), True, True),      # the full Atari action set: 18 lanes of the loss warp
], ids=lambda x: 'x'.join(map(str, x)) if isinstance(x, tuple) else str(x))
def test_parity_with_the_oracle(hw, B, A, taus, tc_torso, packed):
  L = check_loss_and_gradients(B, hw, num_actions=A, taus=taus)[2]
  assert lp.tensor_core_torso(L) == tc_torso
  assert (lp.mma_path(L, 'iqn_fc1_fwd') == 1) == packed
  check_three_optimizer_steps(B, hw, num_actions=A, taus=taus)


@pytest.mark.parametrize('hyper', [mo.Hyper(0.0, 0.03, -1.0), mo.Hyper(0.9, 1.0, -1.0), mo.Hyper(0.9, 0.03, -0.1)],
                         ids=['alpha0', 'tau1', 'l0_0.1'])
def test_non_default_hyperparameters(hyper):
  """Each case's batch holds examples on both sides of the clip (asserted from the oracle's float64 tau log pi)."""
  for scale in (1.0, 5.0, 20.0, 60.0):
    aux, batch = check_loss_and_gradients(32, 84, hyper=hyper, target_scale=scale)[4:]
    _, h = mo.soft_terms(aux['qbar_tm1'], _f32(hyper).tau)
    tlp = -h[torch.arange(32), batch['a_tm1'].long()]
    below, above = int((tlp < hyper.l0).sum()), int((tlp > hyper.l0).sum())
    if below and above:
      break
  assert below > 0 and above > 0, (scale, below, above)
  print('%s: target scale %g, %d examples below l0 and %d above' % (hyper, scale, below, above))


# ---- the fused step and its CUDA graph ------------------------------------------------------------------------------

def _agent(kind=KIND, capacity=512, seed=3, graph=True, min_fill=None, **extra):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  rep = dr.TransitionReplay(capacity, dr.Transition(None, None, None, None, None), np.random.RandomState(seed))
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=(min_fill or capacity) / capacity, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=graph, huber_param=1.0,
                tau_samples_policy=64, tau_samples_s_tm1=64, tau_samples_s_t=64)
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
  spec = lo.NetSpec(KIND, 6)
  O = mo.Learner(spec, L.get_params('online'), hyper=_f32(mo.Hyper()))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params('target').items()}
  B, n = 32, 64
  for step in range(steps):
    agent.learn()
    torch.cuda.synchronize()
    ids = L.sampled_ids.cpu().numpy()
    flat = L.taus[:3 * B * n].cpu()
    taus = [flat[i * B * n:(i + 1) * B * n].reshape(B, n) for i in range(3)]
    batch = lo.batch_from_numpy(*ro._stack_fields(ora._structure, ora.get(ids.tolist())))
    aux = O.update(batch, taus=taus)
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
  for name in ('online', 'target', 'opt_state', 'counters', 'loss', 'per_example', 'taus'):
    assert torch.equal(getattr(graphed.learner, name), getattr(eager.learner, name)), name


# ---- acting ----------------------------------------------------------------------------------------------------------

def test_acting_equals_iqn_on_the_same_blob_and_taus():
  from dqn_zoo_b200 import learner as dl
  rs = np.random.RandomState(8)
  lm = dl.Learner(dl.NetworkSpec(KIND, 6), batch_size=32)
  li = dl.Learner(dl.NetworkSpec('iqn', 6), batch_size=32)
  lm.init_params(4)
  li.set_params(lm.get_params(), also_target=True)
  assert torch.equal(lm.online, li.online)
  obs = torch.as_tensor(rs.randint(0, 256, (256, 84, 84, 4)).astype(np.uint8), device='cuda')
  explore = torch.as_tensor(rs.uniform(size=(2, 256)).astype(np.float32), device='cuda')
  taus = torch.as_tensor(rs.uniform(size=(256, 64)).astype(np.float32), device='cuda')
  for E in (1, 17, 32):
    am, qm = lm.act_batch(obs[:E], epsilon=0.3, explore=explore[:, :E], taus=taus[:E])
    ai, qi = li.act_batch(obs[:E], epsilon=0.3, explore=explore[:, :E], taus=taus[:E])
    assert torch.equal(qm, qi) and torch.equal(am, ai), E
  for E in (1, 33, 256):
    for frozen in (False, True):
      xm, xi = lm.actor(E, frozen=frozen), li.actor(E, frozen=frozen)
      if frozen:
        xm.load_params(lm)
        xi.load_params(li)
      am, qm = xm.act(obs[:E], epsilon=0.3, explore=explore[:, :E].contiguous(), taus=taus[:E].contiguous())
      ai, qi = xi.act(obs[:E], epsilon=0.3, explore=explore[:, :E].contiguous(), taus=taus[:E].contiguous())
      torch.cuda.synchronize()
      assert torch.equal(qm, qi) and torch.equal(am, ai), (E, frozen)
      # the actors' own draws: the same generator, stream and counter as iqn's
      assert torch.equal(xm.generate_randomness(5), xi.generate_randomness(5)), (E, frozen)
  assert torch.equal(lm.q_values(obs[0], taus=taus[0]), li.q_values(obs[0], taus=taus[0]))


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
  # an iqn checkpoint does not load into a munchausen_iqn agent, though its parameters have the same names
  iqn_agent, _ = _agent('iqn', capacity=2000, min_fill=40)
  iqn_agent.save_checkpoint(str(tmp_path / 'iqn'))
  with pytest.raises(ValueError):
    agent.load_checkpoint(str(tmp_path / 'iqn'))
  assert agent.get_state()['online_params'].keys() == iqn_agent.get_state()['online_params'].keys()


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


def test_batched_actor_acting_limits():
  """BatchedEpsilonGreedyActor over a munchausen_iqn learner: streams beyond the batch act through an acting context,
  whose E * tau_samples_policy <= 16384 limit applies as for iqn."""
  from dqn_zoo_b200 import agent as ag
  agent, _ = _agent(capacity=600)
  obs = torch.randint(0, 256, (256, 84, 84, 4), dtype=torch.uint8, device='cuda')
  actor = ag.BatchedEpsilonGreedyActor(agent.learner, 256, exploration_epsilon=0.01, rng_key=[0, 3])
  actions = np.array(actor.step(obs))
  assert actions.shape == (256,) and actions.min() >= 0 and actions.max() < 6
  with pytest.raises(ValueError, match='16384'):
    ag.BatchedEpsilonGreedyActor(agent.learner, 257, exploration_epsilon=0.01, rng_key=[0, 3])


# ---- learning --------------------------------------------------------------------------------------------------------
LEARNING_FRAMES = 1_000_000       # the measured curve reaches 18.77 at 0.8M frames and 18.91 at 1M (DESIGN.md §14)
LEARNING_THRESHOLD = 9.45         # half the measured 18.91 at 1M frames


def _tools(name):
  import importlib
  import sys
  here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools')
  if here not in sys.path:
    sys.path.insert(0, here)
  return importlib.import_module(name)


def test_munchausen_iqn_learns_catch():
  """32 Catch streams for LEARNING_FRAMES frames, then >= 50 evaluation episodes at epsilon 0.01: the mean return
  reaches at least half of the measured one (DESIGN.md §14)."""
  bench_env = _tools('bench_env')
  curve = bench_env.learning_run(LEARNING_FRAMES, seed=0, kind=KIND)
  frames, ret, episodes, _ = curve[-1]
  print('munchausen_iqn catch curve', curve)
  assert frames >= LEARNING_FRAMES and episodes >= 50
  assert ret >= LEARNING_THRESHOLD, curve
