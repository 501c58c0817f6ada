"""GPU: noisy networks (DESIGN.md §17) of dqn, double_q, prioritized and munchausen, plain and dueling.  The learner
against the float64 oracle (oracle/noisy_oracle.py) with the bars of learner_parity.py on the tensor-core and fp32-FMA
paths; the one-stream noisy tensor-core fc forward and input gradient against float64; the noise slots each pass reads;
the fused `_learn()` and its CUDA graph; acting with shared and per-stream noise through act_batch and live and frozen
actors; trainer, evaluator and checkpoint round trips; and NoisyNet-DQN learning Catch."""

import copy
import os
import pickle

import numpy as np
import pytest
import torch

import learner_parity as lp
import test_gpu_fc_dgrad as fcd
import test_gpu_fc_forward as fcf
from oracle import learner_oracle as lo
from oracle import munchausen_oracle as mo
from oracle import noisy_oracle as no

pytestmark = pytest.mark.gpu

KINDS = no.KINDS
LAST = 2
NETS = [False, True]
NET_IDS = ['plain', 'dueling']


def _f32(hyper):
  return mo.Hyper(*(float(np.float32(x)) for x in hyper))


def _raw_noise(spec, dueling, rs):
  one = {}
  for name, n in no.noise_shapes(spec, dueling):
    x = np.clip(rs.standard_normal(n), -2, 2)
    one[name] = (np.sign(x) * np.sqrt(np.abs(x))).astype(np.float32)
  return one


def _noise(spec, net, dueling, rs):
  """Three applies: (oracle dicts of float64 tensors, the device's packed vector)."""
  from dqn_zoo_b200 import learner as dl
  raw = [_raw_noise(spec, dueling, rs) for _ in range(3)]
  return [{k: torch.tensor(v, dtype=torch.float64) for k, v in one.items()} for one in raw], dl.pack_noise(net, raw)


def make_case(kind, dueling, B, hw, seed, num_actions=6):
  """The noisy learner and the noisy oracle on the same online / target parameters (sigma five times the init's, so
  that the noise terms are not small beside mu)."""
  from dqn_zoo_b200 import learner as dl
  H, W = lp._hw(hw)
  spec = lo.NetSpec(kind, num_actions, obs_hw=H, obs_w=W, noisy_sigma0=0.5)
  net = dl.NetworkSpec(kind, num_actions, obs_shape=(H, W, 4), dueling=dueling, noisy=True)
  online = no.init_params(spec, seed, dueling)
  target = no.init_params(spec, seed + 1, dueling)
  L = dl.Learner(net, batch_size=B)
  L.set_params(online)
  L.set_params(target, blob='target')
  O = no.Learner(spec, online, dueling=dueling, hyper=_f32(mo.Hyper()))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  return spec, net, L, O, np.random.RandomState(seed)


def _weights(kind, w):
  return torch.tensor(w) if kind == 'prioritized' else None


def _table(dueling):
  return 'rainbow' if dueling else 'dqn'   # learner_parity's ReLU buffers: adv1 / val1, or fc1


def check_loss_and_gradients(kind, dueling, B, hw, num_actions):
  """Loss, per-example values, global norm and every gradient tensor, sigma tensors included, within 1e-5 of the
  oracle; ReLU kink flips of the torso and of every 512-wide layer are counted."""
  spec, net, L, O, rs = make_case(kind, dueling, B, hw, 3, num_actions)
  arrs, batch, _, _, _, _, _ = lp.make_batch(spec, net, B, rs)
  noise_o, noise_flat = _noise(spec, net, dueling, rs)
  w = np.random.RandomState(B).uniform(0.1, 1.0, B) if kind == 'prioritized' else None
  tap = lo.ReluTap()
  loss, aux, grads = O.grads(batch, _weights(kind, w), noise=noise_o, tap=tap)
  L.update(*arrs, weights=w, noise=noise_flat, apply_update=False)
  torch.cuda.synchronize()
  assert abs(float(L.loss.item()) - float(loss)) <= lp.REL * abs(float(loss)), (float(L.loss.item()), float(loss))
  masks, flips = lp.relu_kink_flips(_table(dueling), L, tap)
  lp.assert_flips_at_the_kink(flips)
  if flips:
    print('relu kink flips noisy %s %s %s B=%d: %s' % (kind, NET_IDS[dueling], hw, B, {k: v[:2] for k, v in flips.items()}))
    loss2, aux, grads = O.grads(batch, _weights(kind, w), noise=noise_o, tap=lo.ReluTap(masks))
    assert abs(float(loss2) - float(loss)) <= 1e-5 * abs(float(loss))
  want_pe = (aux['losses'] if kind == 'munchausen' else aux['td_errors']).numpy()
  assert lp.rel_err(L.per_example.cpu().numpy(), want_pe) <= lp.REL
  if kind == 'prioritized':
    np.testing.assert_allclose(L.priorities.cpu().numpy(), aux['priorities'].numpy(), rtol=5e-5, atol=1e-6)
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
  return spec, net, L, O, rs


def check_three_optimizer_steps(kind, dueling, B, hw, num_actions):
  spec, net, L, O, rs = make_case(kind, dueling, B, hw, 5, num_actions)
  lr = L.opt.learning_rate
  p0 = {k: v.numpy().copy() for k, v in O.online.items()}
  for step in range(3):
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, net, B, rs)
    noise_o, noise_flat = _noise(spec, net, dueling, rs)
    w = rs.uniform(0.1, 1.0, B) if kind == 'prioritized' else None
    tap = lo.ReluTap()
    O.grads(batch, _weights(kind, w), noise=noise_o, tap=tap)
    L.update(*arrs, weights=w, noise=noise_flat, apply_update=True)
    torch.cuda.synchronize()
    masks, flips = lp.relu_kink_flips(_table(dueling), L, tap)
    lp.assert_flips_at_the_kink(flips, step)
    aux = O.update(batch, _weights(kind, w), noise=noise_o, tap=lo.ReluTap(masks) if flips else None)
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 2 * lp.REL * abs(float(aux['loss'])) + 1e-7
  got = L.get_params()
  for name, want in O.online.items():
    moved_ref = want.numpy() - p0[name]
    moved_got = got[name].astype(np.float64) - p0[name]
    assert lp.rel_err(moved_got, moved_ref) <= 1e-2, (name, lp.rel_err(moved_got, moved_ref))
    assert np.abs(moved_got - moved_ref).max() <= 0.5 * lr + 1e-7, name


def check_q_values(spec, net, dueling, L, O, rs):
  H, W = lp.obs_shape(spec)
  obs = rs.randint(0, 256, (H, W, 4)).astype(np.uint8)
  noise_o, noise_flat = _noise(spec, net, dueling, rs)
  want = no.apply_net(spec, O.online, torch.tensor(obs[None]), torch.float64, noise_o[0], dueling)['q_values'][0]
  got = L.q_values(torch.tensor(obs), noise=noise_flat[:L.noise_stride]).cpu().numpy()
  np.testing.assert_allclose(got, want.numpy(), rtol=2e-5, atol=2e-6)


# ---- parity ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dueling', NETS, ids=NET_IDS)
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('hw,B,A,tc_torso', [
    (84, 32, 6, True),          # the stock shape
    (44, 5, 6, True),
    ((84, 88), 32, 6, False),   # odd conv1 width: the fp32-FMA torso and noisy1 GEMMs
    (84, 32, 1, True),
    (84, 32, 18, True),
    (84, 32, 64, True),
], ids=lambda x: 'x'.join(map(str, x)) if isinstance(x, tuple) else str(x))
def test_parity_with_the_oracle(kind, dueling, hw, B, A, tc_torso):
  if kind == 'munchausen' and A > 18:
    pytest.skip('munchausen takes at most 18 actions')
  spec, net, L, O, rs = check_loss_and_gradients(kind, dueling, B, hw, A)
  assert lp.tensor_core_torso(L) == tc_torso
  for tag in ('noisy1_fwd', 'noisy1_dgrad'):   # the noisy 3136 -> 512 layer(s) on the tensor-core launches
    assert (lp.mma_path(L, tag) in (1, 2)) == tc_torso, tag
  check_q_values(spec, net, dueling, L, O, rs)
  check_three_optimizer_steps(kind, dueling, B, hw, A)


# ---- the one-stream noisy tensor-core fc layer -----------------------------------------------------------------------

@pytest.mark.parametrize('B,H,W,npass', [(32, 84, 84, 2), (32, 84, 84, 3), (48, 76, 76, 3)])
def test_one_noisy_stream_fc_forward_against_float64(B, H, W, npass):
  inp = fcf.make_inputs(B, H, W, npass, 1, True, seed=B + H + npass)
  new, _, _ = fcf.run(inp, per_pass=False)
  old, _, _ = fcf.run(inp, per_pass=True)
  want = fcf.reference(inp)
  for got in (new, old):
    assert not np.isnan(got).any()
    assert fcf.rel(got.astype(np.float64).sum(axis=2), want) < 3e-6
  np.testing.assert_array_equal(new, old)


@pytest.mark.parametrize('B,H,W', [(32, 84, 84), (48, 76, 76)])
def test_one_noisy_stream_fc_dgrad_against_float64(B, H, W):
  inp = fcd.make_inputs(B, H, W, 1, True, seed=B + H)
  new, _ = fcd.run(inp, converters=False)
  old, _ = fcd.run(inp, converters=True)
  want = fcd.reference(inp)
  for got in (new, old):
    assert not np.isnan(got).any()
    assert fcd.rel(got.astype(np.float64).sum(axis=1), want) < 3e-6
  np.testing.assert_array_equal(new, old)


# ---- noise slots -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dueling', NETS, ids=NET_IDS)
@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('tc', [True, False], ids=['tc', 'fma'])
def test_each_noise_slot_changes_exactly_the_passes_that_read_it(kind, dueling, tc):
  hw = 84 if tc else (84, 88)
  spec, net, L, O, rs = make_case(kind, dueling, 32, hw, 9)
  arrs, _, _, _, _, _, _ = lp.make_batch(spec, net, 32, rs)
  _, base = _noise(spec, net, dueling, rs)
  stride = L.noise_stride

  def heads(noise):
    L.update(*arrs, noise=noise, apply_update=False)
    torch.cuda.synchronize()
    return [lp.device_buffer(L, 'out%d' % p) for p in range(3)]

  ref = heads(base)
  reads = {0: {0}, 1: set() if kind == 'dqn' else {1}, 2: {2}}
  for k in range(3):
    moved = base.copy()
    moved[k * stride:(k + 1) * stride] = moved[k * stride:(k + 1) * stride] * 0.5 + 0.25
    got = heads(moved)
    changed = {p for p in range(3) if not torch.equal(got[p], ref[p])}
    # pass 1 holds nothing for dqn: its output buffer is never written
    assert changed == reads[k], (k, changed)


# ---- the fused step and its CUDA graph ------------------------------------------------------------------------------

def _agent(kind, capacity=512, seed=3, graph=True, min_fill=None, dueling=False, noisy=True, epsilon=0.1):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  if kind == 'prioritized':
    rep = dr.PrioritizedTransitionReplay(capacity, dr.Transition(None, None, None, None, None), 0.6, lambda t: 0.4, 1e-3,
                                         True, np.random.RandomState(seed))
  else:
    rep = dr.TransitionReplay(capacity, dr.Transition(None, None, None, None, None), np.random.RandomState(seed))
  common = dict(preprocessor=None, sample_network_input=None,
                network=dl.NetworkSpec(kind, 6, dueling=dueling, noisy=noisy), optimizer=None,
                transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=(min_fill or capacity) / capacity, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=graph)
  return ag.AGENTS[kind](exploration_epsilon=lambda t: epsilon, grad_error_bound=1.0 / 32, **common), rep


def _filled(kind, graph, seed=3, dueling=False):
  from dqn_zoo_b200 import replay as dr
  agent, rep = _agent(kind, graph=graph, seed=seed, dueling=dueling)
  dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6)
  return agent, rep


def _split_noise(L, dueling):
  from dqn_zoo_b200 import learner as dl
  flat = L.noise.cpu().numpy()
  out, at = [], 0
  for _ in range(3):
    one = {}
    for name, n in dl.noise_vector_sizes(L.net):
      one[name] = torch.tensor(flat[at:at + n], dtype=torch.float64)
      at += (n + 3) // 4 * 4
    out.append(one)
  return out


@pytest.mark.parametrize('dueling', NETS, ids=NET_IDS)
@pytest.mark.parametrize('kind', KINDS)
def test_fused_learn_matches_the_oracle_step_by_step(kind, dueling):
  """The fused step's loss, per-example values and (prioritized) priorities and sum-tree leaves are the oracle's on the
  sampled batch, its importance weights and the noise the step drew."""
  from oracle import replay_oracle as ro
  cap, seed = 512, 3
  agent, rep = _filled(kind, graph=False, seed=seed, dueling=dueling)
  obs, a, r, d = ro.synthetic_rows(seed, np.arange(cap), 84 * 84 * 4, 6)
  L = agent.learner
  spec = lo.NetSpec(kind, 6)
  O = no.Learner(spec, L.get_params('online'), dueling=dueling, hyper=_f32(mo.Hyper()))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params('target').items()}
  for step in range(3):
    agent.learn()
    torch.cuda.synchronize()
    ids = L.sampled_ids.cpu().numpy()
    batch = lo.batch_from_numpy(obs[ids, 0].reshape(-1, 84, 84, 4), a[ids], r[ids], d[ids], obs[ids, 1].reshape(-1, 84, 84, 4))
    w = torch.tensor(L.sampled_weights.cpu().numpy()) if kind == 'prioritized' else None
    aux = O.update(batch, w, noise=_split_noise(L, dueling))
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 1e-4 * abs(float(aux['loss'])), step
    want = aux['losses'] if kind == 'munchausen' else aux['td_errors']
    np.testing.assert_allclose(L.per_example.cpu().numpy(), want.numpy(), rtol=1e-3, atol=1e-7)
    if kind == 'prioritized':
      prio = L.priorities.cpu().numpy()
      np.testing.assert_allclose(prio, aux['priorities'].numpy(), rtol=1e-3, atol=1e-6)
      leaves = np.asarray(rep._distribution.get_exponentiated_priorities(ids.tolist()), dtype=np.float64)
      np.testing.assert_allclose(leaves, np.power(prio.astype(np.float64), 0.6), rtol=1e-6)


@pytest.mark.parametrize('dueling', NETS, ids=NET_IDS)
@pytest.mark.parametrize('kind', KINDS)
def test_graph_is_bit_identical_to_eager_and_runs_are_deterministic(kind, dueling):
  runs = []
  for graph in (True, False, False):
    agent, _ = _filled(kind, graph=graph, dueling=dueling)
    for _ in range(6):
      agent.learn()
    torch.cuda.synchronize()
    runs.append({n: getattr(agent.learner, n).clone() for n in ('online', 'target', 'opt_state', 'counters', 'loss',
                                                                  'per_example', 'priorities', 'noise')})
  for other in runs[1:]:
    for name, t in runs[0].items():
      assert torch.equal(t, other[name]), name


# ---- acting ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('dueling', NETS, ids=NET_IDS)
@pytest.mark.parametrize('kind', ['dqn', 'prioritized'])
def test_acting_shared_and_per_stream_noise(kind, dueling):
  from dqn_zoo_b200 import learner as dl
  rs = np.random.RandomState(8)
  L = dl.Learner(dl.NetworkSpec(kind, 6, dueling=dueling, noisy=True), batch_size=256)
  L.init_params(4)
  spec = lo.NetSpec(kind, 6)
  online = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params().items()}
  obs_np = rs.randint(0, 256, (256, 84, 84, 4)).astype(np.uint8)
  obs = torch.as_tensor(obs_np, device='cuda')
  explore = torch.as_tensor(rs.uniform(size=(2, 256)).astype(np.float32), device='cuda')
  stride = L.noise_stride
  applies = [_raw_noise(spec, dueling, rs) for _ in range(256)]
  stream = torch.as_tensor(dl.pack_noise(L.net, applies).reshape(256, stride), device='cuda')
  shared = stream[0].clone()
  same = shared[None].repeat(256, 1).contiguous()
  want_shared = no.apply_net(spec, online, torch.tensor(obs_np), torch.float64, applies[0], dueling)['q_values'].numpy()
  want_stream = np.concatenate([no.apply_net(spec, online, torch.tensor(obs_np[e:e + 1]), torch.float64, applies[e],
                                             dueling)['q_values'].numpy() for e in range(256)])
  for E in (1, 17, 32):
    _, q = L.act_batch(obs[:E], explore=explore[:, :E], noise=shared)
    np.testing.assert_allclose(q.cpu().numpy(), want_shared[:E], rtol=2e-5, atol=2e-6)
    _, q2 = L.act_batch(obs[:E], explore=explore[:, :E], stream_noise=stream[:E])
    np.testing.assert_allclose(q2.cpu().numpy(), want_stream[:E], rtol=2e-5, atol=2e-6)
  rows = {}
  for E in (1, 33, 256):
    for frozen in (False, True):
      x = L.actor(E, frozen=frozen)
      if frozen:
        x.load_params(L)
      for mode in ('shared', 'stream', 'same'):
        kw = {'noise': shared} if mode == 'shared' else {'stream_noise': (stream if mode == 'stream' else same)[:E].contiguous()}
        a, q = x.act(obs[:E], epsilon=0.0, explore=explore[:, :E].contiguous(), **kw)
        torch.cuda.synchronize()
        want = want_stream if mode == 'stream' else want_shared
        np.testing.assert_allclose(q.cpu().numpy(), want[:E], rtol=2e-5, atol=2e-6, err_msg=str((E, frozen, mode)))
        assert np.array_equal(a.cpu().numpy(), q.cpu().numpy().argmax(1)), (E, frozen, mode)
        rows[(E, frozen, mode)] = q.clone()
  for frozen in (False, True):
    for mode in ('shared', 'stream', 'same'):
      assert torch.equal(rows[(256, frozen, mode)][:1], rows[(1, frozen, mode)]), (frozen, mode)
      assert torch.equal(rows[(256, frozen, mode)][:33], rows[(33, frozen, mode)]), (frozen, mode)
  # every row carrying the same apply: an actor's shared mode runs the 3136 -> 512 layer on the tensor-core plan and its
  # per-stream mode on the fp32-FMA row-noise kernels, so they agree to the parity bars; act_batch runs both on the
  # fp32-FMA kernels, where they agree bit for bit
  for E in (1, 33, 256):
    for frozen in (False, True):
      q_same, q_shared = rows[(E, frozen, 'same')], rows[(E, frozen, 'shared')]
      np.testing.assert_allclose(q_same.cpu().numpy(), q_shared.cpu().numpy(), rtol=2e-5, atol=2e-6)
  _, qa = L.act_batch(obs[:32], noise=shared)
  _, qb = L.act_batch(obs[:32], stream_noise=same[:32])
  assert torch.equal(qa, qb)


def test_actor_randomness_draws_one_apply_or_one_per_stream():
  from dqn_zoo_b200 import learner as dl
  L = dl.Learner(dl.NetworkSpec('dqn', 6, noisy=True), batch_size=32)
  x = L.actor(8)
  one = x.generate_randomness(5).clone()
  many = x.generate_randomness(5, per_stream=True).clone()
  assert one.shape == (L.noise_stride,) and many.shape == (8, L.noise_stride)
  assert torch.isfinite(many).all() and many.abs().max() <= 2 ** 0.5 + 1e-6
  plain = dl.Learner(dl.NetworkSpec('dqn', 6), batch_size=32)
  with pytest.raises(ValueError):
    plain.actor(8).generate_randomness(5, per_stream=True)


# ---- the vectorised trainer and evaluator on Catch, checkpoints --------------------------------------------------------

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


def _trainer(dueling, seed=5):
  from dqn_zoo_b200 import agent as ag
  agent, _ = _agent('double_q', capacity=2000, min_fill=40, seed=seed, dueling=dueling, epsilon=0.0)
  return agent, ag.VectorTrainer(agent, num_streams=8, rng_key=[0, 11], per_stream_noise=True)


@pytest.mark.parametrize('dueling', NETS, ids=NET_IDS)
def test_vector_trainer_state_and_checkpoint_round_trips(tmp_path, dueling):
  from dqn_zoo_b200 import environments
  E = 8
  agent, tr = _trainer(dueling)
  env = environments.VectorCatch(E, 21)
  out = env.reset()
  out, _ = _drive(tr, env, out, 60)
  assert tr.learn_steps > 0
  state, env_state, record = copy.deepcopy(tr.get_state()), env.get_state(), out[1:]
  tr.save_checkpoint(str(tmp_path / 'ckpt'))
  _, rest = _drive(tr, env, out, 60)
  params = agent.learner.online.clone()
  for restore in ('state', 'checkpoint'):
    agent2, tr2 = _trainer(dueling)
    if restore == 'state':
      tr2.set_state(state)
    else:
      tr2.load_checkpoint(str(tmp_path / 'ckpt'))
    env2 = environments.VectorCatch(E, 21)
    env2.set_state(env_state)
    _, again = _drive(tr2, env2, (env2.frames,) + record, 60)
    np.testing.assert_array_equal(rest, again)
    assert torch.equal(agent2.learner.online, params), restore


def test_mismatched_checkpoints_raise_naming_noisy(tmp_path):
  noisy, _ = _agent('double_q', capacity=600)
  plain, _ = _agent('double_q', capacity=600, noisy=False)
  noisy.save_checkpoint(str(tmp_path / 'noisy'))
  plain.save_checkpoint(str(tmp_path / 'plain'))
  with pytest.raises(ValueError, match='noisy'):
    plain.load_checkpoint(str(tmp_path / 'noisy'))
  with pytest.raises(ValueError, match='noisy'):
    noisy.load_checkpoint(str(tmp_path / 'plain'))
  # a checkpoint written before the field existed (no 'noisy' key) loads as a network without noise
  path = os.path.join(str(tmp_path / 'plain'), 'agent.pkl')
  with open(path, 'rb') as f:
    state = pickle.load(f)
  del state['noisy']
  with open(path, 'wb') as f:
    pickle.dump(state, f)
  plain.load_checkpoint(str(tmp_path / 'plain'))
  with pytest.raises(ValueError, match='noisy'):
    noisy.load_checkpoint(str(tmp_path / 'plain'))


@pytest.mark.parametrize('per_stream', [False, True], ids=['shared', 'per_stream'])
def test_vector_evaluator_state_round_trip(per_stream):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  E, cut, ticks = 16, 40, 90
  agent, _ = _agent('dqn', capacity=600, dueling=True)
  agent.learner.init_params(9)
  ev = ag.VectorEvaluator(agent.learner, E, 0.0, [0, 3], per_stream_noise=per_stream)
  ev.network_params = agent.learner
  env = environments.VectorCatch(E, 7)
  out = env.reset()
  out, _ = _drive(ev, env, out, cut)
  state, env_state, record = copy.deepcopy(ev.get_state()), env.get_state(), out[1:]
  _, rest = _drive(ev, env, out, ticks - cut)
  fresh = ag.VectorEvaluator(agent.learner, E, 0.0, [0, 3], per_stream_noise=per_stream)
  fresh.set_state(state)
  env2 = environments.VectorCatch(E, 7)
  env2.set_state(env_state)
  _, again = _drive(fresh, env2, (env2.frames,) + record, ticks - cut)
  np.testing.assert_array_equal(rest, again)
  np.testing.assert_array_equal(ev.episode_return, fresh.episode_return)


# ---- learning --------------------------------------------------------------------------------------------------------
LEARNING_FRAMES = 1_500_000
LEARNING_THRESHOLD = 9.9          # half of the 19.84 this run reached (H100, one seed)


def test_noisy_dqn_learns_catch():
  """NoisyNet-DQN: noisy dqn with a zero epsilon schedule, 32 Catch streams for LEARNING_FRAMES frames, then >= 50
  evaluation episodes."""
  import importlib
  import sys
  here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools')
  if here not in sys.path:
    sys.path.insert(0, here)
  bench_env = importlib.import_module('bench_env')
  curve = bench_env.learning_run(LEARNING_FRAMES, seed=0, kind='dqn', noisy=True)
  frames, ret, episodes, _ = curve[-1]
  print('noisy dqn catch curve', curve)
  assert frames >= LEARNING_FRAMES and episodes >= 50
  assert ret >= LEARNING_THRESHOLD, curve
