"""GPU: the dueling network (DESIGN.md §16) of dqn, double_q, prioritized and munchausen.  The learner against the
float64 oracle (oracle/dueling_oracle.py) with the bars of learner_parity.py on the tensor-core and fp32-FMA paths;
the two-stream plain tensor-core fc forward and input gradient against float64; the fused `_learn()` and its CUDA
graph; acting through act_batch and live and frozen actors; trainer, evaluator and checkpoint round trips; and a
learning curve on Catch."""

import copy

import numpy as np
import pytest
import torch

import learner_parity as lp
import test_gpu_fc_dgrad as fcd
import test_gpu_fc_forward as fcf
from oracle import dueling_oracle as do
from oracle import learner_oracle as lo
from oracle import munchausen_oracle as mo

pytestmark = pytest.mark.gpu

KINDS = do.KINDS
LAST = 2


def _f32(hyper):
  return mo.Hyper(*(float(np.float32(x)) for x in hyper))


def make_case(kind, B, hw, seed, num_actions=6):
  """The dueling learner and the dueling oracle on the same online / target parameters."""
  from dqn_zoo_b200 import learner as dl
  H, W = lp._hw(hw)
  spec = lo.NetSpec(kind, num_actions, obs_hw=H, obs_w=W)
  net = dl.NetworkSpec(kind, num_actions, obs_shape=(H, W, 4), dueling=True)
  online = do.init_params(spec, seed)
  target = do.init_params(spec, seed + 1)
  L = dl.Learner(net, batch_size=B)
  L.set_params(online)
  L.set_params(target, blob='target')
  O = do.Learner(spec, online, hyper=_f32(mo.Hyper()))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in target.items()}
  return spec, net, L, O, np.random.RandomState(seed)


def _weights(kind, w):
  return torch.tensor(w) if kind == 'prioritized' else None


def check_loss_and_gradients(kind, B, hw, num_actions):
  """Loss, per-example values, global norm and every gradient tensor within 1e-5 of the oracle; ReLU kink flips of
  the torso and of both h1 streams are counted (learner_parity's rainbow table names adv1 / val1 by the same buffers)."""
  spec, net, L, O, rs = make_case(kind, B, hw, 3, num_actions)
  arrs, batch, w, _, _, _, _ = lp.make_batch(spec, net, B, rs)
  w = np.random.RandomState(B).uniform(0.1, 1.0, B) if kind == 'prioritized' else None
  tap = lo.ReluTap()
  loss, aux, grads = O.grads(batch, _weights(kind, w), tap=tap)
  L.update(*arrs, weights=w, apply_update=False)
  torch.cuda.synchronize()
  assert abs(float(L.loss.item()) - float(loss)) <= lp.REL * abs(float(loss)), (float(L.loss.item()), float(loss))
  masks, flips = lp.relu_kink_flips('rainbow', L, tap)
  lp.assert_flips_at_the_kink(flips)
  if flips:
    print('relu kink flips dueling %s %s B=%d: %s' % (kind, hw, B, {k: v[:2] for k, v in flips.items()}))
    loss2, aux, grads = O.grads(batch, _weights(kind, w), tap=lo.ReluTap(masks))
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


def check_three_optimizer_steps(kind, B, hw, num_actions):
  spec, net, L, O, rs = make_case(kind, B, hw, 5, num_actions)
  lr = L.opt.learning_rate
  p0 = {k: v.numpy().copy() for k, v in O.online.items()}
  for step in range(3):
    arrs, batch, _, _, _, _, _ = lp.make_batch(spec, net, B, rs)
    w = rs.uniform(0.1, 1.0, B) if kind == 'prioritized' else None
    tap = lo.ReluTap()
    O.grads(batch, _weights(kind, w), tap=tap)
    L.update(*arrs, weights=w, apply_update=True)
    torch.cuda.synchronize()
    masks, flips = lp.relu_kink_flips('rainbow', L, tap)
    lp.assert_flips_at_the_kink(flips, step)
    aux = O.update(batch, _weights(kind, w), tap=lo.ReluTap(masks) if flips else None)
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 2 * lp.REL * abs(float(aux['loss'])) + 1e-7
  got = L.get_params()
  for name, want in O.online.items():
    moved_ref = want.numpy() - p0[name]
    moved_got = got[name].astype(np.float64) - p0[name]
    assert lp.rel_err(moved_got, moved_ref) <= 1e-2, (name, lp.rel_err(moved_got, moved_ref))
    assert np.abs(moved_got - moved_ref).max() <= 0.5 * lr + 1e-7, name
  st = L.get_opt_state()
  for name in L.tensors:
    assert lp.rel_err(st['mu'][name], O.state['mu'][name].numpy()) <= 5e-5 or np.abs(st['mu'][name]).max() < 1e-12, name


def check_q_values(spec, L, O, rs):
  H, W = lp.obs_shape(spec)
  obs = rs.randint(0, 256, (H, W, 4)).astype(np.uint8)
  want = do.apply_net(spec, O.online, torch.tensor(obs[None]), torch.float64)['q_values'][0]
  got = L.q_values(torch.tensor(obs)).cpu().numpy()
  np.testing.assert_allclose(got, want.numpy(), rtol=2e-5, atol=2e-6)


# ---- parity ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('hw,B,A,tc_torso', [
    (84, 32, 6, True),          # the stock shape
    (44, 5, 6, True),
    ((84, 88), 32, 6, False),   # odd conv1 width: the fp32-FMA torso and fc1 GEMMs
    (84, 32, 1, True),          # one action: q = v, no advantage gradient
    (84, 32, 18, True),
    (84, 32, 64, True),
], ids=lambda x: 'x'.join(map(str, x)) if isinstance(x, tuple) else str(x))
def test_parity_with_the_oracle(kind, hw, B, A, tc_torso):
  if kind == 'munchausen' and A > 18:
    pytest.skip('munchausen takes at most 18 actions')
  spec, net, L, O, rs = check_loss_and_gradients(kind, B, hw, A)
  assert lp.tensor_core_torso(L) == tc_torso
  for tag in ('fc1_fwd', 'fc1_dgrad'):   # both streams' 3136 -> 512 layer on the tensor-core launches
    assert (lp.mma_path(L, tag) in (1, 2)) == tc_torso, tag
  check_q_values(spec, L, O, rs)
  check_three_optimizer_steps(kind, B, hw, A)


# ---- the two-stream plain tensor-core fc layer -----------------------------------------------------------------------

@pytest.mark.parametrize('B,H,W,npass', [(32, 84, 84, 1), (32, 84, 84, 3), (32, 76, 76, 2), (48, 84, 84, 3)])
def test_two_plain_streams_fc_forward_against_float64(B, H, W, npass):
  inp = fcf.make_inputs(B, H, W, npass, 2, False, seed=B + H + npass)
  new, S, wb = fcf.run(inp, per_pass=False)
  old, _, _ = fcf.run(inp, per_pass=True)
  want = fcf.reference(inp)
  for got in (new, old):
    assert not np.isnan(got).any()
    assert fcf.rel(got.astype(np.float64).sum(axis=2), want) < 3e-6
  np.testing.assert_array_equal(new, old)
  assert wb == (1 if npass == 1 else 2) * 2 * inp['feat'] * 512 * 4   # both streams' weights staged once per blob


@pytest.mark.parametrize('B,H,W', [(32, 84, 84), (48, 76, 76)])
def test_two_plain_streams_fc_dgrad_against_float64(B, H, W):
  inp = fcd.make_inputs(B, H, W, 2, False, seed=B + H)
  new, _ = fcd.run(inp, converters=False)
  old, _ = fcd.run(inp, converters=True)
  want = fcd.reference(inp)
  for got in (new, old):
    assert not np.isnan(got).any()
    assert fcd.rel(got.astype(np.float64).sum(axis=1), want) < 3e-6
  np.testing.assert_array_equal(new, old)


# ---- the fused step and its CUDA graph ------------------------------------------------------------------------------

def _agent(kind, capacity=512, seed=3, graph=True, min_fill=None, dueling=True):
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import learner as dl
  from dqn_zoo_b200 import replay as dr
  if kind == 'prioritized':
    rep = dr.PrioritizedTransitionReplay(capacity, dr.Transition(None, None, None, None, None), 0.6, lambda t: 0.4, 1e-3,
                                         True, np.random.RandomState(seed))
  else:
    rep = dr.TransitionReplay(capacity, dr.Transition(None, None, None, None, None), np.random.RandomState(seed))
  common = dict(preprocessor=None, sample_network_input=None, network=dl.NetworkSpec(kind, 6, dueling=dueling),
                optimizer=None, transition_accumulator=dr.NStepTransitionAccumulator(1), replay=rep, batch_size=32,
                min_replay_capacity_fraction=(min_fill or capacity) / capacity, learn_period=4,
                target_network_update_period=16, rng_key=[0, seed], use_cuda_graph=graph)
  return ag.AGENTS[kind](exploration_epsilon=lambda t: 0.1, grad_error_bound=1.0 / 32, **common), rep


def _filled(kind, graph, seed=3):
  from dqn_zoo_b200 import replay as dr
  agent, rep = _agent(kind, graph=graph, seed=seed)
  dr.bulk_fill_synthetic(rep, (84, 84, 4), seed, 6)
  return agent, rep


@pytest.mark.parametrize('kind', ['dqn', 'double_q', 'munchausen'])
def test_fused_learn_matches_the_oracle_step_by_step(kind):
  from oracle import replay_oracle as ro
  cap, seed = 512, 3
  agent, _ = _filled(kind, graph=False, seed=seed)
  ora = ro.TransitionReplay(cap, ro.Transition(None, None, None, None, None), np.random.RandomState(seed))
  obs, a, r, d = ro.synthetic_rows(seed, np.arange(cap), 84 * 84 * 4, 6)
  for i in range(cap):
    ora.add(ro.Transition(obs[i, 0].reshape(84, 84, 4), int(a[i]), float(r[i]), float(d[i]), obs[i, 1].reshape(84, 84, 4)))
  L = agent.learner
  O = do.Learner(lo.NetSpec(kind, 6), L.get_params('online'), hyper=_f32(mo.Hyper()))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params('target').items()}
  for step in range(4):
    agent.learn()
    torch.cuda.synchronize()
    ids = L.sampled_ids.cpu().numpy()
    batch = lo.batch_from_numpy(*ro._stack_fields(ora._structure, ora.get(ids.tolist())))
    aux = O.update(batch)
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 1e-4 * abs(float(aux['loss'])), step
    want = aux['losses'] if kind == 'munchausen' else aux['td_errors']
    np.testing.assert_allclose(L.per_example.cpu().numpy(), want.numpy(), rtol=1e-3, atol=1e-7)


def test_prioritized_fused_learn_matches_the_oracle_priorities():
  """The fused step's loss and written-back priorities are the oracle's on the sampled batch and importance weights."""
  agent, rep = _filled('prioritized', graph=False)
  L = agent.learner
  O = do.Learner(lo.NetSpec('prioritized', 6), L.get_params('online'))
  O.target = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params('target').items()}
  from oracle import replay_oracle as ro
  obs, a, r, d = ro.synthetic_rows(3, np.arange(512), 84 * 84 * 4, 6)
  for step in range(3):
    agent.learn()
    torch.cuda.synchronize()
    ids = L.sampled_ids.cpu().numpy()
    w = L.sampled_weights.cpu().numpy()
    batch = lo.batch_from_numpy(obs[ids, 0].reshape(-1, 84, 84, 4), a[ids], r[ids], d[ids], obs[ids, 1].reshape(-1, 84, 84, 4))
    aux = O.update(batch, torch.tensor(w))
    assert abs(float(L.loss.item()) - float(aux['loss'])) <= 1e-4 * abs(float(aux['loss'])), step
    prio = L.priorities.cpu().numpy()
    np.testing.assert_allclose(prio, aux['priorities'].numpy(), rtol=1e-3, atol=1e-6)
    # the write-back: the replay's sum-tree leaves of the sampled ids hold the step's priorities ** 0.6
    leaves = np.asarray(rep._distribution.get_exponentiated_priorities(ids.tolist()), dtype=np.float64)
    np.testing.assert_allclose(leaves, np.power(prio.astype(np.float64), 0.6), rtol=1e-6)


@pytest.mark.parametrize('kind', KINDS)
def test_graph_is_bit_identical_to_eager_and_runs_are_deterministic(kind):
  runs = []
  for graph in (True, False, False):
    agent, _ = _filled(kind, graph=graph)
    for _ in range(6):
      agent.learn()
    torch.cuda.synchronize()
    runs.append({n: getattr(agent.learner, n).clone() for n in ('online', 'target', 'opt_state', 'counters', 'loss',
                                                                  'per_example', 'priorities')})
  for other in runs[1:]:
    for name, t in runs[0].items():
      assert torch.equal(t, other[name]), name


# ---- acting ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize('kind', ['dqn', 'double_q'])
def test_acting_against_the_oracle_and_row_invariant(kind):
  from dqn_zoo_b200 import learner as dl
  rs = np.random.RandomState(8)
  L = dl.Learner(dl.NetworkSpec(kind, 6, dueling=True), batch_size=32)
  L.init_params(4)
  spec = lo.NetSpec(kind, 6)
  online = {k: torch.tensor(v, dtype=torch.float64) for k, v in L.get_params().items()}
  obs_np = rs.randint(0, 256, (256, 84, 84, 4)).astype(np.uint8)
  obs = torch.as_tensor(obs_np, device='cuda')
  explore = torch.as_tensor(rs.uniform(size=(2, 256)).astype(np.float32), device='cuda')
  want = do.apply_net(spec, online, torch.tensor(obs_np), torch.float64)['q_values'].numpy()
  for E in (1, 17, 32):
    _, q = L.act_batch(obs[:E], epsilon=0.0, explore=explore[:, :E])
    np.testing.assert_allclose(q.cpu().numpy(), want[:E], rtol=2e-5, atol=2e-6)
  rows = {}
  for E in (1, 33, 256):
    for frozen in (False, True):
      x = L.actor(E, frozen=frozen)
      if frozen:
        x.load_params(L)
      a, q = x.act(obs[:E], epsilon=0.0, explore=explore[:, :E].contiguous())
      torch.cuda.synchronize()
      np.testing.assert_allclose(q.cpu().numpy(), want[:E], rtol=2e-5, atol=2e-6, err_msg=str((E, frozen)))
      assert np.array_equal(a.cpu().numpy(), q.cpu().numpy().argmax(1)), (E, frozen)
      rows[(E, frozen)] = q.clone()
  for frozen in (False, True):
    assert torch.equal(rows[(256, frozen)][:1], rows[(1, frozen)]), frozen
    assert torch.equal(rows[(256, frozen)][:33], rows[(33, frozen)]), frozen
  assert torch.equal(rows[(256, False)], rows[(256, True)])


def test_actor_features_match_the_learner_bit_for_bit():
  """The actor's conv3 features of an observation equal the learner step's features of the same observation."""
  from dqn_zoo_b200 import _lib
  import ctypes as C
  spec, net, L, O, rs = make_case('dqn', 32, 84, 7)
  arrs, _, _, _, _, _, _ = lp.make_batch(spec, net, 32, rs)
  L.update(*arrs, apply_update=False)
  torch.cuda.synchronize()
  feat = lp.device_buffer(L, 'act3').reshape(32, -1)
  x = L.actor(32)
  x.act(torch.as_tensor(arrs[0], device='cuda'))
  ptr, n = C.c_void_p(), C.c_int64()
  _lib.call('dz_test_actor_buffer', x._h, b'act3', C.byref(ptr), C.byref(n))
  out = torch.empty(n.value, dtype=torch.float32, device='cuda')
  _lib.call('dz_test_copy', out.data_ptr(), ptr, 4 * n.value, torch.cuda.current_stream().cuda_stream)
  torch.cuda.synchronize()
  assert torch.equal(out.cpu().reshape(32, -1), feat)


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


def _trainer(kind='double_q', seed=5, dueling=True):
  from dqn_zoo_b200 import agent as ag
  agent, _ = _agent(kind, capacity=2000, min_fill=40, seed=seed, dueling=dueling)
  return agent, ag.VectorTrainer(agent, num_streams=8, rng_key=[0, 11])


def test_vector_trainer_state_and_checkpoint_round_trips(tmp_path):
  from dqn_zoo_b200 import environments
  from dqn_zoo_b200 import reporting
  E = 8
  agent, tr = _trainer()
  env = environments.VectorCatch(E, 21)
  out = env.reset()
  out, _ = _drive(tr, env, out, 60)
  assert tr.learn_steps > 0
  state, env_state, record = copy.deepcopy(tr.get_state()), env.get_state(), out[1:]
  tr.save_checkpoint(str(tmp_path / 'ckpt'))
  cp = reporting.DirectoryCheckpoint(str(tmp_path / 'dir'))
  cp.state.trainer = tr
  cp.save()
  _, rest = _drive(tr, env, out, 60)
  params = agent.learner.online.clone()
  for restore in ('state', 'checkpoint', 'directory'):
    agent2, tr2 = _trainer()
    if restore == 'state':
      tr2.set_state(state)
    elif restore == 'checkpoint':
      tr2.load_checkpoint(str(tmp_path / 'ckpt'))
    else:   # through reporting.DirectoryCheckpoint, as a run driver registers the trainer
      cp = reporting.DirectoryCheckpoint(str(tmp_path / 'dir'))
      cp.state.trainer = tr2
      cp.restore()
    env2 = environments.VectorCatch(E, 21)
    env2.set_state(env_state)
    _, again = _drive(tr2, env2, (env2.frames,) + record, 60)
    np.testing.assert_array_equal(rest, again)
    assert torch.equal(agent2.learner.online, params), restore


def test_mismatched_checkpoints_raise_naming_dueling(tmp_path):
  dueling, _ = _agent('double_q', capacity=600)
  plain, _ = _agent('double_q', capacity=600, dueling=False)
  dueling.save_checkpoint(str(tmp_path / 'dueling'))
  plain.save_checkpoint(str(tmp_path / 'plain'))
  with pytest.raises(ValueError, match='dueling'):
    plain.load_checkpoint(str(tmp_path / 'dueling'))
  with pytest.raises(ValueError, match='dueling'):
    dueling.load_checkpoint(str(tmp_path / 'plain'))
  # a checkpoint written before the field existed (no 'dueling' key) loads as the plain network
  import os
  import pickle
  path = os.path.join(str(tmp_path / 'plain'), 'agent.pkl')
  with open(path, 'rb') as f:
    state = pickle.load(f)
  del state['dueling']
  with open(path, 'wb') as f:
    pickle.dump(state, f)
  plain.load_checkpoint(str(tmp_path / 'plain'))
  with pytest.raises(ValueError, match='dueling'):
    dueling.load_checkpoint(str(tmp_path / 'plain'))


def test_vector_evaluator_state_round_trip():
  from dqn_zoo_b200 import agent as ag
  from dqn_zoo_b200 import environments
  E, cut, ticks = 16, 40, 90
  agent, _ = _agent('dqn', capacity=600)
  agent.learner.init_params(9)
  ev = ag.VectorEvaluator(agent.learner, E, 0.05, [0, 3])
  ev.network_params = agent.learner
  env = environments.VectorCatch(E, 7)
  out = env.reset()
  out, _ = _drive(ev, env, out, cut)
  state, env_state, record = copy.deepcopy(ev.get_state()), env.get_state(), out[1:]
  _, rest = _drive(ev, env, out, ticks - cut)
  fresh = ag.VectorEvaluator(agent.learner, E, 0.05, [0, 3])
  fresh.set_state(state)
  env2 = environments.VectorCatch(E, 7)
  env2.set_state(env_state)
  _, again = _drive(fresh, env2, (env2.frames,) + record, ticks - cut)
  np.testing.assert_array_equal(rest, again)
  np.testing.assert_array_equal(ev.episode_return, fresh.episode_return)


# ---- learning --------------------------------------------------------------------------------------------------------
LEARNING_FRAMES = 1_500_000
LEARNING_THRESHOLD = 9.8          # test_munchausen_learns_catch's bar, at its frame budget


def test_dueling_double_q_learns_catch():
  """32 Catch streams for LEARNING_FRAMES frames, then >= 50 evaluation episodes at epsilon 0.01."""
  import importlib
  import os
  import sys
  here = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools')
  if here not in sys.path:
    sys.path.insert(0, here)
  bench_env = importlib.import_module('bench_env')
  curve = bench_env.learning_run(LEARNING_FRAMES, seed=0, kind='double_q', dueling=True)
  frames, ret, episodes, _ = curve[-1]
  print('dueling double_q catch curve', curve)
  assert frames >= LEARNING_FRAMES and episodes >= 50
  assert ret >= LEARNING_THRESHOLD, curve
