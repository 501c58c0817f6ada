"""CPU: the frame-pool model (oracle/frame_pool_oracle.py) on hand-built frame-stack streams: plane counts the
dedup rules imply, eviction and reuse of planes, and the invariants the device pool is checked against."""

import numpy as np
import pytest

from oracle import frame_pool_oracle as fpo
from oracle import replay_oracle as ro

OBS = (6, 8, 4)


def _run(capacity, transitions, frame_capacity=None, obs_shape=OBS):
  model = fpo.DedupReplayModel(capacity, obs_shape, frame_capacity or 2 * capacity + 64)
  stored = {}
  for k, tr in enumerate(transitions):
    model.add(tr.s_tm1, tr.s_t)
    stored[k % capacity] = (tr.s_tm1, tr.s_t)
  _check_invariants(model, stored)
  return model


def _check_invariants(model, stored):
  pool = model.pool
  slots = model.live_slots()
  # refcounts: 2 * channels references per live row, plus plane 0's permanent one
  assert pool.refcount.sum() - 1 == 2 * pool.channels * len(slots)
  want = np.bincount(pool.planes[slots].reshape(-1), minlength=pool.frame_capacity)
  want[0] += 1
  np.testing.assert_array_equal(pool.refcount, want)
  # live planes are pairwise distinct, and free stack + live planes partition the pool
  live = pool.live_planes()
  assert len({pool.bytes_of[p] for p in live}) == len(live)
  assert sorted(live + pool.free) == list(range(pool.frame_capacity))
  assert pool.frames_in_use == len(live)
  # reconstructed bytes equal the inputs
  for s in slots:
    a, b = pool.reconstruct(s)
    np.testing.assert_array_equal(a, stored[s][0])
    np.testing.assert_array_equal(b, stored[s][1])


def _episode_transitions(n, episodes, seed=0, static=False):
  rs = np.random.RandomState(seed)
  acc = ro.NStepTransitionAccumulator(n)
  out = []
  for length in episodes:
    for ts in fpo.stacked_episode(rs, length, OBS, static=static):
      out.extend(acc.step(ts, int(rs.randint(0, 6))))
  return out


@pytest.mark.parametrize('T', [1, 2, 3, 4, 9])
def test_one_step_episode_uses_transitions_plus_two_planes(T):
  trs = _episode_transitions(1, [T])
  assert len(trs) == T
  model = _run(64, trs)
  assert model.pool.frames_in_use == T + 2            # T + 1 frames and plane 0


def test_nstep3_last_flush_adds_no_planes():
  for T in (1, 2, 5, 8):
    trs = _episode_transitions(3, [T])
    assert _run(64, trs).pool.frames_in_use == T + 2
    if T >= 3:   # the first transition emitted at LAST brings the last frame; the two flushed after it add nothing
      assert _run(64, trs[:-2]).pool.frames_in_use == T + 2


def test_interleaved_streams_and_static_frames_share_planes():
  rs = np.random.RandomState(3)
  lengths = [[5, 3], [7], [2, 2, 2]]
  episodes = [[fpo.stacked_episode(rs, L, OBS) for L in ls] for ls in lengths]
  trs = fpo.interleave_episodes(rs, [ro.NStepTransitionAccumulator(1) for _ in lengths], episodes)
  model = _run(256, trs)
  assert model.pool.frames_in_use == sum(L + 1 for ls in lengths for L in ls) + 1
  static = _episode_transitions(1, [12], seed=4, static=True)
  assert _run(64, static).pool.frames_in_use == 2       # plane 0 and the one screen


def test_eviction_wraps_and_frees_planes():
  trs = _episode_transitions(1, [40, 15], seed=5)
  model = _run(6, trs)
  # the 6 newest transitions are steps 9..14 of the second episode: 6 new frames + the 4 of the first s_tm1 + plane 0
  assert model.pool.frames_in_use == 6 + 4 + 1
  assert model.t == 55 and max(model.pool.planes.reshape(-1)) < 6 * 2 + 64
  # planes freed by eviction are handed out again (LIFO): ids stay small however long the stream runs
  more = _episode_transitions(1, [200], seed=6)
  model2 = _run(6, more)
  assert max(model2.pool.planes.reshape(-1)) <= 6 + 4 + 1


def test_capacity_below_stack_depth():
  trs = _episode_transitions(3, [7, 1, 4], seed=7)
  model = _run(2, trs)
  assert model.pool.frames_in_use <= 2 * 2 * OBS[2] + 1


def test_pool_exhaustion_maps_to_plane_zero():
  rs = np.random.RandomState(8)
  model = fpo.DedupReplayModel(4, OBS, 5)
  for _ in range(3):
    model.add(rs.randint(1, 256, size=OBS).astype(np.uint8), rs.randint(1, 256, size=OBS).astype(np.uint8))
  assert model.pool.full and model.pool.frames_in_use == 5
  assert (model.pool.planes[1:3] == 0).all()


def test_synthetic_stacked_rows_are_frame_stacks():
  obs, a, r, d = fpo.synthetic_stacked_rows(9, np.arange(12), OBS, 5, 6)
  o = obs.reshape(12, 2, *OBS)
  np.testing.assert_array_equal(o[:-1, 1][np.arange(11) % 5 != 4], o[1:, 0][np.arange(11) % 5 != 4])
  assert (o[0, 0][:, :, 1:] == 0).all() and (o[0, 1][:, :, 2:] == 0).all() and (o[5, 0][:, :, 1:] == 0).all()
  model = _run(12, [ro.Transition(o[i, 0], 0, 0.0, 0.0, o[i, 1]) for i in range(12)])
  assert model.pool.frames_in_use == 12 + 3 + 1       # n + episodes distinct frames, plane 0
  # plane ids in order of first appearance: frame f of episode e is plane 1 + e * (L + 1) + f
  assert model.pool.planes[7, 4 + 3] == 1 + 1 * 6 + 3 and model.pool.planes[0, 0] == 1
  _, a2, r2, d2 = ro.synthetic_rows(9, np.arange(12), 8, 6)
  np.testing.assert_array_equal(a, a2)
