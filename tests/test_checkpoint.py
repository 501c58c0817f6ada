"""CPU: checkpoint directories (DESIGN.md §9) — the chunk digest's host twin against the numpy restatement in
oracle/checkpoint_oracle.py, `reporting.DirectoryCheckpoint` (round trip, generations, an interrupted save), host
array files and their corruption, and manifest validation."""

import os

import numpy as np
import pytest

from dqn_zoo_b200 import checkpoint as ck
from dqn_zoo_b200 import reporting
from oracle import checkpoint_oracle as co


@pytest.mark.parametrize('n', [0, 1, 7, 8, 9, 15, 16, 17, 63, 64, 65, 1000, 28224, 4097 * 8 + 3])
def test_digest_host_twin_equals_the_oracle(n):
  rs = np.random.RandomState(n)
  for data in (rs.randint(0, 256, size=n).astype(np.uint8), np.zeros(n, np.uint8), np.full(n, 255, np.uint8)):
    assert ck.digest_host(data) == co.digest(data.tobytes())


def test_digest_separates_length_position_and_content():
  base = np.arange(64, dtype=np.uint8)
  d = ck.digest_host(base)
  assert ck.digest_host(base[:63]) != d                         # trailing zero byte vs shorter range
  assert ck.digest_host(np.concatenate([base, [0]]).astype(np.uint8)) != d
  swapped = base.copy()
  swapped[[0, 8]] = swapped[[8, 0]]                             # same bytes, two words exchanged
  assert ck.digest_host(swapped) != d
  for k in (0, 31, 63):
    flipped = base.copy()
    flipped[k] ^= 1
    assert ck.digest_host(flipped) != d


class FakeCheckpointable:
  """Stands in for an agent or replay: state written into, and read back from, its own subdirectory."""

  def __init__(self, value):
    self.value = value

  def save_checkpoint(self, directory):
    os.makedirs(directory, exist_ok=True)
    with open(os.path.join(directory, 'value.txt'), 'w') as f:
      f.write(repr(self.value))

  def load_checkpoint(self, directory):
    with open(os.path.join(directory, 'value.txt')) as f:
      self.value = eval(f.read())


def _registered(path, value, seed):
  cp = reporting.DirectoryCheckpoint(str(path))
  cp.state.iteration = value
  cp.state.agent = FakeCheckpointable([value, 'x'])
  cp.state.random_state = np.random.RandomState(seed)
  cp.state.writer = reporting.CsvWriter(str(path) + '.csv')
  return cp


def test_directory_checkpoint_round_trip_and_generations(tmp_path):
  path = tmp_path / 'ck'
  cp = _registered(path, 3, 5)
  assert not cp.can_be_restored()
  cp.state.random_state.uniform(size=7)
  want_draw = np.random.RandomState(5)
  want_draw.uniform(size=7)
  cp.save()
  assert cp.can_be_restored()
  cp.state.iteration = 4
  cp.save()                                                     # second generation replaces the first
  assert sorted(n for n in os.listdir(path) if n.startswith('gen-')) == ['gen-000002']
  assert open(path / 'LATEST').read().strip() == 'gen-000002'

  fresh = _registered(path, 0, 99)
  assert fresh.can_be_restored()
  agent, rs = fresh.state.agent, fresh.state.random_state
  fresh.restore()
  assert fresh.state.iteration == 4
  assert fresh.state.agent is agent and agent.value == [3, 'x']        # restored in place, from its own directory
  assert fresh.state.random_state is rs and rs.uniform() == want_draw.uniform()


def test_interrupted_save_leaves_the_previous_generation_restorable(tmp_path, monkeypatch):
  path = tmp_path / 'ck'
  cp = _registered(path, 1, 0)
  cp.save()

  def interrupted(self, gen):
    raise KeyboardInterrupt('interrupted before the LATEST switch')
  monkeypatch.setattr(reporting.DirectoryCheckpoint, '_publish', interrupted)
  cp.state.iteration = 2
  cp.state.agent.value = [2, 'y']
  with pytest.raises(KeyboardInterrupt):
    cp.save()
  assert len([n for n in os.listdir(path) if n.startswith('gen-')]) == 2   # the new generation's files exist

  fresh = _registered(path, 0, 0)
  fresh.restore()
  assert fresh.state.iteration == 1 and fresh.state.agent.value == [1, 'x']
  monkeypatch.undo()
  cp.save()                                                     # the next save cleans the abandoned generation up
  assert sorted(n for n in os.listdir(path) if n.startswith('gen-')) == ['gen-000003']
  fresh.restore()
  assert fresh.state.iteration == 2 and fresh.state.agent.value == [2, 'y']


def test_restore_needs_a_registered_object(tmp_path):
  cp = _registered(tmp_path / 'ck', 1, 0)
  cp.save()
  other = reporting.DirectoryCheckpoint(str(tmp_path / 'ck'))
  with pytest.raises(KeyError):
    other.restore()
  with pytest.raises(FileNotFoundError):
    reporting.DirectoryCheckpoint(str(tmp_path / 'none')).restore()


def test_host_array_files_and_their_corruption(tmp_path):
  a = np.arange(5000, dtype=np.int64).reshape(-1, 2) * 7 - 3
  entry = ck.Transfer.save_host(str(tmp_path / 'a.bin'), a)
  got = ck.Transfer.load_host(str(tmp_path / 'a.bin'), entry)
  assert got.dtype == a.dtype and np.array_equal(got, a)
  raw = bytearray(open(tmp_path / 'a.bin', 'rb').read())
  raw[12345] ^= 0x10
  open(tmp_path / 'b.bin', 'wb').write(bytes(raw))
  with pytest.raises(RuntimeError, match=r'b\.bin: chunk 0 digest'):
    ck.Transfer.load_host(str(tmp_path / 'b.bin'), entry)
  open(tmp_path / 'c.bin', 'wb').write(bytes(raw[:-8]))
  with pytest.raises(RuntimeError, match='truncated'):
    ck.Transfer.load_host(str(tmp_path / 'c.bin'), entry)
  with pytest.raises(RuntimeError, match='missing'):
    ck.Transfer.load_host(str(tmp_path / 'd.bin'), entry)


def test_manifest_validation_errors(tmp_path):
  want = {'version': 1, 'kind': 'TransitionReplay', 'layout': 'frames', 'capacity': 1000, 'frame_capacity': 2064}
  saved = dict(want, format='dqn_zoo_b200.replay', files={})
  ck.write_json(str(tmp_path / ck.MANIFEST), saved)
  m = ck.read_manifest(str(tmp_path), 'dqn_zoo_b200.replay')
  ck.validate(m, want, 'here')
  for key, other in [('version', 2), ('kind', 'PrioritizedTransitionReplay'), ('layout', 'rows'), ('capacity', 999),
                     ('frame_capacity', None)]:
    with pytest.raises(ValueError, match=key):
      ck.validate(dict(m, **{key: other}), want, 'here')
  with pytest.raises(ValueError, match='not a dqn_zoo_b200.agent checkpoint'):
    ck.read_manifest(str(tmp_path), 'dqn_zoo_b200.agent')
  with pytest.raises(ValueError, match='not a readable'):
    ck.read_manifest(str(tmp_path / 'missing'), 'dqn_zoo_b200.replay')
  (tmp_path / 'bad').mkdir()
  (tmp_path / 'bad' / ck.MANIFEST).write_text('{"format": "dqn_zoo_b200.replay", ')
  with pytest.raises(ValueError, match='not a readable'):
    ck.read_manifest(str(tmp_path / 'bad'), 'dqn_zoo_b200.replay')
