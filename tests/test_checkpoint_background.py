"""CPU: `reporting.DirectoryCheckpoint.save(blocking=False)` (DESIGN.md §9) with stand-in entries whose snapshots are
written slowly, held at a gate, or fail: `LATEST` names the previous generation until the write completes, a second
save and a restore wait for the first, a writer's exception surfaces at `wait()` with its partial generation removed,
the values pickled beside the snapshots are those of the call, and a budget too small for the snapshots makes the save
blocking."""

import os
import threading

import numpy as np
import pytest

from dqn_zoo_b200 import reporting


class FakeSnapshot:
  def __init__(self, owner, value):
    self.owner, self.value = owner, value
    self.device_bytes = owner.nbytes
    self.released = False

  def write(self, directory):
    if self.released:
      raise RuntimeError('write after release')
    if self.owner.gate is not None:
      self.owner.entered.set()
      assert self.owner.gate.wait(30), 'the test never opened the gate'
    if self.owner.fail is not None:
      os.makedirs(directory, exist_ok=True)
      with open(os.path.join(directory, 'partial.txt'), 'w') as f:
        f.write('half')
      raise self.owner.fail
    _write_value(directory, self.value)

  def release(self):
    self.released = True


def _write_value(directory, value):
  os.makedirs(directory, exist_ok=True)
  with open(os.path.join(directory, 'value.txt'), 'w') as f:
    f.write(repr(value))


class FakeSnapshottable:
  """Stands in for an agent or trainer: a subdirectory written by `save_checkpoint` or by a snapshot's `write`, which
  can be held at a gate or made to fail."""

  def __init__(self, value, nbytes=1000):
    self.value = value
    self.nbytes = nbytes
    self.gate = None
    self.entered = threading.Event()
    self.fail = None
    self.snapshots = []
    self.blocking_saves = 0

  def save_checkpoint(self, directory):
    self.blocking_saves += 1
    _write_value(directory, self.value)

  def load_checkpoint(self, directory):
    with open(os.path.join(directory, 'value.txt')) as f:
      self.value = eval(f.read())

  def snapshot_checkpoint(self):
    snap = FakeSnapshot(self, list(self.value))
    self.snapshots.append(snap)
    return snap

  def snapshot_checkpoint_bytes(self):
    return self.nbytes


def _registered(path, value, budget=1 << 40):
  cp = reporting.DirectoryCheckpoint(str(path), snapshot_budget=budget)
  cp.state.iteration = value
  cp.state.agent = FakeSnapshottable([value, 'x'])
  cp.state.random_state = np.random.RandomState(value)
  return cp


def _gens(path):
  return sorted(n for n in os.listdir(path) if n.startswith('gen-'))


def _latest(path):
  return open(os.path.join(path, 'LATEST')).read().strip()


def test_latest_switches_only_after_the_background_write(tmp_path):
  path = tmp_path / 'ck'
  cp = _registered(path, 1)
  assert cp.save() == 'blocking'
  agent = cp.state.agent
  agent.gate = threading.Event()
  cp.state.iteration = 2
  agent.value = [2, 'y']
  assert cp.save(blocking=False) == 'background'
  cp.state.iteration = 3                                       # changes after the call are not in the checkpoint
  agent.value = [3, 'z']
  assert agent.entered.wait(30)
  assert _latest(path) == 'gen-000001'                         # the new generation is still being written
  fresh = _registered(path, 0)
  fresh.restore()
  assert fresh.state.iteration == 1 and fresh.state.agent.value == [1, 'x']
  agent.gate.set()
  cp.wait()
  assert _latest(path) == 'gen-000002' and _gens(path) == ['gen-000002']
  assert agent.snapshots[-1].released and agent.blocking_saves == 1
  fresh.restore()
  assert fresh.state.iteration == 2 and fresh.state.agent.value == [2, 'y']


def test_a_second_save_and_a_restore_wait_for_the_first(tmp_path):
  path = tmp_path / 'ck'
  cp = _registered(path, 1)
  agent = cp.state.agent
  agent.gate = threading.Event()
  assert cp.save(blocking=False) == 'background'
  assert agent.entered.wait(30)
  done = []

  def second():
    cp.state.iteration = 2
    done.append(cp.save(blocking=False))
  t = threading.Thread(target=second)
  t.start()
  t.join(0.5)
  assert t.is_alive() and not done                             # the second save is waiting
  assert len(agent.snapshots) == 1                             # and has not snapshotted: one snapshot at a time
  agent.gate.set()
  t.join(30)
  assert done == ['background']
  cp.state.iteration = 7
  cp.restore()                                                  # waits for the second save, then reads it
  assert _latest(path) == 'gen-000002' and _gens(path) == ['gen-000002']
  assert cp.state.iteration == 2
  assert all(s.released for s in agent.snapshots)


def test_writer_error_surfaces_at_wait_and_removes_the_partial_generation(tmp_path):
  path = tmp_path / 'ck'
  cp = _registered(path, 1)
  cp.save()
  agent = cp.state.agent
  agent.fail = OSError('disk full')
  cp.state.iteration = 2
  assert cp.save(blocking=False) == 'background'
  with pytest.raises(OSError, match='disk full'):
    cp.wait()
  cp.wait()                                                     # raised once
  assert _gens(path) == ['gen-000001'] and _latest(path) == 'gen-000001'
  assert agent.snapshots[-1].released
  fresh = _registered(path, 0)
  fresh.restore()
  assert fresh.state.iteration == 1 and fresh.state.agent.value == [1, 'x']


@pytest.mark.parametrize('then', ['save', 'restore'])
def test_writer_error_surfaces_at_the_next_save_or_restore(tmp_path, then):
  path = tmp_path / 'ck'
  cp = _registered(path, 1)
  cp.save()
  cp.state.agent.fail = RuntimeError('writer failed')
  cp.save(blocking=False)
  with pytest.raises(RuntimeError, match='writer failed'):
    getattr(cp, then)()
  cp.state.agent.fail = None
  cp.state.iteration = 5
  cp.save(blocking=False)
  cp.wait()
  assert _gens(path) == ['gen-000002']
  fresh = _registered(path, 0)
  fresh.restore()
  assert fresh.state.iteration == 5


def test_a_budget_too_small_makes_the_save_blocking(tmp_path):
  path = tmp_path / 'ck'
  cp = _registered(path, 1, budget=0)
  assert cp.save(blocking=False) == 'blocking'
  agent = cp.state.agent
  assert agent.blocking_saves == 1 and not agent.snapshots
  cp.snapshot_budget = agent.nbytes                             # exactly enough
  cp.state.iteration = 2
  assert cp.save(blocking=False) == 'background'
  cp.wait()
  assert agent.blocking_saves == 1 and len(agent.snapshots) == 1
  fresh = _registered(path, 0)
  fresh.restore()
  assert fresh.state.iteration == 2


def test_an_entry_that_cannot_snapshot_makes_the_save_blocking(tmp_path):
  class SaveOnly:
    def __init__(self):
      self.saves = 0

    def save_checkpoint(self, directory):
      self.saves += 1
      _write_value(directory, 'only')

    def load_checkpoint(self, directory):
      pass
  path = tmp_path / 'ck'
  cp = _registered(path, 1)
  cp.state.other = SaveOnly()
  assert cp.save(blocking=False) == 'blocking'
  assert cp.state.other.saves == 1 and not cp.state.agent.snapshots


def test_the_writer_thread_is_not_a_daemon(tmp_path):
  cp = _registered(tmp_path / 'ck', 1)
  agent = cp.state.agent
  agent.gate = threading.Event()
  cp.save(blocking=False)
  assert agent.entered.wait(30)
  writers = [t for t in threading.enumerate() if t.name == 'DirectoryCheckpoint-writer']
  assert writers and not any(t.daemon for t in writers)
  agent.gate.set()
  cp.wait()
