"""Run-loop reporting and persistence around the agent surface (SURVEY §8(f) #4; reference `dqn_zoo/parts.py`).

Behavioural contract kept from the reference so that its plotting notebook and run drivers work unchanged:
  * `generate_statistics(trackers, sequence)` — parts.py:125-146: reset every tracker, feed every
    `(environment, timestep, agent, action)` item, merge the trackers' dicts (first tracker wins on key clashes,
    as `collections.ChainMap` does).
  * `EpisodeTracker` — parts.py:149-247: the seven keys `mean_episode_return, current_episode_return, episode_return,
    num_episodes, num_steps_over_episodes, current_episode_step, num_steps_since_reset` with the same conventions
    (`episode_return` falls back to the running return until one episode has completed; NaN before any step).
  * `StepRateTracker` — parts.py:250-287: `step_rate, num_steps, duration`.
  * `UnbiasedExponentialWeightedAverageAgentTracker` — parts.py:290-333 (Sutton & Barto's unbiased constant-step-size
    trick on `agent.statistics`).
  * `CsvWriter` / `NullWriter` — parts.py:448-504: one header row from the first dict's keys, append mode, resumable.
  * `NullCheckpoint` / `AttributeDict` — parts.py:507-541.  `FileCheckpoint` is the working implementation behind the
    same three methods (`save`, `can_be_restored`, `restore`) that the reference leaves as a placeholder;
    `DirectoryCheckpoint` is the same surface over a directory, for agents and replays too large to pickle.

Everything here is host-side bookkeeping; the GPU is touched only through the registered objects, and to read the free
device memory when `DirectoryCheckpoint.save(blocking=False)` has no explicit budget."""

import collections
import csv
import math
import os
import pickle
import shutil
import tempfile
import threading
import timeit
import traceback
from typing import Any, Iterable, Mapping, Optional, Sequence


def generate_statistics(trackers: Sequence[Any], timestep_action_sequence: Iterable[Any]) -> Mapping[str, Any]:
  for t in trackers:
    t.reset()
  for environment, timestep, agent, action in timestep_action_sequence:
    for t in trackers:
      t.step(environment, timestep, agent, action)
  merged = {}
  for t in reversed(list(trackers)):     # earlier trackers take precedence, like ChainMap(*dicts)
    merged.update(t.get())
  return merged


class EpisodeTracker:
  """Episode returns and step counts."""

  def __init__(self):
    self._ready = False

  def reset(self) -> None:
    self._ready = True
    self._steps = 0                # num_steps_since_reset
    self._steps_in_done = 0        # num_steps_over_episodes
    self._returns = []             # completed episodes
    self._rewards = []             # rewards of the episode in progress
    self._episode_step = 0

  def step(self, environment, timestep, agent, action) -> None:
    del environment, agent, action
    if not self._ready:
      raise RuntimeError('reset() must be called before first call to step().')
    if timestep.first():
      if self._rewards:
        raise ValueError('Current episode reward list should be empty.')
      if self._episode_step != 0:
        raise ValueError('Current episode step should be zero.')
    else:
      self._rewards.append(timestep.reward)
    self._steps += 1
    self._episode_step += 1
    if timestep.last():
      self._returns.append(sum(self._rewards))
      self._rewards = []
      self._steps_in_done += self._episode_step
      self._episode_step = 0

  def get(self) -> Mapping[str, Any]:
    if not self._ready:
      raise RuntimeError('reset() must be called before first call to get().')
    running = sum(self._rewards)
    if self._returns:
      mean = sum(self._returns) / len(self._returns)
      current, shown = running, mean
    else:
      mean = math.nan
      current = running if self._steps > 0 else math.nan
      shown = current
    return {
        'mean_episode_return': mean,
        'current_episode_return': current,
        'episode_return': shown,
        'num_episodes': len(self._returns),
        'num_steps_over_episodes': self._steps_in_done,
        'current_episode_step': self._episode_step,
        'num_steps_since_reset': self._steps,
    }


class StepRateTracker:
  """Steps per second since the last reset."""

  def __init__(self):
    self._steps = None
    self._t0 = None

  def reset(self) -> None:
    self._steps = 0
    self._t0 = timeit.default_timer()

  def step(self, environment, timestep, agent, action) -> None:
    del environment, timestep, agent, action
    self._steps += 1

  def get(self) -> Mapping[str, float]:
    if self._steps is None:
      raise RuntimeError('reset() must be called before first call to get().')
    duration = timeit.default_timer() - self._t0
    return {'step_rate': self._steps / duration if self._steps > 0 else math.nan, 'num_steps': self._steps,
            'duration': duration}


class UnbiasedExponentialWeightedAverageAgentTracker:
  """Bias-corrected exponential average of `agent.statistics` (a flat mapping of floats)."""

  def __init__(self, step_size: float, initial_agent):
    self._initial = dict(initial_agent.statistics)
    self._alpha = step_size
    self.reset()

  def reset(self) -> None:
    self.trace = 0.0
    self._avg = dict(self._initial)

  def step(self, environment, timestep, agent, action) -> None:
    del environment, timestep, action
    self.trace = (1 - self._alpha) * self.trace + self._alpha
    beta = self._alpha / self.trace
    assert 0 <= beta <= 1
    stats = agent.statistics
    if beta == 1:
      self._avg = dict(stats)
    else:
      self._avg = {k: (1 - beta) * self._avg[k] + beta * stats[k] for k in self._avg}

  def get(self) -> Mapping[str, float]:
    return self._avg


def make_default_trackers(initial_agent) -> Sequence[Any]:
  return [EpisodeTracker(), StepRateTracker(),
          UnbiasedExponentialWeightedAverageAgentTracker(step_size=1e-3, initial_agent=initial_agent)]


class NullWriter:
  def write(self, *args, **kwargs) -> None:
    pass

  def close(self) -> None:
    pass


class CsvWriter:
  """Appends one row per `write(OrderedDict)`; the first call fixes the columns."""

  def __init__(self, fname: str):
    folder = os.path.dirname(fname)
    if folder and not os.path.exists(folder):
      os.makedirs(folder)
    self._fname = fname
    self._header_written = False
    self._fieldnames = None

  def write(self, values: Mapping[str, Any]) -> None:
    if self._fieldnames is None:
      self._fieldnames = list(values.keys())
    with open(self._fname, 'a', newline='') as f:
      w = csv.DictWriter(f, fieldnames=self._fieldnames)
      if not self._header_written:
        w.writeheader()
        self._header_written = True
      w.writerow(values)

  def close(self) -> None:
    pass

  def get_state(self) -> Mapping[str, Any]:
    return {'header_written': self._header_written, 'fieldnames': self._fieldnames}

  def set_state(self, state: Mapping[str, Any]) -> None:
    self._header_written = state['header_written']
    self._fieldnames = state['fieldnames']


class AttributeDict(dict):
  """dict with attribute access (`state.iteration = 3`)."""

  def __getattr__(self, key):
    try:
      return self[key]
    except KeyError as e:
      raise AttributeError(key) from e

  def __setattr__(self, key, value):
    self[key] = value

  def __delattr__(self, key):
    del self[key]


class NullCheckpoint:
  """Checkpointing disabled: same surface, no effect."""

  def __init__(self):
    self.state = AttributeDict()

  def save(self) -> None:
    pass

  def can_be_restored(self) -> bool:
    return False

  def restore(self) -> None:
    pass


class FileCheckpoint:
  """Working checkpoint behind NullCheckpoint's interface.

  The run driver registers live objects in `checkpoint.state` (`state.train_agent = agent`, `state.iteration = 0`,
  `state.random_state = np.random.RandomState(...)`, `state.writer = CsvWriter(...)`, as dqn/run_atari.py:237-256 does).
  `save()` pickles a snapshot — `get_state()` of every entry that has one (agents, replay, writers), numpy
  `RandomState.get_state()` for random states, the value itself otherwise — atomically (write + rename).
  `restore()` pushes the snapshot back INTO the registered objects (`set_state`) and overwrites plain values, so the
  objects the driver already holds continue from the checkpoint."""

  def __init__(self, path: str):
    self._path = path
    self.state = AttributeDict()

  @staticmethod
  def _snapshot(value):
    if hasattr(value, 'get_state') and hasattr(value, 'set_state'):
      return ('stateful', value.get_state())
    return ('value', value)

  def save(self) -> None:
    payload = {k: self._snapshot(v) for k, v in self.state.items()}
    folder = os.path.dirname(os.path.abspath(self._path))
    os.makedirs(folder, exist_ok=True)
    fd, tmp = tempfile.mkstemp(dir=folder, suffix='.tmp')
    try:
      with os.fdopen(fd, 'wb') as f:
        pickle.dump(payload, f, protocol=pickle.HIGHEST_PROTOCOL)
      os.replace(tmp, self._path)
    except BaseException:
      if os.path.exists(tmp):
        os.remove(tmp)
      raise

  def can_be_restored(self) -> bool:
    return os.path.exists(self._path)

  def restore(self) -> None:
    with open(self._path, 'rb') as f:
      payload = pickle.load(f)
    _apply(self.state, payload)


def _fsync(path):
  fd = os.open(path, os.O_RDONLY)
  try:
    os.fsync(fd)
  finally:
    os.close(fd)


def _apply(state, payload):
  for key, (kind, value) in payload.items():
    if kind == 'stateful':
      if key not in state:
        raise KeyError('checkpoint entry %r has no registered object to restore into' % key)
      state[key].set_state(value)
    else:
      state[key] = value


class DirectoryCheckpoint:
  """Checkpoint directory behind NullCheckpoint's interface, for state too large to pickle in one piece (DESIGN.md §9).

  Entries of `state` with `save_checkpoint` / `load_checkpoint` (agents, replays, `VectorTrainer`) write into a
  subdirectory of their own; every other entry is pickled as `FileCheckpoint` pickles it, into `state.pkl`.  Each
  `save()` writes a new generation directory `gen-<n>` and fsyncs it, then switches the `LATEST` file to it by
  write-and-rename, and only then removes the older generations: a save interrupted at any point leaves the previous
  checkpoint restorable.

  `save(blocking=False)` snapshots instead: every directory entry's `snapshot_checkpoint()` (device copies taken on the
  current CUDA stream) and the pickle of the other entries are taken at the call, which then returns; one background
  thread (not a daemon, so interpreter exit waits for it) writes the generation from the snapshots, fsyncs it,
  switches `LATEST` and prunes, in the blocking save's order.  One save is in flight at a time: `save`, `restore` and
  `wait` first wait for it, and re-raise its exception if it failed (its partial generation is removed; `LATEST`
  still names the previous one).  When the snapshots would not fit in `snapshot_budget` bytes of device memory
  (default: the free device memory plus what the caching allocator holds unused, less `SNAPSHOT_MARGIN`), or an
  entry can save but not snapshot, that save is blocking."""

  LATEST = 'LATEST'
  SNAPSHOT_MARGIN = 2 << 30

  def __init__(self, path: str, snapshot_budget: Optional[int] = None):
    self._path = path
    self.state = AttributeDict()
    self.snapshot_budget = snapshot_budget
    self._writer = None            # the background save's thread
    self._error = None             # its exception, re-raised by the next wait()

  def _latest(self) -> Optional[str]:
    try:
      with open(os.path.join(self._path, self.LATEST)) as f:
        name = f.read().strip()
    except OSError:
      return None
    return name if name and os.path.isdir(os.path.join(self._path, name)) else None

  def save(self, blocking: bool = True) -> str:
    """Writes a new generation; returns 'blocking' or 'background', the mode used (see the class)."""
    self.wait()
    os.makedirs(self._path, exist_ok=True)
    if not blocking and self._can_snapshot():
      self._save_background()
      return 'background'
    gen = self._write_generation()
    self._publish(gen)
    self._prune(gen)
    return 'blocking'

  def wait(self) -> None:
    """Returns when no save is in flight; raises the exception of a background save that failed."""
    if self._writer is not None:
      self._writer.join()
      self._writer = None
    if self._error is not None:
      error, self._error = self._error, None
      raise error

  def _directory_entries(self):
    return {k: v for k, v in self.state.items() if hasattr(v, 'save_checkpoint') and hasattr(v, 'load_checkpoint')}

  def _can_snapshot(self) -> bool:
    entries = self._directory_entries()
    if not all(hasattr(v, 'snapshot_checkpoint') for v in entries.values()):
      return False
    need = sum(int(v.snapshot_checkpoint_bytes()) for v in entries.values())
    return need <= self._snapshot_budget()

  def _snapshot_budget(self) -> int:
    if self.snapshot_budget is not None:
      return int(self.snapshot_budget)
    import torch
    free, _ = torch.cuda.mem_get_info()
    return free + torch.cuda.memory_reserved() - torch.cuda.memory_allocated() - self.SNAPSHOT_MARGIN

  def _next_generation(self) -> str:
    taken = [int(n[4:]) for n in os.listdir(self._path) if n.startswith('gen-') and n[4:].isdigit()]
    return 'gen-%06d' % (max(taken, default=0) + 1)

  def _prune(self, gen: str) -> None:
    for name in os.listdir(self._path):
      if name.startswith('gen-') and name != gen:
        shutil.rmtree(os.path.join(self._path, name), ignore_errors=True)

  def _write_generation(self) -> str:
    gen = self._next_generation()
    folder = os.path.join(self._path, gen)
    os.makedirs(folder)
    payload = {}
    for key, value in self.state.items():
      if hasattr(value, 'save_checkpoint') and hasattr(value, 'load_checkpoint'):
        value.save_checkpoint(os.path.join(folder, key))
        payload[key] = ('directory', key)
      else:
        payload[key] = FileCheckpoint._snapshot(value)
    self._finish(folder, pickle.dumps(payload, protocol=pickle.HIGHEST_PROTOCOL))
    return gen

  @staticmethod
  def _finish(folder: str, payload: bytes) -> None:
    with open(os.path.join(folder, 'state.pkl'), 'wb') as f:
      f.write(payload)
    for root, _, names in os.walk(folder):
      for name in names:
        _fsync(os.path.join(root, name))
      _fsync(root)

  def _save_background(self) -> None:
    snapshots, payload = {}, {}
    try:
      for key, value in self.state.items():
        if key in self._directory_entries():
          snapshots[key] = value.snapshot_checkpoint()
          payload[key] = ('directory', key)
        else:
          payload[key] = FileCheckpoint._snapshot(value)
      blob = pickle.dumps(payload, protocol=pickle.HIGHEST_PROTOCOL)
    except BaseException:
      for snap in snapshots.values():
        snap.release()
      raise
    self._writer = threading.Thread(target=self._write_background, args=(self._next_generation(), snapshots, blob),
                                    name='DirectoryCheckpoint-writer', daemon=False)
    self._writer.start()

  def _write_background(self, gen, snapshots, blob) -> None:
    folder = os.path.join(self._path, gen)
    try:
      os.makedirs(folder)
      for key, snap in snapshots.items():
        snap.write(os.path.join(folder, key))
      self._finish(folder, blob)
      self._publish(gen)
      self._prune(gen)
    except BaseException as e:     # kept for the next wait(); the previous generation stays the latest
      if self._latest() != gen:
        shutil.rmtree(folder, ignore_errors=True)
      traceback.clear_frames(e.__traceback__)      # the frames' locals would keep the snapshot's buffers alive
      self._error = e
    finally:
      for snap in snapshots.values():
        snap.release()

  def _publish(self, gen: str) -> None:
    tmp = os.path.join(self._path, self.LATEST + '.tmp')
    with open(tmp, 'w') as f:
      f.write(gen + '\n')
      f.flush()
      os.fsync(f.fileno())
    os.replace(tmp, os.path.join(self._path, self.LATEST))
    _fsync(self._path)

  def can_be_restored(self) -> bool:
    return self._latest() is not None

  def restore(self) -> None:
    self.wait()
    gen = self._latest()
    if gen is None:
      raise FileNotFoundError('no checkpoint generation under %s' % self._path)
    folder = os.path.join(self._path, gen)
    with open(os.path.join(folder, 'state.pkl'), 'rb') as f:
      payload = pickle.load(f)
    for key, (kind, value) in payload.items():
      if kind == 'directory':
        if key not in self.state:
          raise KeyError('checkpoint entry %r has no registered object to restore into' % key)
        self.state[key].load_checkpoint(os.path.join(folder, value))
    _apply(self.state, {k: v for k, v in payload.items() if v[0] != 'directory'})
