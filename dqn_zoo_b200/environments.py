"""Games at Atari geometry, simulated and rendered on the device: Catch (csrc/dz_catch.cu; rules in DESIGN.md §10),
Breakout (csrc/dz_breakout.cu; DESIGN.md §11) and Pong (csrc/dz_pong.cu; DESIGN.md §12).

`VectorCatch` / `VectorBreakout` / `VectorPong` step E streams of a game with one kernel launch per tick and leave their 210x160x3 RGB
frames in a device tensor, where `agent.VectorTrainer.step` / `agent.VectorEvaluator.step` read them in place: the
whole loop (environment -> preprocess -> act -> insert -> learn) stays on the GPU but for the actions and a small
per-stream record.  `Catch` / `Breakout` / `Pong` are one stream with the reference's dm_env surface, for `parts.run_loop` and
the one-stream agents.
"""

import ctypes as C
from typing import Any, Mapping, Optional

import numpy as np
import torch

from dqn_zoo_b200 import _lib
from dqn_zoo_b200 import parts

HEIGHT, WIDTH = 210, 160


def _check_arguments(num_streams, seed, num_actions, min_noop_steps, max_noop_steps, stream_offset, max_streams,
                     min_actions, max_noops, noop_reason):
  """Raises ValueError for arguments a game's C ABI would refuse; returns E."""
  E = int(num_streams)
  if not 1 <= E <= max_streams:
    raise ValueError('num_streams must be in [1, %d], got %d' % (max_streams, E))
  if not min_actions <= num_actions <= 18:
    raise ValueError('num_actions must be in [%d, 18], got %d' % (min_actions, num_actions))
  if not 0 <= min_noop_steps <= max_noop_steps:
    raise ValueError('need 0 <= min_noop_steps <= max_noop_steps, got %d, %d' % (min_noop_steps, max_noop_steps))
  if max_noop_steps > max_noops:
    raise ValueError('max_noop_steps %d > %d: %s during the no-op frames of a reset'
                     % (max_noop_steps, max_noops, noop_reason))
  if not 0 <= seed < 2 ** 32:
    raise ValueError('seed must be in [0, 2^32)')
  if stream_offset < 0 or stream_offset + E > 2 ** 32:
    raise ValueError('stream_offset + num_streams must be in [0, 2^32]')
  return E


class _VectorGame:
  """The host side shared by the device games: a configuration struct, the int32 [fields][E] device state, the frames
  tensor, pinned control and record buffers, and the tick, state and render calls of one game's C ABI."""

  _STEP = _RENDER = None           # the game's dz_<game>_step / dz_<game>_render
  _FIELDS = ()                     # its state fields, in the order of the device arrays

  def _setup(self, cfg, device):
    E = cfg.num_streams
    self._cfg = cfg
    self._E = E
    self._device = torch.device(device)
    F = len(self._FIELDS)
    self._state = torch.zeros((F, E), dtype=torch.int32, device=self._device)
    self._state[self._FIELDS.index('over')] = 1                # the first tick of every stream is a reset
    self._frames = torch.zeros((E, HEIGHT, WIDTH, 3), dtype=torch.uint8, device=self._device)
    self._control = torch.zeros((2, E), dtype=torch.int32, device=self._device)
    self._record = torch.zeros((4, E), dtype=torch.int32, device=self._device)
    self._control_host = torch.zeros((2, E), dtype=torch.int32).pin_memory()
    self._record_host = torch.zeros((4, E), dtype=torch.int32).pin_memory()

  def reset(self, stream=None):
    """A new episode in every stream."""
    control = self._control_host.numpy()
    control[0] = 0
    control[1] = 1
    return self._tick(stream)

  def step(self, actions, reset=None, stream=None):
    """actions: int [E] in [0, num_actions) (ignored for the streams that reset); reset: bool [E] or None."""
    actions = np.asarray(actions)
    if actions.shape != (self._E,):
      raise ValueError('actions must have shape (%d,), got %s' % (self._E, actions.shape))
    control = self._control_host.numpy()
    control[0] = actions
    if reset is None:
      control[1] = 0
    else:
      reset = np.asarray(reset, bool)
      if reset.shape != (self._E,):
        raise ValueError('reset must have shape (%d,), got %s' % (self._E, reset.shape))
      control[1] = reset
    return self._tick(stream)

  def _tick(self, stream):
    s = torch.cuda.current_stream(self._device) if stream is None else stream
    _lib.call(self._STEP, C.byref(self._cfg), self._state.data_ptr(), self._control_host.data_ptr(),
              self._control.data_ptr(), self._frames.data_ptr(), self._record.data_ptr(), self._record_host.data_ptr(),
              s.cuda_stream)
    s.synchronize()
    rec = self._record_host.numpy()
    step_type = rec[0].astype(np.int64)
    first = step_type == int(parts.StepType.FIRST)
    reward = np.where(first, np.nan, rec[1].astype(np.float64))
    discount = np.where(first, np.nan, rec[2].astype(np.float64))
    return self._frames, step_type, reward, discount, rec[3].astype(np.int64)

  @property
  def num_streams(self) -> int:
    return self._E

  @property
  def num_actions(self) -> int:
    return self._cfg.num_actions

  @property
  def frames(self) -> torch.Tensor:
    """The device frames of the last tick, uint8 [E, 210, 160, 3]."""
    return self._frames

  def _config(self):
    c = self._cfg
    return (c.num_streams, c.num_actions, c.min_noop_steps, c.max_noop_steps, c.seed, c.stream_offset)

  def get_state(self, stream=None) -> Mapping[str, Any]:
    """The configuration and the device state arrays (one int32 [E] array per field of the game's
    `_lib.CATCH_STATE_FIELDS` / `_lib.BREAKOUT_STATE_FIELDS` / `_lib.PONG_STATE_FIELDS`), copied to the host."""
    s = torch.cuda.current_stream(self._device) if stream is None else stream
    with torch.cuda.stream(s):
      state = self._state.cpu().numpy()
    return {'config': self._config(), 'fields': {k: state[i].copy() for i, k in enumerate(self._FIELDS)}}

  def set_state(self, state: Mapping[str, Any], stream=None) -> None:
    """Restores `get_state()` of an environment with the same configuration and re-renders every stream's frame from
    it: the environment continues bit for bit."""
    if tuple(state['config']) != self._config():
      raise ValueError('state is for the configuration %s, this environment has %s'
                       % (tuple(state['config']), self._config()))
    arrays = np.stack([np.asarray(state['fields'][k], np.int32) for k in self._FIELDS])
    s = torch.cuda.current_stream(self._device) if stream is None else stream
    with torch.cuda.stream(s):
      self._state.copy_(torch.from_numpy(arrays))
      _lib.call(self._RENDER, C.byref(self._cfg), self._state.data_ptr(), self._frames.data_ptr(), s.cuda_stream)


class VectorCatch(_VectorGame):
  """E streams of Catch on the device.

  `reset()` starts a new episode in every stream; `step(actions, reset=None)` applies stream e's action, or starts a
  new episode in the streams where `reset` is true (a stream whose last step was LAST starts one too, as a dm_env
  environment does).  Both return `(frames, step_type, reward, discount, lives)`: `frames` is the device tensor uint8
  [E, 210, 160, 3] that every tick overwrites in place (clone it to keep a frame); step_type int64, reward / discount
  float64 with NaN on FIRST, lives int64, all host arrays [E].  That is the form `VectorTrainer.step` takes.

  A reset simulates k no-op frames, k uniform in [min_noop_steps, max_noop_steps], and its FIRST timestep carries the
  last of them (the reference's `RandomNoopsEnvironmentWrapper`).  Stream e's trajectory depends only on `seed`,
  `stream_offset + e` and its own actions and resets, not on E.  A tick is one pinned host-to-device copy of the actions
  and reset flags, one kernel, one device-to-host copy of the record, and one synchronisation, all on `stream` (default:
  the current CUDA stream)."""

  _STEP, _RENDER, _FIELDS = 'dz_catch_step', 'dz_catch_render', _lib.CATCH_STATE_FIELDS

  def __init__(self, num_streams: int, seed: int, num_actions: int = 6, min_noop_steps: int = 1,
               max_noop_steps: int = 30, stream_offset: int = 0, device='cuda'):
    E = _check_arguments(num_streams, seed, num_actions, min_noop_steps, max_noop_steps, stream_offset,
                         _lib.CATCH_MAX_STREAMS, 3, _lib.CATCH_MAX_NOOP_STEPS, 'a ball could land')
    self._setup(_lib.CatchConfig(E, num_actions, min_noop_steps, max_noop_steps, seed, stream_offset), device)


class _OneStream:
  """One stream of a `_VectorGame` with the reference's dm_env surface."""

  _env: _VectorGame

  @staticmethod
  def _timestep(out):
    frames, step_type, reward, discount, lives = out
    st = parts.StepType(int(step_type[0]))
    first = st == parts.StepType.FIRST
    return parts.TimeStep(st, None if first else float(reward[0]), None if first else float(discount[0]),
                          (frames[0].cpu().numpy(), int(lives[0])))

  def reset(self) -> parts.TimeStep:
    return self._timestep(self._env.reset())

  def step(self, action) -> parts.TimeStep:
    return self._timestep(self._env.step(np.array([int(action)])))

  @property
  def num_actions(self) -> int:
    return self._env.num_actions

  def get_state(self) -> Mapping[str, Any]:
    return self._env.get_state()

  def set_state(self, state: Mapping[str, Any]) -> None:
    self._env.set_state(state)


class Catch(_OneStream):
  """One stream of Catch with the reference's dm_env surface: `reset()` / `step(action)` return a `parts.TimeStep`
  whose observation is (rgb uint8 [210, 160, 3] host array, lives).  Backed by `VectorCatch(1)`; its trajectory is
  stream 0 of a `VectorCatch` with the same arguments."""

  def __init__(self, seed: int, num_actions: int = 6, min_noop_steps: int = 1, max_noop_steps: int = 30,
               stream_offset: int = 0, device='cuda'):
    self._env = VectorCatch(1, seed, num_actions, min_noop_steps, max_noop_steps, stream_offset, device)


class VectorBreakout(_VectorGame):
  """E streams of Breakout on the device (the project's own game, DESIGN.md §11, not ALE Breakout).

  The surface is `VectorCatch`'s: `reset()` and `step(actions, reset=None, stream=None)` return `(frames, step_type,
  reward, discount, lives)` with `frames` the device tensor uint8 [E, 210, 160, 3] that every tick overwrites, and
  `get_state` / `set_state` restore the state and re-render the frames.  Actions: 0 NOOP, 1 FIRE, 2 RIGHT, 3 LEFT (the
  order of ALE's minimal Breakout set); 4 .. num_actions - 1 do nothing.  A brick is worth 7, 4 or 1 points (432 in
  all); a lost ball costs one of 5 lives and gives no reward; the episode ends (LAST) on the last life or the last
  brick.  A reset simulates k no-op frames, k uniform in [min_noop_steps, max_noop_steps] with max <= 63, below the
  64-frame serve delay, so no ball is served during them.  The game has no frame limit: a driver truncates."""

  _STEP, _RENDER, _FIELDS = 'dz_breakout_step', 'dz_breakout_render', _lib.BREAKOUT_STATE_FIELDS

  def __init__(self, num_streams: int, seed: int, num_actions: int = 4, min_noop_steps: int = 1,
               max_noop_steps: int = 30, stream_offset: int = 0, device='cuda'):
    E = _check_arguments(num_streams, seed, num_actions, min_noop_steps, max_noop_steps, stream_offset,
                         _lib.BREAKOUT_MAX_STREAMS, 4, _lib.BREAKOUT_MAX_NOOP_STEPS, 'a ball could be served')
    self._setup(_lib.BreakoutConfig(E, num_actions, min_noop_steps, max_noop_steps, seed, stream_offset), device)


class Breakout(_OneStream):
  """One stream of Breakout with the reference's dm_env surface: `reset()` / `step(action)` return a `parts.TimeStep`
  whose observation is (rgb uint8 [210, 160, 3] host array, lives).  Backed by `VectorBreakout(1)`; its trajectory is
  stream 0 of a `VectorBreakout` with the same arguments."""

  def __init__(self, seed: int, num_actions: int = 4, min_noop_steps: int = 1, max_noop_steps: int = 30,
               stream_offset: int = 0, device='cuda'):
    self._env = VectorBreakout(1, seed, num_actions, min_noop_steps, max_noop_steps, stream_offset, device)


class VectorPong(_VectorGame):
  """E streams of Pong on the device (the project's own game, DESIGN.md §12, not ALE Pong).

  The surface is `VectorCatch`'s: `reset()` and `step(actions, reset=None, stream=None)` return `(frames, step_type,
  reward, discount, lives)` with `frames` the device tensor uint8 [E, 210, 160, 3] that every tick overwrites, and
  `get_state` / `set_state` restore the state and re-render the frames.  Actions: 0 NOOP, 1 FIRE, 2 RIGHT (paddle up),
  3 LEFT (paddle down), 4 RIGHTFIRE, 5 LEFTFIRE (the order of ALE's minimal Pong set); 6 .. num_actions - 1 do nothing.
  The agent's paddle is on the right, a scripted opponent's on the left; a point is +1 or -1, lives are always 0, and
  the episode ends (LAST) when either side reaches 21.  A reset simulates k no-op frames, k uniform in
  [min_noop_steps, max_noop_steps] with max <= 63, below the 64-frame serve delay, so no ball is served during them.
  The game has no frame limit: a driver truncates."""

  _STEP, _RENDER, _FIELDS = 'dz_pong_step', 'dz_pong_render', _lib.PONG_STATE_FIELDS

  def __init__(self, num_streams: int, seed: int, num_actions: int = 6, min_noop_steps: int = 1,
               max_noop_steps: int = 30, stream_offset: int = 0, device='cuda'):
    E = _check_arguments(num_streams, seed, num_actions, min_noop_steps, max_noop_steps, stream_offset,
                         _lib.PONG_MAX_STREAMS, 6, _lib.PONG_MAX_NOOP_STEPS, 'a ball could be served')
    self._setup(_lib.PongConfig(E, num_actions, min_noop_steps, max_noop_steps, seed, stream_offset), device)


class Pong(_OneStream):
  """One stream of Pong with the reference's dm_env surface: `reset()` / `step(action)` return a `parts.TimeStep`
  whose observation is (rgb uint8 [210, 160, 3] host array, lives).  Backed by `VectorPong(1)`; its trajectory is
  stream 0 of a `VectorPong` with the same arguments."""

  def __init__(self, seed: int, num_actions: int = 6, min_noop_steps: int = 1, max_noop_steps: int = 30,
               stream_offset: int = 0, device='cuda'):
    self._env = VectorPong(1, seed, num_actions, min_noop_steps, max_noop_steps, stream_offset, device)
