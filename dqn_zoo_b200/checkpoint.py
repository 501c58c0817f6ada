"""Checkpoint directories of device-resident state (DESIGN.md §9): streamed device-to-file transfers with bounded host
memory, a 64-bit digest per chunk, and a JSON manifest that is validated before anything is written to the device.

A file of a checkpoint directory is raw bytes, written and read in chunks of at most `CHUNK_BYTES`.  Device data goes
through a fixed staging ring (`Transfer`: `depth` pinned host buffers and as many device buffers of `CHUNK_BYTES`
each), so D2H copies overlap file writes and file reads overlap H2D copies, and host memory does not grow with the
size of what is saved.  Each chunk is digested on the device before its D2H copy on save (`dz_ckpt_digest`, or for the
replay's bulk records `dz_ckpt_snapshot`, which packs and digests them in one read) and after its H2D copy on load, so
one comparison covers the file and both transfers; host arrays are digested on the CPU with the same function
(`dz_ckpt_digest_host`).  The manifest records every file's size, chunk size and digests.

`Files` is the one description of a directory's files that the blocking save and a `Snapshot` both write; a
`Snapshot` holds device and host copies taken at one point of a CUDA stream and writes them later, on any thread."""

from __future__ import annotations

import ctypes as C
import json
import os
from typing import Any, Dict, Mapping, Optional

import numpy as np
import torch

from dqn_zoo_b200 import _lib

CHUNK_BYTES = 64 << 20
MANIFEST = 'manifest.json'


def digest_host(buf) -> int:
  """`dz_ckpt_digest_host` of a contiguous host buffer (numpy array or bytes)."""
  a = np.ascontiguousarray(np.frombuffer(buf, np.uint8) if isinstance(buf, (bytes, bytearray, memoryview)) else buf)
  out = C.c_uint64()
  _lib.call('dz_ckpt_digest_host', a.ctypes.data if a.nbytes else None, a.nbytes, C.byref(out))
  return out.value


def write_json(path: str, obj: Mapping[str, Any]) -> None:
  with open(path, 'w') as f:
    json.dump(obj, f, indent=1, sort_keys=True)
    f.flush()
    os.fsync(f.fileno())


def read_manifest(directory: str, kind: str) -> Dict[str, Any]:
  """The manifest of a checkpoint directory written for `kind`; ValueError if there is none or it is not one."""
  path = os.path.join(directory, MANIFEST)
  try:
    with open(path) as f:
      m = json.load(f)
  except (OSError, ValueError) as e:
    raise ValueError('%s is not a readable checkpoint manifest: %s' % (path, e)) from e
  if not isinstance(m, dict) or m.get('format') != kind:
    raise ValueError('%s is not a %s checkpoint (format %r)' % (path, kind, m.get('format') if isinstance(m, dict) else m))
  return m


def validate(saved: Mapping[str, Any], want: Mapping[str, Any], where: str) -> None:
  """ValueError naming the first key of `want` whose saved value differs (kind, layout, capacity, shapes, version)."""
  for key, value in want.items():
    got = saved.get(key)
    if isinstance(value, tuple):
      got = tuple(got) if isinstance(got, list) else got
    if got != value:
      raise ValueError('%s: checkpoint has %s = %r, this object needs %r' % (where, key, got, value))


class Transfer:
  """The staging ring of one save or load on the current CUDA stream.  Every method returns or takes the manifest
  entry of one file: {'bytes', 'chunk', 'digests'} (digests as hex strings, one per chunk)."""

  def __init__(self, device, chunk_bytes: int = CHUNK_BYTES, depth: int = 2, device_staging: bool = True):
    self.chunk = int(chunk_bytes)
    self.host = [torch.empty(self.chunk, dtype=torch.uint8).pin_memory() for _ in range(depth)]
    # a writer of snapshot buffers copies straight from them and needs no device staging
    self.dev = [torch.empty(self.chunk, dtype=torch.uint8, device=device) for _ in range(depth)] if device_staging else []
    self.device = device
    self._digests = torch.zeros(64, dtype=torch.int64, device=device)

  def _digest_slots(self, n):
    if n > self._digests.numel():
      self._digests = torch.zeros(n, dtype=torch.int64, device=self.device)
    return self._digests

  # -- save --------------------------------------------------------------------------------------------------------
  def save_device(self, path: str, nbytes: int, produce, chunk: Optional[int] = None,
                  digests: Optional[torch.Tensor] = None) -> Dict[str, Any]:
    """Writes `nbytes` device bytes to `path`.  `produce` is either a flat uint8 CUDA tensor of at least `nbytes` bytes,
    or a callable (offset, n, staging, digest) -> uint8 CUDA tensor of the n bytes at `offset` that fills the device
    staging buffer it is given and writes the chunk's digest to the device uint64 at address `digest` (the snapshot
    pass, `dz_ckpt_snapshot`).  `chunk` (<= CHUNK_BYTES) lets a file keep whole records per chunk.  `digests`: the
    chunks' digests, already computed on the device (int64 CUDA tensor), for a tensor `produce`."""
    chunk = min(self.chunk, int(chunk or self.chunk))
    nchunks = (nbytes + chunk - 1) // chunk
    dig = self._digest_slots(max(nchunks, 1)) if digests is None else digests
    stream = torch.cuda.current_stream()
    pending = [None] * len(self.host)
    with open(path, 'wb') as f:
      def drain(slot):
        if pending[slot] is not None:
          ev, n = pending[slot]
          ev.synchronize()
          f.write(memoryview(self.host[slot].numpy())[:n])
          pending[slot] = None
      for k in range(nchunks):
        slot = k % len(self.host)
        drain(slot)                     # chunk k - depth: the older pending chunk, so the file is written in order
        off, n = k * chunk, min(chunk, nbytes - k * chunk)
        if isinstance(produce, torch.Tensor):
          src = produce[off:off + n]
          if digests is None:
            _lib.call('dz_ckpt_digest', src.data_ptr(), n, dig[k:].data_ptr(), stream.cuda_stream)
        else:
          src = produce(off, n, self.dev[slot][:n], dig[k:].data_ptr())
        self.host[slot][:n].copy_(src[:n], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(stream)
        pending[slot] = (ev, n)
      for k in range(nchunks, nchunks + len(self.host)):
        drain(k % len(self.host))
      f.flush()
      os.fsync(f.fileno())
    digests = dig[:nchunks].cpu().numpy().view(np.uint64)
    return {'bytes': int(nbytes), 'chunk': chunk, 'digests': ['%016x' % d for d in digests]}

  @staticmethod
  def save_host(path: str, array: np.ndarray) -> Dict[str, Any]:
    """A host array's bytes to `path` (C order), with its dtype and shape."""
    a = np.ascontiguousarray(array)
    raw = a.reshape(-1).view(np.uint8)
    chunk = CHUNK_BYTES
    with open(path, 'wb') as f:
      f.write(memoryview(raw))
      f.flush()
      os.fsync(f.fileno())
    digests = ['%016x' % digest_host(raw[o:o + chunk]) for o in range(0, raw.size, chunk)]
    return {'bytes': int(raw.size), 'chunk': chunk, 'digests': digests, 'dtype': a.dtype.str, 'shape': list(a.shape)}

  # -- load --------------------------------------------------------------------------------------------------------
  def load_device(self, path: str, entry: Mapping[str, Any], consume) -> None:
    """Reads the file `entry` describes into the device.  `consume` is either a flat uint8 CUDA tensor of at least
    entry['bytes'] bytes (chunks are copied straight into it) or a callable (offset, n, staging) that moves the n
    staged device bytes at `offset` to their place.  RuntimeError, naming the file and chunk, for a file of the
    wrong size or a chunk whose digest differs from the manifest's (the device then holds partial data)."""
    nbytes, chunk = int(entry['bytes']), int(entry['chunk'])
    check_size(path, nbytes)
    if not 0 < chunk <= self.chunk:
      raise RuntimeError('%s: chunk size %d exceeds the staging buffers (%d)' % (path, chunk, self.chunk))
    nchunks = (nbytes + chunk - 1) // chunk
    if len(entry['digests']) != nchunks:
      raise RuntimeError('%s: the manifest lists %d chunk digests for %d chunks' % (path, len(entry['digests']), nchunks))
    dig = self._digest_slots(max(nchunks, 1))
    stream = torch.cuda.current_stream()
    copied = [None] * len(self.host)
    with open(path, 'rb') as f:
      for k in range(nchunks):
        slot = k % len(self.host)
        if copied[slot] is not None:
          copied[slot].synchronize()    # the H2D copy out of this pinned buffer has completed
        off, n = k * chunk, min(chunk, nbytes - k * chunk)
        host = self.host[slot][:n]
        got = f.readinto(memoryview(host.numpy()))
        if got != n:
          raise RuntimeError('%s: chunk %d is truncated (%d of %d bytes)' % (path, k, got, n))
        dst = consume[off:off + n] if isinstance(consume, torch.Tensor) else self.dev[slot][:n]
        dst.copy_(host, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(stream)
        copied[slot] = ev
        _lib.call('dz_ckpt_digest', dst.data_ptr(), n, dig[k:].data_ptr(), stream.cuda_stream)
        if not isinstance(consume, torch.Tensor):
          consume(off, n, dst)
    got = dig[:nchunks].cpu().numpy().view(np.uint64)
    for k, (g, w) in enumerate(zip(got, entry['digests'])):
      if '%016x' % g != w:
        raise RuntimeError('%s: chunk %d digest %016x differs from the manifest\'s %s' % (path, k, g, w))

  @staticmethod
  def load_host(path: str, entry: Mapping[str, Any]) -> np.ndarray:
    """The host array `save_host` wrote; RuntimeError naming the file and chunk on a size or digest mismatch."""
    nbytes, chunk = int(entry['bytes']), int(entry['chunk'])
    check_size(path, nbytes)
    raw = np.fromfile(path, dtype=np.uint8)
    if raw.size != nbytes:
      raise RuntimeError('%s: read %d of %d bytes' % (path, raw.size, nbytes))
    digests = ['%016x' % digest_host(raw[o:o + chunk]) for o in range(0, nbytes, chunk)]
    if len(digests) != len(entry['digests']):
      raise RuntimeError('%s: the manifest lists %d chunk digests for %d chunks' % (path, len(entry['digests']), len(digests)))
    for k, (g, w) in enumerate(zip(digests, entry['digests'])):
      if g != w:
        raise RuntimeError('%s: chunk %d digest %s differs from the manifest\'s %s' % (path, k, g, w))
    return raw.view(np.dtype(entry['dtype'])).reshape(entry['shape'])


def check_size(path: str, nbytes: int) -> None:
  try:
    size = os.path.getsize(path)
  except OSError as e:
    raise RuntimeError('%s: missing (%s)' % (path, e)) from e
  if size != nbytes:
    raise RuntimeError('%s: %d bytes on disk, the manifest says %d (%s)'
                       % (path, size, nbytes, 'truncated' if size < nbytes else 'extra bytes at the end'))


def write_bytes(path: str, data: bytes) -> None:
  with open(path, 'wb') as f:
    f.write(data)


class Files:
  """The files of one checkpoint directory written through `Transfer`, and its manifest: one definition for the
  blocking save, which fills it from the live arrays, and for a snapshot, which fills it from copies.

  `host`: name -> zero-argument callable returning the host array (`save_host`), so a snapshot can copy containers at
  the snapshot point and convert them in the writer.  `dev`: name -> flat uint8 CUDA tensor (`save_device`).  `bulk`:
  None or (name, nbytes, produce, chunk, digests), the arguments of one `save_device` call.  `manifest`: every manifest
  key but `files`, which `write` adds."""

  def __init__(self):
    self.host: Dict[str, Any] = {}
    self.dev: Dict[str, torch.Tensor] = {}
    self.bulk = None
    self.manifest: Dict[str, Any] = {}

  def write(self, directory: str, xfer: Transfer) -> None:
    os.makedirs(directory, exist_ok=True)
    path = lambda name: os.path.join(directory, name + '.bin')
    files = {}
    for name, make in self.host.items():
      files[name] = Transfer.save_host(path(name), make())
    for name, t in self.dev.items():
      files[name] = xfer.save_device(path(name), t.numel(), t)
    if self.bulk is not None:
      name, nbytes, produce, chunk, digests = self.bulk
      files[name] = xfer.save_device(path(name), nbytes, produce, chunk, digests=digests)
    write_json(os.path.join(directory, MANIFEST), dict(self.manifest, files=files))


class Snapshot:
  """A checkpoint captured at one point of the CUDA stream that was current when it was made (DESIGN.md §9): device
  copies plus host copies, which `write(directory)` turns into exactly the files `save_checkpoint(directory)` would have
  written at that point.  The object keeps training's arrays out of the write, so training may go on meanwhile.

  `write` may run on any thread, once: it makes a CUDA stream and a staging ring (`Transfer`) of its own, orders its
  stream after the snapshot point, reads only the snapshot's buffers and returns when every copy out of them has
  completed.  `device_bytes` is the HBM the snapshot holds; `release()` drops it (after `write`, or instead of it)."""

  def __init__(self, writer, buffers, device):
    self._writer = writer                 # callable(directory, xfer)
    self._buffers = list(buffers)         # the device copies `writer` reads (it holds them too, until released)
    self._device = torch.device(device)
    self.device_bytes = int(sum(t.numel() * t.element_size() for t in self._buffers))
    self._ready = torch.cuda.Event()
    self._ready.record()                  # the snapshot point on the caller's stream

  def write(self, directory: str) -> None:
    if self._writer is None:
      raise RuntimeError('this snapshot was released')
    with torch.cuda.device(self._device):
      stream = torch.cuda.Stream()
      try:
        with torch.cuda.stream(stream):
          stream.wait_event(self._ready)
          self._writer(directory, Transfer(self._device, device_staging=False))
      finally:
        stream.synchronize()              # no copy out of the buffers is pending when they are released

  def release(self) -> None:
    self._writer, self._buffers = None, []
