"""numpy restatement of the checkpoint chunk digest (dqn_zoo_b200/csrc/dz_checkpoint.cu, dz_ckpt_digest).

Bytes b of length n -> 8-byte little-endian words w_i, i < ceil(n / 8), the last one zero padded;
digest = mix64(S ^ n), S = sum_i mix64(w_i ^ ((i + 1) * 0x9E3779B97F4A7C15)) mod 2^64, with mix64 the splitmix64
finaliser.  uint64 array arithmetic in numpy wraps mod 2^64, as the CUDA integer ops do."""

import numpy as np

_K = np.uint64(0x9E3779B97F4A7C15)


def mix64(x):
  x = np.asarray(x, dtype=np.uint64)
  x = (x ^ (x >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
  x = (x ^ (x >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
  return x ^ (x >> np.uint64(31))


def digest(data) -> int:
  raw = np.frombuffer(bytes(data), dtype=np.uint8)
  n = raw.size
  words = (n + 7) // 8
  padded = np.zeros(8 * words, dtype=np.uint8)
  padded[:n] = raw
  w = padded.view('<u8').astype(np.uint64)
  with np.errstate(over='ignore'):
    i = np.arange(1, words + 1, dtype=np.uint64)
    s = mix64(w ^ (i * _K)).sum(dtype=np.uint64) if words else np.uint64(0)
    return int(mix64(np.array([s ^ np.uint64(n)], dtype=np.uint64))[0])
