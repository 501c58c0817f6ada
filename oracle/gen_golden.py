"""Generates tests/golden/replay_*.npz by running oracle/scenarios.py against the
REFERENCE's own replay.py (imported from /root/reference, build container only).

  python -m oracle.gen_golden

TEST INFRASTRUCTURE ONLY.  The fixtures are committed; this script is committed
so they can be regenerated and audited.

One documented deviation: for scenarios with priority_exponent != 0.5 the
reference's `_power` is evaluated through the canonical float32 definition
round_f32(pow_f64(x, (double)(float)alpha)) (SURVEY §8(a) R3) because numpy's
float32 SIMD `powf` is library/version dependent (differs by 1 ulp on ~20 % of
inputs between the pinned numpy 1.21.5 and this image's 2.3.5).  alpha = 0.5
(every BASELINE.json PER config) needs no such pin: `**0.5` is a correctly
rounded sqrt everywhere.
"""

import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_import, replay_oracle, scenarios  # noqa: E402

# a long random prioritized-replay run (ring wrap-around, many priority updates), recorded from the original
LONG_RANDOM_PER = dict(capacity=257, alpha=0.5, usp=1e-3, normalize=True, batch=32, rounds=400, seed=31)


def main():
  ref = ref_import.load_reference_replay()
  out_dir = os.path.join(os.path.dirname(HERE), 'tests', 'golden')
  os.makedirs(out_dir, exist_ok=True)
  stock_power = ref._power
  for name, fn in scenarios.ALL.items():
    ref._power = replay_oracle.power_keep_zero if 'pow06' in name else stock_power
    res = fn(ref)
    np.savez_compressed(os.path.join(out_dir, name + '.npz'), **res)
    print(name, {k: tuple(v.shape) for k, v in res.items()})
  ref._power = stock_power
  res = scenarios.prioritized_replay_script(ref, **LONG_RANDOM_PER)
  np.savez_compressed(os.path.join(out_dir, 'replay_long_random_per.npz'), **res)
  print('replay_long_random_per', {k: tuple(v.shape) for k, v in res.items()})


if __name__ == '__main__':
  main()
