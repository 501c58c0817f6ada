"""dqn_zoo_b200 — H100-native replay-sampler + learner-update hot path of dqn_zoo.

Python host code calling hand-written sm_90a CUDA through the C ABI in
include/dqn_zoo_b200.h.  There is no CPU fallback: importing `dqn_zoo_b200.replay`
or `dqn_zoo_b200.agent` without the built library raises.
"""

__version__ = '0.1'
