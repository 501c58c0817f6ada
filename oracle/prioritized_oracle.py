"""The priority rule of prioritized replay for all ten agent kinds (DESIGN.md §19), over the `aux` of the float64
oracles (learner_oracle, munchausen_oracle, munchausen_iqn_oracle, fqf_oracle).

Each priority comes from the example's UNWEIGHTED loss, as the reference's two prioritized agents take theirs:
  dqn, double_q, prioritized           |td|                          (`prioritized/agent.py:202`)
  munchausen                           |td| against its soft target  (the same rule on M-DQN's TD error)
  c51, rainbow                         clip(|loss|, 0, 100)          (`rainbow/agent.py:194`)
  qrdqn, iqn, munchausen_iqn, fqf      clip(|loss|, 0, 100) of the per-example quantile Huber loss (fqf: at the
                                       proposed fractions, not the fraction loss)
learner_oracle keeps its own two-kind rule for prioritized and rainbow; this one reproduces it.
"""

import torch

TD_KINDS = ('dqn', 'double_q', 'prioritized', 'munchausen')
LOSS_KINDS = ('c51', 'rainbow', 'qrdqn', 'iqn', 'munchausen_iqn', 'fqf')
KINDS = TD_KINDS + LOSS_KINDS


def priorities(kind, aux):
  """The [B] priorities of one update of `kind` from its oracle's `aux` ('td_errors' for the |td| kinds, 'losses' for
  the others), in aux's dtype."""
  if kind in TD_KINDS:
    return torch.as_tensor(aux['td_errors']).abs()
  if kind in LOSS_KINDS:
    return torch.as_tensor(aux['losses']).abs().clamp(0.0, 100.0)
  raise ValueError(kind)
