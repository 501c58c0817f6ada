"""Writes tests/golden/cql_hand_vectors.json: CQL(H) regularisers and their gradients computed BY HAND (plain python
arithmetic spelled out below, from the closed forms of each case), not by the oracle they check.

  R = logsumexp_a Q_a - Q_{a_tm1},   dR/dQ_a = softmax(Q)_a - [a = a_tm1]

Equal Q over A actions: logsumexp = Q + log A, so R = log A and softmax = 1/A.  Q_{a_tm1} ahead of every other action by
d: R = log(1 + (A - 1) e^-d) -> 0 as d grows.  Adding c to every Q_a adds c to both terms: R and softmax are unchanged.
Run: python tests/golden/make_cql_hand_vectors.py
"""

import json
import math
import os

cases = []


def case(name, q, a_tm1, R, grad, derivation):
  cases.append(dict(name=name, q=q, a_tm1=a_tm1, R=R, grad=grad, derivation=derivation))


def onehot_minus(A, a_tm1, p):
  return [p[a] - (1.0 if a == a_tm1 else 0.0) for a in range(A)]


case('equal_q_two', [0.5, 0.5], 1, math.log(2.0), [0.5, -0.5],
     'two equal values: R = log 2, softmax = 1/2 each.')
case('equal_q_six', [-3.0] * 6, 4, math.log(6.0), onehot_minus(6, 4, [1.0 / 6] * 6),
     'six equal values: R = log 6, softmax = 1/6 each.')
case('equal_q_sixty_four_shifted', [1000.0] * 64, 0, math.log(64.0), onehot_minus(64, 0, [1.0 / 64] * 64),
     'sixty-four equal values at 1000 (a naive exp overflows): R = log 64 = 6 log 2, softmax = 1/64 each.')
case('one_action', [7.25], 0, 0.0, [0.0], 'A = 1: logsumexp = Q, R = 0 and softmax = 1, so the gradient is 0.')
for d in (1.0, 10.0, 50.0):
  e = math.exp(-d)
  den = 1.0 + 2.0 * e
  case('taken_action_ahead_by_%g' % d, [0.0, d, 0.0], 1, math.log1p(2.0 * e),
       [e / den, 1.0 / den - 1.0, e / den],
       'Q_{a_tm1} = %g above the other two: R = log(1 + 2 e^-%g), softmax = (e^-d, 1, e^-d) / (1 + 2 e^-d).' % (d, d))
case('taken_action_behind_by_20', [20.0, 0.0], 1, 20.0 + math.log1p(math.exp(-20.0)),
     [1.0 / (1.0 + math.exp(-20.0)), math.exp(-20.0) / (1.0 + math.exp(-20.0)) - 1.0],
     'Q_{a_tm1} 20 below the other: R = 20 + log(1 + e^-20), softmax = (1, e^-20) / (1 + e^-20).')
for c in (-5.0, 123.0):
  base = [0.0, 1.0, 3.0]
  s = 1.0 + math.e + math.exp(3.0)
  p = [1.0 / s, math.e / s, math.exp(3.0) / s]
  case('shift_%g' % c, [x + c for x in base], 1, math.log(s) - 1.0, onehot_minus(3, 1, p),
       '(0, 1, 3) + %g: the shift cancels; R = log(1 + e + e^3) - 1, softmax = (1, e, e^3) / (1 + e + e^3).' % c)

if __name__ == '__main__':
  out = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'cql_hand_vectors.json')
  with open(out, 'w') as f:
    json.dump({'_about': 'CQL(H) regularisers computed by hand; see make_cql_hand_vectors.py', 'cases': cases}, f,
              indent=1)
  print(out, len(cases))
