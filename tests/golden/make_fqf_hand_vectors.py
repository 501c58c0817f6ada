"""Writes tests/golden/fqf_hand_vectors.json: FQF's fraction proposals, selection, targets and fraction gradient
computed BY HAND (the closed forms below, written out per case), not by the oracle they check.

  q = softmax(logits), tau_0 = 0, tau_i = sum_{k<i} q_k, tau_N = 1, tau_hat_i = (tau_i + tau_{i+1}) / 2, w_i = tau_{i+1} - tau_i
  a* = argmax_a sum_i w_i zsel_i(a) (first maximum),  y_j = r + discount ztgt_j(a*)
  g_i = 2 F(tau_i) - F(tau_hat_i) - F(tau_hat_{i-1}), i = 1..N-1
  dq_k = sum_{i>k} g_i,  dlogit_k = q_k (dq_k - sum_j q_j dq_j)            (cot = 1)

F_tau[i] = F(tau_i) (entry 0 unused) and F_hat[i] = F(tau_hat_i) are the quantile function of the case at its fractions.
Run: python tests/golden/make_fqf_hand_vectors.py
"""

import json
import math
import os

cases = []


def case(name, logits, F_tau, F_hat, zsel, ztgt, r_t, discount_t, q, tau, tau_hat, w, a_star, targets, tau_grad, dlogits,
         derivation):
  cases.append(dict(name=name, logits=logits, F_tau=F_tau, F_hat=F_hat, zsel=zsel, ztgt=ztgt, r_t=r_t,
                    discount_t=discount_t, q=q, tau=tau, tau_hat=tau_hat, w=w, a_star=a_star, targets=targets,
                    tau_grad=tau_grad, dlogits=dlogits, derivation=derivation))


ztgt = [[1.0, -1.0], [2.0, -2.0], [3.0, -3.0], [4.0, -4.0]]
case('zero_logits_n4', [0.0, 0.0, 0.0, 0.0], [0.0, 1 / 16, 1 / 4, 9 / 16], [1 / 64, 9 / 64, 25 / 64, 49 / 64],
     [[1.0, 0.0], [1.0, 0.0], [1.0, 0.0], [0.0, 2.0]], ztgt, 0.5, 0.9,
     [0.25] * 4, [0.0, 0.25, 0.5, 0.75, 1.0], [0.125, 0.375, 0.625, 0.875], [0.25] * 4, 0,
     [0.5 + 0.9 * z for z in (1.0, 2.0, 3.0, 4.0)], [-1 / 32] * 3, [-3 / 256, -1 / 256, 1 / 256, 3 / 256],
     'Zero logits: q = 1/4, tau = i/4, tau_hat = (2i + 1)/8, w = 1/4.  Selection: 3/4 against 1/2, a* = 0.  F(tau) = '
     'tau^2: g_i = 2 tau_i^2 - tau_hat_i^2 - tau_hat_{i-1}^2 = -2 (1/8)^2 = -1/32 for every i.  dq = [-3, -2, -1, 0]/32, '
     'sum_j q_j dq_j = -3/64, dlogit_k = (dq_k + 3/64) / 4 = [-3, -1, 1, 3]/256.')
case('saturated_fraction', [-200.0, 0.0, 0.0, 0.0], [0.0, 0.0, 1 / 3, 2 / 3], [0.0, 1 / 6, 1 / 2, 5 / 6],
     [[0.0, 100.0], [1.0, 0.0], [1.0, 0.0], [1.0, 0.0]], ztgt, -1.0, 0.99,
     [0.0, 1 / 3, 1 / 3, 1 / 3], [0.0, 0.0, 1 / 3, 2 / 3, 1.0], [0.0, 1 / 6, 1 / 2, 5 / 6], [0.0, 1 / 3, 1 / 3, 1 / 3],
     0, [-1.0 + 0.99 * z for z in (1.0, 2.0, 3.0, 4.0)], [-1 / 6, 0.0, 0.0], [0.0, 0.0, 0.0, 0.0],
     'q_0 = e^-200 / (3 + e^-200) is 0 to 1e-87: tau_0 = tau_1 = 0 coincide and interval 0 has weight 0, so the 100 '
     'of action 1 there does not count: weighted 1 against 0, a* = 0 (the unweighted mean would pick 1).  F(tau) = '
     'tau: g_1 = 0 - 1/6 - 0, g_2 = 2/3 - 1/2 - 1/6 = 0, g_3 = 4/3 - 5/6 - 1/2 = 0; dq = [-1/6, 0, 0, 0] and '
     'sum_j q_j dq_j = 0, so dlogit = q dq = 0: the saturated softmax passes no gradient.')
case('weights_decide_selection', [math.log(4.0), math.log(2.0), 0.0, 0.0], [0.0, 0.5, 0.75, 0.875],
     [0.25, 0.625, 0.8125, 0.9375], [[1.0, 0.0], [1.0, 0.0], [1.0, 3.0], [1.0, 3.0]], ztgt, 0.0, 0.5,
     [0.5, 0.25, 0.125, 0.125], [0.0, 0.5, 0.75, 0.875, 1.0], [0.25, 0.625, 0.8125, 0.9375], [0.5, 0.25, 0.125, 0.125],
     0, [0.5 * z for z in (1.0, 2.0, 3.0, 4.0)], [0.125, 0.0625, 0.0],
     [0.5 * 0.078125, 0.25 * -0.046875, 0.125 * -0.109375, 0.125 * -0.109375],
     'q = [4, 2, 1, 1]/8: tau = [0, 1/2, 3/4, 7/8, 1], w = q.  Action 0 gives sum w z = 1, action 1 gives 3/8 + 3/8 = '
     '3/4 < 1, though its mean 3/2 exceeds action 0\'s 1: a* = 0.  F(tau) = tau: g_1 = 1 - 5/8 - 1/4 = 1/8, g_2 = '
     '3/2 - 13/16 - 5/8 = 1/16, g_3 = 7/4 - 15/16 - 13/16 = 0.  dq = [3/16, 1/16, 0, 0], sum q dq = 7/64, '
     'dlogit = q (dq - 7/64) = [5/128, -3/256, -7/512, -7/512] (sums to 0).')
case('terminal', [0.0, 0.0, 0.0, 0.0], [0.0, -0.5, 0.0, 0.5], [-0.75, -0.25, 0.25, 0.75],
     [[0.0, 1.0], [0.0, 1.0], [0.0, 1.0], [0.0, 1.0]], ztgt, 1.0, 0.0,
     [0.25] * 4, [0.0, 0.25, 0.5, 0.75, 1.0], [0.125, 0.375, 0.625, 0.875], [0.25] * 4, 1, [1.0] * 4,
     [0.0, 0.0, 0.0], [0.0] * 4,
     'discount 0: y_j = r = 1 whatever the target quantiles.  a* = 1 (1 against 0).  F(tau) = 2 tau - 1 is linear and '
     'the fractions are uniform, which is optimal for it: g_i = 4 tau_i - 2 (tau_hat_i + tau_hat_{i-1}) = 0.')

if __name__ == '__main__':
  out = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'fqf_hand_vectors.json')
  with open(out, 'w') as f:
    json.dump({'_about': 'FQF fractions, selection, targets and fraction gradients computed by hand; see '
                         'make_fqf_hand_vectors.py', 'cases': cases}, f, indent=1)
  print(out, len(cases))
