"""Writes tests/golden/munchausen_iqn_hand_vectors.json: Munchausen-IQN targets computed BY HAND (plain python arithmetic
spelled out below, from the closed forms of each case), not by the oracle they check.

  qbar(s, a) = mean_j zbar_j(s, a);  pi = softmax(qbar / tau);  h(a) = v + tau log S - qbar(a) = -tau log pi(a)
  bonus = alpha clip(tau log pi(a_tm1|s_tm1), l0, 0)
  y_j   = r + bonus + discount sum_a pi(a|s_t) (zbar_j(s_t, a) + h_t(a)) = r + bonus + discount (sum_a pi zbar_j + E)

Every case has a uniform or a degenerate policy at s_t: with m actions tied at the maximum and the others far below,
pi = 1/m on the tied actions, h = tau ln m there, E = sum_a pi h = tau ln m, and sum_a pi zbar_j is the mean of the
tied actions' samples j.
Run: python tests/golden/make_munchausen_iqn_hand_vectors.py
"""

import json
import math
import os

LN2 = math.log(2.0)
cases = []


def case(name, zbar_tm1, zbar_t, a_tm1, r_t, discount_t, alpha, tau, l0, bonus, entropy, targets, derivation):
  cases.append(dict(name=name, zbar_tm1=zbar_tm1, zbar_t=zbar_t, a_tm1=a_tm1, r_t=r_t, discount_t=discount_t,
                    alpha=alpha, tau=tau, l0=l0, bonus=bonus, entropy=entropy, targets=targets,
                    derivation=derivation))


b = 0.9 * (-0.5 * LN2)
case('clip_inactive', [[0.0, 2.0], [2.0, 0.0]], [[1.0, 0.0], [3.0, 2.0], [-1.0, 1.0]], 0, 1.0, 0.99, 0.9, 0.5, -1.0,
     b, 0.5 * LN2, [1.0 + b + 0.99 * (m + 0.5 * LN2) for m in (0.5, 2.5, 0.0)],
     'qbar(s_tm1) = [1, 1]: uniform, tau log pi = 0.5 ln(1/2) = -0.347 > l0, bonus = -0.45 ln 2. qbar(s_t) = [1, 1]: '
     'uniform, E = 0.5 ln 2; sum_a pi zbar_j = row means 0.5, 2.5, 0. y_j = 1 - 0.45 ln 2 + 0.99 (mean_j + 0.5 ln 2).')
case('clip_active', [[0.0, 3.0], [0.0, 3.0]], [[2.0, 2.0], [1.0, 3.0], [3.0, 1.0]], 0, 0.0, 0.5, 0.9, 1.0, -1.0,
     -0.9, LN2, [-0.9 + 0.5 * (2.0 + LN2)] * 3,
     'qbar(s_tm1) = [0, 3]: tau log pi(0) = -3 - ln(1 + e^-3) = -3.049 < l0 = -1, clipped: bonus = -0.9. qbar(s_t) = '
     '[2, 2]: uniform, E = ln 2, every row mean 2. y_j = -0.9 + 0.5 (2 + ln 2).')
case('terminal_bonus_survives', [[1.0, 1.0]], [[7.0, -3.0], [5.0, -1.0]], 1, -1.0, 0.0, 0.9, 0.5, -1.0,
     0.9 * (-0.5 * LN2), None, [-1.0 - 0.9 * 0.5 * LN2] * 2,
     'discount 0 removes the bootstrap but not the bonus: tau log pi(1) = 0.5 ln(1/2), y_j = -1 - 0.45 ln 2. '
     '(E at s_t is not a closed form here and is not checked.)')
case('one_action', [[5.0], [7.0]], [[-2.0], [0.0], [1.0]], 0, 0.5, 0.9, 0.9, 0.03, -1.0,
     0.0, 0.0, [0.5 + 0.9 * z for z in (-2.0, 0.0, 1.0)],
     'A = 1: pi = 1, tau log pi = 0, bonus 0, h = 0 and E = 0. y_j = r + discount zbar_j = 0.5 + 0.9 zbar_j.')
wide_t = [[-100.0, 0.0, 100.0], [-110.0, 10.0, 90.0], [-90.0, -10.0, 110.0]]
case('wide_q_small_tau_greedy', [[0.0, 50.0, 100.0], [0.0, 50.0, 100.0]], wide_t, 2, 0.0, 0.99, 0.9, 0.03, -1.0,
     0.0, 0.0, [0.99 * z for z in (100.0, 90.0, 110.0)],
     'tau = 0.03 and qbar spread over 100: the other exponents are -1667 and -3333, exp underflows to 0 without '
     'overflow. tau log pi(2) = 0, bonus 0. At s_t qbar = [-100, 0, 100]: pi = onehot(2), h(2) = 0, E = 0 (the other '
     'terms are 0 * h, h finite). y_j = 0.99 zbar_j(2) = 0.99 [100, 90, 110].')
case('wide_q_small_tau_clipped', [[0.0, 50.0, 100.0], [0.0, 50.0, 100.0]], wide_t, 0, 0.0, 0.99, 0.9, 0.03, -1.0,
     -0.9, 0.0, [-0.9 + 0.99 * z for z in (100.0, 90.0, 110.0)],
     'tau log pi(0) = 0 - 100 - 0.03 ln 1 = -100 < l0: bonus = -0.9 (exp(100 / 0.03) would overflow in the naive '
     'form). y_j = -0.9 + 0.99 zbar_j(2).')
case('two_way_tie_at_s_t', [[2.0, 2.0, 2.0, 2.0], [2.0, 2.0, 2.0, 2.0]],
     [[3.0, 5.0, -50.0, -60.0], [5.0, 3.0, -50.0, -60.0]], 3, 0.25, 0.9, 0.5, 0.1, -0.2, 0.5 * (-0.2 * LN2), 0.1 * LN2,
     [0.25 + 0.5 * (-0.2 * LN2) + 0.9 * (4.0 + 0.1 * LN2)] * 2,
     'qbar(s_tm1) uniform over 4 actions: tau log pi = 0.1 ln(1/4) = -0.2 ln 2 = -0.139, inside [l0, 0] = [-0.2, 0]: '
     'bonus = 0.5 * -0.2 ln 2. qbar(s_t) = [4, 4, -50, -60]: two actions tie, the others lie 540 and 640 temperatures '
     'below (exp underflows in fp32): pi = 1/2 on each, E = 0.1 ln 2, sum_a pi zbar_j = 4. '
     'y_j = 0.25 - 0.1 ln 2 + 0.9 (4 + 0.1 ln 2).')

if __name__ == '__main__':
  out = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'munchausen_iqn_hand_vectors.json')
  with open(out, 'w') as f:
    json.dump({'_about': 'Munchausen-IQN targets computed by hand; see make_munchausen_iqn_hand_vectors.py',
               'cases': cases}, f, indent=1)
  print(out, len(cases))
