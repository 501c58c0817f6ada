"""Writes tests/golden/munchausen_hand_vectors.json: Munchausen DQN targets computed BY HAND (plain python arithmetic
spelled out below, from the closed forms of each case), not by the oracle they check.

  tau log pi(a|s) = qbar(s, a) - v - tau log sum_a' exp((qbar(s, a') - v) / tau),  v = max_a' qbar(s, a')
  target = r + alpha clip(tau log pi(a_tm1|s_tm1), l0, 0) + discount sum_a pi(a|s_t) (qbar(s_t, a) - tau log pi(a|s_t))

Every case below has a uniform or a degenerate policy at s_t, where the bootstrap sum_a pi (qbar - tau log pi) is
v_t + tau log(number of actions at the maximum) exactly (each term of the sum is that value).
Run: python tests/golden/make_munchausen_hand_vectors.py
"""

import json
import math
import os

LN2 = math.log(2.0)
cases = []


def case(name, qbar_tm1, qbar_t, q_tm1, a_tm1, r_t, discount_t, alpha, tau, l0, bonus, target, derivation):
  cases.append(dict(name=name, qbar_tm1=qbar_tm1, qbar_t=qbar_t, q_tm1=q_tm1, a_tm1=a_tm1, r_t=r_t,
                    discount_t=discount_t, alpha=alpha, tau=tau, l0=l0, bonus=bonus, target=target,
                    td=target - q_tm1[a_tm1], derivation=derivation))


case('clip_inactive', [1.0, 1.0], [0.0, 0.0], [0.25, -0.5], 0, 1.0, 0.99, 0.9, 0.5, -1.0,
     0.9 * (-0.5 * LN2), 1.0 - 0.9 * 0.5 * LN2 + 0.99 * (0.0 + 0.5 * LN2),
     'uniform pi at s_tm1: tau log pi = 0.5 ln(1/2) = -0.3466 > l0, bonus = 0.9 * -0.5 ln 2. uniform pi at s_t: '
     'every qbar - tau log pi = 0 + 0.5 ln 2. target = 1 - 0.45 ln 2 + 0.99 * 0.5 ln 2 = 1 + 0.045 ln 2.')
case('clip_active', [0.0, 3.0], [2.0, 2.0], [0.5, 1.0], 0, 0.0, 0.5, 0.9, 1.0, -1.0,
     0.9 * -1.0, -0.9 + 0.5 * (2.0 + LN2),
     'tau log pi(0) = 0 - 3 - ln(1 + e^-3) = -3.0486 < l0 = -1: clipped, bonus = -0.9. uniform pi at s_t: '
     'boot = 2 + ln 2. target = -0.9 + 0.5 (2 + ln 2) = 0.1 + 0.5 ln 2.')
case('terminal_bonus_survives', [1.0, 1.0], [7.0, -3.0], [0.0, 0.125], 1, -1.0, 0.0, 0.9, 0.5, -1.0,
     0.9 * (-0.5 * LN2), -1.0 - 0.9 * 0.5 * LN2,
     'discount 0 removes the bootstrap but not the bonus: tau log pi(1) = 0.5 ln(1/2), target = -1 - 0.45 ln 2.')
case('one_action', [5.0], [-2.0], [0.75], 0, 0.5, 0.9, 0.9, 0.03, -1.0,
     0.0, 0.5 + 0.9 * -2.0,
     'A = 1: pi = 1, tau log pi = 0, bonus 0; boot = qbar_t = -2. target = 0.5 - 1.8 = -1.3.')
case('wide_q_small_tau_greedy', [0.0, 50.0, 100.0], [-100.0, 0.0, 100.0], [1.0, 2.0, 3.0], 2, 0.0, 0.99, 0.9, 0.03,
     -1.0, 0.0, 0.99 * 100.0,
     'tau = 0.03, q spread 100: the other exponents are -3333 and -1667, exp underflows to 0 without overflow; '
     'tau log pi(2) = -0.03 ln 1 = 0, bonus 0; boot = 100 + 0.03 ln 1 = 100. target = 99.')
case('wide_q_small_tau_clipped', [0.0, 50.0, 100.0], [-100.0, 0.0, 100.0], [1.0, 2.0, 3.0], 0, 0.0, 0.99, 0.9, 0.03,
     -1.0, -0.9, -0.9 + 0.99 * 100.0,
     'tau log pi(0) = 0 - 100 - 0.03 ln 1 = -100 < l0: bonus = -0.9 (exp(100 / 0.03) would overflow in the naive '
     'form). target = -0.9 + 99 = 98.1.')
case('two_way_tie_at_s_t', [2.0, 2.0, 2.0, 2.0], [4.0, 4.0, -50.0, -60.0], [0.0, 0.0, 0.0, 1.5], 3, 0.25, 0.9, 0.5,
     0.1, -0.2, 0.5 * (-0.2 * LN2), 0.25 + 0.5 * (-0.2 * LN2) + 0.9 * (4.0 + 0.1 * LN2),
     'uniform pi over 4 actions at s_tm1: tau log pi = 0.1 ln(1/4) = -0.2 ln 2 = -0.1386, inside [l0, 0] = [-0.2, 0]: '
     'bonus = 0.5 * -0.2 ln 2. At s_t two actions tie at 4 and the others lie 540 and 640 temperatures below (exp '
     'underflows to 0): pi = 1/2 on each, qbar - tau log pi = 4 + 0.1 ln 2. '
     'target = 0.25 - 0.1 ln 2 + 0.9 (4 + 0.1 ln 2).')

if __name__ == '__main__':
  out = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'munchausen_hand_vectors.json')
  with open(out, 'w') as f:
    json.dump({'_about': 'Munchausen DQN targets computed by hand; see make_munchausen_hand_vectors.py', 'cases': cases},
              f, indent=1)
  print(out, len(cases))
