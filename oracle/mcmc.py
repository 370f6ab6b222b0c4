"""Oracle: the Metropolis-Hastings acceptance ratio of the reference's LMH / RMH (TEST INFRASTRUCTURE ONLY).

Restates pyprob/model.py:149-160 (log alpha) and pyprob/state.py:235-256 (the RMH site transition term) in fp64 from
recorded traces, so that a test can recompute what the engine decided from the traces it decided on.
"""
import math

import numpy as np

ALPHA = 0.5      # state.py:247


def normal_log_prob(x, loc, scale):
    return -((x - loc) ** 2) / (2.0 * scale * scale) - math.log(scale) - 0.5 * math.log(2 * math.pi)


def _std_normal_cdf(x):
    return 0.5 * (1.0 + math.erf(x / math.sqrt(2.0)))


def truncated_normal_log_prob(x, loc, scale, low, high):
    """pyprob/distributions/truncated_normal.py:24-45"""
    if not (low <= x <= high):
        return -math.inf
    z = (x - loc) / scale
    Z = _std_normal_cdf((high - loc) / scale) - _std_normal_cdf((low - loc) / scale)
    return -(z * z) / 2.0 - 0.5 * math.log(2 * math.pi) - math.log(scale * Z)


def _log_mix(a, b):
    """log(ALPHA e^a + (1 - ALPHA) e^b)"""
    p, q = math.log(ALPHA) + a, math.log(1 - ALPHA) + b
    m = max(p, q)
    return -math.inf if m == -math.inf else m + math.log(math.exp(p - m) + math.exp(q - m))


def rmh_transition(family, x_old, lp_old, x_new, lp_new, p0, p1):
    """The RMH site term of state.py:255-256.  family 'Normal': p0, p1 = loc, scale of the prior; 'Uniform': low, high.
    lp_old is the chosen site's log-prob in the current trace, lp_new the new value's under the candidate's prior."""
    if family == 'Normal':
        def q(a, b):
            return normal_log_prob(a, b, p1)
    elif family == 'Uniform':
        def q(a, b):
            return truncated_normal_log_prob(a, b, 0.1 * (p1 - p0), p0, p1)
    else:
        return 0.0
    return _log_mix(q(x_old, x_new), lp_old) + lp_new - _log_mix(q(x_new, x_old), lp_new) - lp_old


def log_acceptance(cur_num_controlled, cand_num_controlled, cur_log_prob_observed, cand_log_prob_observed,
                   reused_lp_cand, reused_lp_cur, transition):
    """model.py:151-162: log|cur| - log|cand| + lpo_cand - lpo_cur + sum over reused sites (lp_cand - lp_cur) + transition."""
    la = math.log(cur_num_controlled) - math.log(cand_num_controlled) + cand_log_prob_observed - cur_log_prob_observed
    la += float(np.sum(np.asarray(reused_lp_cand, dtype=np.float64) - np.asarray(reused_lp_cur, dtype=np.float64)))
    return la + transition
