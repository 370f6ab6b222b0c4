"""CPU: oracle/mcmc.py restates the reference's LMH / RMH acceptance ratio (pyprob/model.py:151-162) and RMH site
transition term (pyprob/state.py:235-256); pinned to tests/golden/mcmc_golden.npz, recorded from the unmodified
reference (tests/golden/make_mcmc_golden.py)."""
import math
import os

import numpy as np
import pytest

from oracle import mcmc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RTOL = 1e-6


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'mcmc_golden.npz')))


def _close(a, b):
    return abs(a - b) <= RTOL * max(1.0, abs(a), abs(b))


def test_fixture_covers_models_engines_reuse_and_kernels(golden):
    g = golden
    assert set(np.unique(g['step/model'])) == {0, 1, 2, 3} and set(np.unique(g['step/engine'])) == {0, 1}
    assert g['site/reused'].sum() > 0
    rmh_kernel = (g['step/engine'] == 1) & np.isin(g['step/family'], (0, 1)) & ~np.isnan(g['step/transition'])
    assert np.any(rmh_kernel & (g['step/family'] == 0)) and np.any(rmh_kernel & (g['step/family'] == 1))
    assert np.any(g['step/cur_n'] != g['step/cand_n'])       # the loop and the branch change |controlled|


def test_log_acceptance_matches_reference(golden):
    g = golden
    for s in range(len(g['step/model'])):
        sel = g['site/step'] == s
        cur = sel & (g['site/trace'] == 0)
        cand = sel & (g['site/trace'] == 1) & (g['site/reused'] == 1)
        cur_lp = dict(zip(g['site/address'][cur], g['site/log_prob'][cur]))
        reused_cand = g['site/log_prob'][cand]
        reused_cur = [cur_lp[a] for a in g['site/address'][cand]]
        t = g['step/transition'][s]
        la = mcmc.log_acceptance(g['step/cur_n'][s], g['step/cand_n'][s], g['step/cur_lpo'][s], g['step/cand_lpo'][s],
                                 reused_cand, reused_cur, 0.0 if np.isnan(t) else t)
        assert _close(la, g['step/log_alpha'][s]), (s, la, g['step/log_alpha'][s])


def test_rmh_transition_matches_reference(golden):
    g = golden
    checked = 0
    for s in range(len(g['step/model'])):
        t = g['step/transition'][s]
        if np.isnan(t):
            continue
        family = {0: 'Normal', 1: 'Uniform'}.get(int(g['step/family'][s]))
        if g['step/engine'][s] == 0 or family is None:
            assert t == 0.0          # LMH, and RMH at a family without a kernel: the prior proposal cancels
            continue
        got = mcmc.rmh_transition(family, g['step/x_old'][s], g['step/lp_old'][s], g['step/x_new'][s],
                                  g['step/lp_new'][s], g['step/p0'][s], g['step/p1'][s])
        # the reference computes the term in fp32 from fp32 log-probs: a few ulp of its largest summand
        scale = max(1.0, abs(g['step/lp_old'][s]), abs(g['step/lp_new'][s]))
        assert abs(got - t) <= 1e-6 * scale + 1e-6 * abs(t), (s, got, t)
        checked += 1
    assert checked > 20


def test_log_mix_limits():
    assert mcmc._log_mix(-math.inf, -math.inf) == -math.inf
    assert _close(mcmc._log_mix(0.0, 0.0), 0.0)
