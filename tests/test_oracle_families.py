"""CPU: the Exponential .. VonMises oracle (tests/families_oracle.py) against the UNMODIFIED reference
(tests/golden/families_golden.npz) and against the known answers of the reference's own tests/test_distributions.py."""
import math
import os

import numpy as np
import pytest
import torch

from tests import families_oracle as fo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'families_golden.npz')

# family -> (oracle, parameter names in the oracle's argument order)
FAMILIES = {
    'exponential': (fo.exponential_log_prob, ['rate']),
    'gamma': (fo.gamma_log_prob, ['concentration', 'rate']),
    'lognormal': (fo.lognormal_log_prob, ['loc', 'scale']),
    'weibull': (fo.weibull_log_prob, ['scale', 'concentration']),
    'beta': (fo.beta_log_prob, ['concentration1', 'concentration0']),
    'beta_lowhigh': (fo.beta_log_prob, ['concentration1', 'concentration0', 'low', 'high']),
    'binomial': (fo.binomial_log_prob, ['total_count', 'probs']),
    'binomial_logits': (lambda v, n, lg: fo.binomial_log_prob(v, n, logits=lg), ['total_count', 'logits']),
    'von_mises': (fo.von_mises_log_prob, ['loc', 'concentration']),
}


def load(family):
    g = np.load(GOLDEN)
    return {k.split('/', 1)[1]: g[k] for k in g.files if k.split('/', 1)[0] == family}


def check_same(got, want, rtol=1e-6, atol=0.0):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert np.array_equal(np.isnan(got), np.isnan(want)), np.nonzero(np.isnan(got) != np.isnan(want))
    assert np.array_equal(np.isposinf(got), np.isposinf(want))
    assert np.array_equal(np.isneginf(got), np.isneginf(want))
    fin = np.isfinite(want)
    np.testing.assert_allclose(got[fin], want[fin], rtol=rtol, atol=atol)


@pytest.mark.parametrize('family', sorted(FAMILIES))
def test_oracle_vs_reference_fixture(family):
    g = load(family)
    fn, names = FAMILIES[family]
    lp = fn(torch.from_numpy(g['value']), *[torch.from_numpy(g[k]) for k in names])
    check_same(lp.numpy(), g['lp'])


def test_fixture_covers_the_edges():
    g = load('gamma')
    assert np.isposinf(g['lp'][(g['value'] == 0) & (g['concentration'] == 0.5) & (g['rate'] > 0)]).all()
    assert np.isneginf(g['lp'][(g['value'] == 0) & (g['concentration'] == 2.7) & (g['rate'] > 0)]).all()
    b = load('beta')
    assert np.isposinf(b['lp'][(b['value'] == 1) & (b['concentration0'] == 0.1) & (b['concentration1'] > 0)]).all()
    v = load('von_mises')
    assert np.isfinite(v['lp'][v['concentration'] == 1e4]).all()
    assert np.isnan(load('exponential')['lp'][load('exponential')['value'] < 0]).all()
    n = load('binomial')
    assert np.isfinite(n['lp'][(n['value'] == n['total_count']) & (n['total_count'] == 1000) & (n['probs'] == 0)]).all()


# the reference's tests/test_distributions.py: (distribution, value) -> log_prob, mean, stddev (4 decimals there)
KNOWN = [
    (lambda v: fo.gamma_log_prob(v, 0.5, 1.2), 0.4167, -0.5435, 0.5 / 1.2, math.sqrt(0.5) / 1.2),
    (lambda v: fo.exponential_log_prob(v, 4.0), 0.25, 0.3863, 0.25, 0.25),
    (lambda v: fo.lognormal_log_prob(v, 0.5, 0.2), 1.6820, 0.1655, 1.6820, 0.3398),
    (lambda v: fo.weibull_log_prob(v, 1.1, 0.5), 2.2, -2.5492, 2.2, 4.9193),
    (lambda v: fo.beta_log_prob(v, 2.0, 5.0), 0.285714, 0.802545, 0.285714, 0.159719),
    # the low / high test's 0.546965 at 0.8 is not what the reference computes (0.4416, in the fixture), so not here
    (lambda v: fo.binomial_log_prob(v, 10.0, 0.2), 2.0, -1.1974, 2.0, 1.2649),
    (lambda v: fo.von_mises_log_prob(v, 3.1415, 2.0), 3.1415, -0.6619, 3.1415, None),
]


@pytest.mark.parametrize('i', range(len(KNOWN)))
def test_reference_known_answers(i):
    fn, value, lp, _, _ = KNOWN[i]
    assert abs(float(fn(value)) - lp) < 1e-4


def test_reference_moments():
    """The fixture's reference moments against closed forms and the reference's known answers (Exponential(1.5): mean
    0.6667 and median log(2) / 1.5 = 0.4621; Weibull(1.1, 0.5): mean 2.2, stddev 4.9193)."""
    e = load('exponential')
    ok = e['rate'] > 0
    np.testing.assert_allclose(e['mean'][ok], 1 / e['rate'][ok], rtol=1e-6)
    assert abs(1 / 1.5 - 0.666667) < 1e-6 and abs(math.log(2) / 1.5 - 0.462098) < 1e-6
    g = load('gamma')
    ok = (g['concentration'] > 0) & (g['rate'] > 0)
    np.testing.assert_allclose(g['mean'][ok], (g['concentration'] / g['rate'])[ok], rtol=1e-6)
    np.testing.assert_allclose(g['variance'][ok], (g['concentration'] / g['rate'] ** 2)[ok], rtol=1e-6)
    assert np.isnan(g['mean'][~ok]).all()
    b = load('beta_lowhigh')
    a, c = b['concentration1'], b['concentration0']
    np.testing.assert_allclose(b['mean'], -2 + 7 * a / (a + c), rtol=1e-5)
    np.testing.assert_allclose(b['variance'], 49 * a * c / ((a + c) ** 2 * (a + c + 1)), rtol=1e-5)
    w = load('weibull')
    sel = (w['scale'] == np.float32(1.1)) & (w['concentration'] == 0.5)
    assert abs(float(w['mean'][sel][0]) - 2.2) < 1e-4 and abs(math.sqrt(float(w['variance'][sel][0])) - 4.9193) < 1e-4
    v = load('von_mises')     # circular variance 1 - I1 / I0
    sel = (v['concentration'] == np.float32(1.1)) & (v['loc'] == 0)
    want = 1 - float(torch.special.i1e(torch.tensor(1.1)) / torch.special.i0e(torch.tensor(1.1)))
    assert abs(float(v['variance'][sel][0]) - want) < 1e-5
