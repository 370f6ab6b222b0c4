"""CPU: oracle/diagnostics.py restates the reference's Gelman-Rubin R-hat (pyprob/diagnostics.py:788-802) and
autocorrelation (:720-736); pinned to tests/golden/diagnostics_golden.npz, recorded from the unmodified reference
(tests/golden/make_diagnostics_golden.py: GUM and a two-variable model under LMH and RMH, four chains each)."""
import os

import numpy as np
import pytest

from oracle import diagnostics

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-12
CASES = ['gum_lmh', 'gum_rmh', 'two_lmh', 'two_rmh']


@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'diagnostics_golden.npz')))


def _names(g, case):
    return sorted(k.split('/')[-1] for k in g if k.startswith(case + '/values/'))


def _same(got, want):
    """equal NaN / inf pattern, and within TOL relative (to max(1, |want|)) where finite"""
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape
    fin = np.isfinite(want)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    np.testing.assert_array_equal(got[~fin & ~np.isnan(want)], want[~fin & ~np.isnan(want)])
    err = np.abs(got[fin] - want[fin]) / np.maximum(1.0, np.abs(want[fin]))
    assert err.size == 0 or err.max() <= TOL, err.max()


def test_fixture_covers_cases_and_edges(golden):
    g = golden
    assert _names(g, 'gum_lmh') == ['mu'] and _names(g, 'two_rmh') == ['mu', 's']
    for case in CASES:
        S = g[case + '/values/mu'].shape[1]
        assert g[case + '/values/mu'].shape == (4, S)
        assert 1 in g[case + '/iters_custom'] and S in g[case + '/iters_custom']
        assert 0 in g[case + '/lags_custom'] and S in g[case + '/lags_custom']
        assert np.isnan(g[case + '/rhat/mu'][0])                       # one-step prefix
    rh = np.concatenate([g[c + '/rhat/' + n] for c in CASES for n in _names(g, c)])
    assert np.isinf(rh).any() and np.isfinite(rh).sum() > 100         # chains that have not moved yet: w = 0


@pytest.mark.parametrize('case', CASES)
def test_r_hat_matches_reference(golden, case):
    g = golden
    for n in _names(g, case):
        values = g['{}/values/{}'.format(case, n)]
        _same(diagnostics.r_hats(values, g[case + '/iters']), g['{}/rhat/{}'.format(case, n)])
        _same(diagnostics.r_hats(values, g[case + '/iters_custom']), g['{}/rhat_custom/{}'.format(case, n)])


@pytest.mark.parametrize('case', CASES)
def test_autocorrelation_matches_reference(golden, case):
    g = golden
    for n in _names(g, case):
        values = g['{}/values/{}'.format(case, n)]
        _same(diagnostics.autocorrelation(values, g[case + '/lags']), g['{}/acf/{}'.format(case, n)])
        _same(diagnostics.autocorrelation(values, g[case + '/lags_custom']), g['{}/acf_custom/{}'.format(case, n)])
        # and one chain at a time, the reference's shape
        _same(diagnostics.autocorrelation(values[0], g[case + '/lags']), g['{}/acf/{}'.format(case, n)][0])


def test_default_iters_and_lags_are_the_reference_expressions(golden):
    S = golden['gum_lmh/values/mu'].shape[1]
    np.testing.assert_array_equal(golden['gum_lmh/iters'], np.unique(np.logspace(0, np.log10(S)).astype(int)))
    np.testing.assert_array_equal(golden['gum_lmh/lags'], np.unique(np.logspace(0, np.log10(S / 2)).astype(int)))


def test_oracle_edges():
    with pytest.raises(ValueError, match='at least two chains'):
        diagnostics.r_hat(np.zeros((1, 5)))
    assert np.isnan(diagnostics.r_hat(np.full((3, 4), 2.5)))                  # w = 0 and b = 0
    assert np.isinf(diagnostics.r_hat(np.array([[1.0, 1.0], [2.0, 2.0]])))  # w = 0, b > 0
    np.testing.assert_array_equal(diagnostics.autocorrelation(np.full(6, 3.0), [0, 2, 6]), [0.0, 0.0, 0.0])
