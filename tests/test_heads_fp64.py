"""CPU: the plain restatement of the proposal heads (tests/heads_fp64.py) against the project's earlier evidence — the fp32
oracle's head_log_prob / head_params (oracle/network.py, tests/bernoulli_oracle.py) at benign head outputs, and the
proposals that the unmodified reference recorded in tests/golden/infer_golden.npz — and its own edge behaviour."""
import math
from unittest import mock

import numpy as np
import pytest
import torch

from oracle import network as onet
from tests import bernoulli_oracle as bo
from tests import heads_fp64 as hf
from tests.test_oracle_infer import load_infer_golden

EPS32 = hf.EPS32


def _params_emitting(x):
    """A head whose output is exactly x for every input row: zero weights, bias x."""
    x = torch.as_tensor(np.asarray(x, np.float32))
    p = '_layers_proposal.a._ff._layers.'
    return {p + '0.weight': torch.zeros(1, 1), p + '0.bias': torch.zeros(1),
            p + '1.weight': torch.zeros(x.numel(), 1), p + '1.bias': x}


def _oracle_row(family, x, v, p0, p1, K, C):
    """fp32 oracle: log q and d(-log q)/dx of one row, autograd through the head bias."""
    params = _params_emitting(x)
    b = params['_layers_proposal.a._ff._layers.1.bias'].requires_grad_(True)
    lp = bo.head_log_prob(params, 'a', family, C, K, torch.zeros(1, 1), torch.tensor([v], dtype=torch.float32),
                          torch.tensor([p0], dtype=torch.float32), torch.tensor([p1], dtype=torch.float32))[0]
    (-lp).backward()
    q = bo.head_params(params, 'a', family, K, torch.zeros(1, 1), [p0], [p1])
    return float(lp), b.grad.double().numpy(), tuple(t[0].detach().double().numpy() for t in q)


def _benign_rows():
    rng = np.random.default_rng(5)
    rows = []
    for K in (1, 3, 10):
        for _ in range(4):
            x = rng.normal(0, 1, 3 * K).astype(np.float32)
            p0, p1 = float(rng.normal()), float(rng.uniform(0.5, 2))
            rows.append(('Normal', x, p0 + p1 * rng.normal(), p0, p1, K, 0))
            lo = float(rng.uniform(-2, 0))
            hi = lo + float(rng.uniform(0.5, 3))
            rows.append(('Uniform', x, lo + (hi - lo) * rng.uniform(0.05, 0.95), lo, hi, K, 0))
            rows.append(('Poisson', x, float(rng.poisson(3)), 0.0, 0.0, K, 0))
    for C in (2, 5, 33):
        for _ in range(3):
            rows.append(('Categorical', rng.normal(0, 1, C).astype(np.float32), float(rng.integers(0, C)), 0.0, 0.0, 0, C))
    for x in (-2.0, 0.3, 4.0):
        for v in (0.0, 1.0):
            rows.append(('Bernoulli', np.array([x], np.float32), v, 0.0, 0.0, 0, 0))
    return rows


@pytest.mark.parametrize('row', range(len(_benign_rows())))
def test_matches_fp32_oracle_at_benign_rows(row):
    family, x, v, p0, p1, K, C = _benign_rows()[row]
    lp32, g32, q32 = _oracle_row(family, x, v, p0, p1, K, C)
    got = hf.head(family, x, v, p0, p1, K=K or None, num_categories=C)
    # the oracle rounds every operation to fp32: a few ulps of the row's largest term (|log q| and its parts are O(10) here)
    assert abs(got['lp'] - lp32) <= 64 * EPS32 * (1 + abs(got['lp'])), (got['lp'], lp32)
    np.testing.assert_allclose(got['grad'], g32, rtol=1e-4, atol=1e-5 * (1 + np.abs(g32).max()))
    for a, b in zip(got['params'], q32):
        # a few rounded operations; p0 + sigmoid(x) (p1 - p0) rounds on the scale of the priors
        np.testing.assert_allclose(a, b, rtol=16 * EPS32, atol=16 * EPS32 * (1 + abs(p0) + abs(p1)))
    same = hf.head(family, x, v, p0, p1, K=K or None, num_categories=C, dtype=torch.float32)
    assert same['lp'] == pytest.approx(lp32, rel=1e-6, abs=1e-6)   # the float32 form is the oracle's arithmetic


def test_matches_reference_infer_step_proposals():
    """The raw head outputs the oracle's LSTM replay produces for the fixture's traces, through this module, give the
    means, stddevs, probs and log q that the unmodified reference recorded."""
    fx = load_infer_golden()
    seen = set()
    for tr in fx['traces']:
        xs = []
        with mock.patch.object(onet, 'head_params', _capture(xs)):
            onet.infer_sequence(fx['params'], tr['obs'], fx['observe_names'], fx['observe_in_dims'], fx['K'], tr['steps'])
        for st, x in zip(tr['steps'], xs):
            fam = st['family']
            seen.add(fam)
            got = hf.head(fam, x.numpy(), st['value'], st['prior0'], st['prior1'], K=fx['K'] if fam in hf.MIXTURES else None,
                          num_categories=st['num_categories'])
            want = st['want']
            if fam == 'Categorical':
                np.testing.assert_allclose(got['params'][0] / got['params'][0].sum(), want['probs'], rtol=1e-5, atol=1e-7)
            else:
                for a, k in zip(got['params'], ('means', 'stddevs', 'probs')):
                    np.testing.assert_allclose(a, want[k], rtol=1e-5, atol=1e-6)
            # the reference's fp32 log q against the unrounded one
            assert got['lp'] == pytest.approx(float(want['log_prob_of_value']), rel=1e-4, abs=1e-5)
    assert seen == {'Uniform', 'Categorical', 'Normal', 'Poisson'}


def _capture(xs):
    orig = onet.head_params

    def f(params, address, family, K, h, prior0, prior1):
        xs.append(onet._ff(h, params, '_layers_proposal.{}._ff'.format(address), False)[0].detach())
        return orig(params, address, family, K, h, prior0, prior1)
    return f


def test_gradient_matches_finite_differences():
    """fp64 autograd through the restated formulas against central differences, one row per family."""
    rng = np.random.default_rng(9)
    for family, x, v, p0, p1, K, C in [('Normal', rng.normal(0, 1, 9), 0.4, 0.1, 1.5, 3, 0),
                                       ('Uniform', rng.normal(0, 1, 9), 0.2, -1.0, 2.0, 3, 0),
                                       ('Poisson', rng.normal(0, 1, 9), 7.0, 0.0, 0.0, 3, 0),
                                       ('Categorical', rng.normal(0, 1, 6), 4.0, 0.0, 0.0, 0, 6),
                                       ('Bernoulli', [0.7], 1.0, 0.0, 0.0, 0, 0)]:
        x = np.asarray(x, np.float32)
        g = hf.head(family, x, v, p0, p1, K=K or None, num_categories=C)['grad']
        for j in range(len(x)):
            def f(d):
                xt = torch.tensor(x, dtype=torch.float64)
                xt[j] += d
                q = hf.proposal(family, xt, K, torch.tensor(float(np.float32(p0)), dtype=torch.float64),
                                torch.tensor(float(np.float32(p1)), dtype=torch.float64))
                return -float(hf.log_prob(family, q, v, torch.tensor(float(np.float32(p0)), dtype=torch.float64),
                                          torch.tensor(float(np.float32(p1)), dtype=torch.float64), C))
            fd = (f(1e-6) - f(-1e-6)) / 2e-6
            assert g[j] == pytest.approx(fd, rel=1e-5, abs=1e-7), (family, j)


def test_edges():
    # -inf (a Uniform value outside its range; Poisson 41) is repaired with a zero gradient
    for fam, v, p0, p1 in (('Uniform', 2.5, 0.0, 2.0), ('Poisson', 41.0, 0.0, 0.0)):
        r = hf.head(fam, np.zeros(6, np.float32), v, p0, p1)
        assert r['repaired'] and r['lp'] == hf.LOG_EPSILON and not r['grad'].any()
    # out-of-support Categorical / Bernoulli values score NaN
    assert math.isnan(hf.head('Categorical', np.zeros(4, np.float32), 4.0)['lp'])
    assert math.isnan(hf.head('Bernoulli', np.zeros(1, np.float32), 0.5)['lp'])
    # the mixture-weight clamp: a weight below the fp32 epsilon contributes log(eps) and no gradient to its logit
    x = np.array([0, 0, 0, 0, 0, 0, 0, 0, -20], np.float32)      # K = 3, identical components, weights (1/2, 1/2, ~1e-9)
    r = hf.head('Normal', x, 0.0, 0.0, 1.0)
    ph = math.exp(-20) / (2 + math.exp(-20))
    assert ph < EPS32
    # d(-lp)/dx_p of the clamped weight comes only through the softmax normaliser: prob_2 * (sum of the other responsibilities)
    assert r['grad'][8] == pytest.approx(ph, rel=1e-6)
    # Bernoulli beyond |x| ~ 15.9: the clamp is active and the gradient is zero
    assert hf.head('Bernoulli', np.array([17.0], np.float32), 1.0)['grad'][0] == 0.0
    assert hf.head('Bernoulli', np.array([15.0], np.float32), 1.0)['grad'][0] != 0.0
