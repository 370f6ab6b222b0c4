"""GPU: pyprob_b200.diagnostics (csrc/diagnostics.cu) against the reference's outputs (tests/golden/diagnostics_golden.npz)
and against the numpy oracle (oracle/diagnostics.py) over chain counts, lengths, variables and value types, including
constant chains, chains constant but for one chain, and offset chains (1e6 + N(0, 1)); a long few-chain case; the list
and the single-Empirical forms; determinism; an LMH run end to end; AR(1) chains; and the errors."""
import math
import os

import numpy as np
import pytest
import torch

import pyprob_b200 as pyprob
from oracle import diagnostics as odiag
from pyprob_b200 import InferenceEngine, Model, diagnostics, ops
from pyprob_b200.distributions import Normal
from pyprob_b200.empirical import Empirical

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = ['gum_lmh', 'gum_rmh', 'two_lmh', 'two_rmh']


def _same(got, want, tol, scale=0.0):
    """Same NaN / inf pattern; where want is finite |got - want| <= tol * max(scale, |want|).  R-hat is compared
    relatively (scale 0).  An autocorrelation lies in [-1, 1] with r(0) ~ 1 its natural unit, and a near-zero r is a
    cancelling sum, so it is compared relative to max(1, |want|) (scale 1)."""
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    assert got.shape == want.shape, (got.shape, want.shape)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
    inf = np.isinf(want)
    np.testing.assert_array_equal(got[inf], want[inf])
    fin = np.isfinite(want)
    assert np.isfinite(got[fin]).all()
    err = np.abs(got[fin] - want[fin]) / np.maximum(scale, np.abs(want[fin]))
    assert err.size == 0 or err.max() <= tol, (err.max(), np.argmax(err))


def _posterior_empirical(vals, C):
    """An Empirical laid out like posterior(..., num_chains=C): vals [S, C] or [S, C, V] -> [S * C] or [S * C, V]."""
    e = Empirical(vals.reshape(vals.shape[0] * C, *vals.shape[2:]), None)
    e.add_metadata(op='posterior', num_chains=C)
    return e


# ---- the reference's fixture --------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def golden():
    return dict(np.load(os.path.join(ROOT, 'tests', 'golden', 'diagnostics_golden.npz')))


def _names(g, case):
    return ['mu'] if case.startswith('gum') else ['mu', 's']


@pytest.mark.parametrize('case', CASES)
def test_reference_fixture_through_the_kernels(golden, case):
    g = golden
    names = _names(g, case)
    vals = np.stack([g['{}/values/{}'.format(case, n)] for n in names], axis=-1)       # [4, S, V]
    x = torch.from_numpy(vals).cuda().permute(1, 0, 2)                                  # [S, 4, V]
    for kind in ('', '_custom'):
        rh = ops.diag_rhat(x, g[case + '/iters' + kind]).cpu().numpy()
        ac = ops.diag_autocorr(x, g[case + '/lags' + kind]).cpu().numpy()
        for i, n in enumerate(names):
            _same(rh[i], g['{}/rhat{}/{}'.format(case, kind, n)], 1e-10)
            _same(ac[i], g['{}/acf{}/{}'.format(case, kind, n)], 1e-10, 1.0)
    # the public interface in the reference's form: a list of one-chain Empiricals, one Empirical per autocorrelation
    chains = [Empirical(x[:, c].contiguous(), None) for c in range(4)]
    iters, res = diagnostics.gelman_rubin(chains, names=names)
    np.testing.assert_array_equal(iters, g[case + '/iters'])
    for n in names:
        _same(res[n]['rhat'], g['{}/rhat/{}'.format(case, n)], 1e-10)
    lags, res = diagnostics.autocorrelation(chains[1], names=names, lags=g[case + '/lags_custom'])
    for n in names:
        assert res[n]['autocorrelation'].shape == (len(lags),)
        _same(res[n]['autocorrelation'], g['{}/acf_custom/{}'.format(case, n)][1], 1e-10, 1.0)


# ---- shapes, types and edge data against the oracle ---------------------------------------------------------------------

SHAPES = [(C, S) for C in (2, 3, 31, 32, 33, 1000, 65536) for S in (1, 2, 3, 1000, 10007) if C * S <= 10 ** 8]
DTYPES = [torch.float32, torch.float64, torch.int64]


def _data(C, S, V, dtype, k, gen):
    """[S, C, V].  V = 1: by k, general chains (noise + a slow walk + a per-chain offset), offset chains 1e6 + N(0, 1), or
    constant chains (c % 2).  V = 3: general or offset, constant except chain 0, every chain the same constant."""
    def general():
        walk = torch.randn(S, C, generator=gen, dtype=torch.float64).cumsum(0) * 0.05
        return torch.randn(S, C, generator=gen, dtype=torch.float64) + walk + \
            torch.randn(1, C, generator=gen, dtype=torch.float64) * 0.3

    def offset():
        return 1e6 + torch.randn(S, C, generator=gen, dtype=torch.float64)

    if V == 1:
        cols = [[general, offset, lambda: (torch.arange(C, dtype=torch.float64) % 2).expand(S, C)][k % 3]()]
    else:
        one = torch.full((S, C), 2.5, dtype=torch.float64)
        one[:, 0] = torch.randn(S, generator=gen, dtype=torch.float64)
        cols = [general() if k % 2 == 0 else offset(), one, torch.full((S, C), 2.5, dtype=torch.float64)]
    x = torch.stack(cols, -1)
    if dtype == torch.int64:
        x = (x * 10).round()
    return x.to(dtype).cuda()


def _iters_lags(S, C):
    rng = np.random.default_rng(S * 7 + C)
    iters = rng.permutation(np.unique([1, S, S + 1, 3 * S + 5, max(1, S // 2), min(S, 7)]))
    if S <= 3:
        lags = rng.permutation(np.arange(S + 1))
    else:
        lags = rng.permutation(np.unique([0, 1, 2, S // 3, S - 1, S]))
    small = C * S <= 2 * 10 ** 6          # the defaults too where the oracle is quick
    return iters, lags, small


@pytest.mark.parametrize('C,S', SHAPES)
def test_against_oracle(C, S):
    gen = torch.Generator().manual_seed(C * 100003 + S)
    iters, lags, small = _iters_lags(S, C)
    for k, V in enumerate((1, 3) if C * S <= 10 ** 7 else (1,)):   # host memory of the oracle
        dtype = DTYPES[(SHAPES.index((C, S)) + k) % 3]
        x = _data(C, S, V, dtype, SHAPES.index((C, S)) + k, gen)
        post = _posterior_empirical(x, C)
        xs = x.double().cpu().numpy().transpose(2, 1, 0)                   # [V, C, S]
        names = ['a', 'b', 'c'][:V]
        for it in ([iters] + ([None] if small else [])):
            got_iters, res = diagnostics.gelman_rubin(post, names=names, iters=it)
            for i, n in enumerate(names):
                assert res[n]['values'].shape == (C, S) and res[n]['values'].dtype == dtype
                _same(res[n]['rhat'], odiag.r_hats(xs[i], got_iters), 1e-9)
        for lg in ([lags] + ([None] if small else [])):
            got_lags, res = diagnostics.autocorrelation(post, names=names, lags=lg)
            for i, n in enumerate(names):
                want = odiag.autocorrelation(xs[i], got_lags)
                _same(res[n]['autocorrelation'], want, 1e-9, 1.0)


def test_rhat_at_every_iteration():
    """Per-iteration curves.  With few chains the segments end on every iteration; at C = 65,536 the statistics per
    (chain, iteration) would pass 256 MiB, so the segments containing iterations are read again from the values piece by
    piece (checked against the oracle at a subset of the iterations, where the oracle is quick)."""
    for C, S, V, dtype, check in ((64, 1000, 3, torch.float32, None), (3, 5000, 3, torch.float64, None),
                                  (300, 700, 3, torch.int64, None), (65536, 260, 1, torch.float32, 40)):
        gen = torch.Generator().manual_seed(C + S)
        x = _data(C, S, V, dtype, 0, gen)
        post = _posterior_empirical(x, C)
        xs = x.double().cpu().numpy().transpose(2, 1, 0)
        iters = np.random.default_rng(C).permutation(np.arange(1, S + 3))
        _, res = diagnostics.gelman_rubin(post, iters=iters)
        sel = np.arange(len(iters)) if check is None else np.random.default_rng(S).choice(len(iters), check, False)
        for i in range(V):
            _same(res[i]['rhat'][sel], odiag.r_hats(xs[i], iters[sel]), 1e-9)


def test_long_few_chains():
    C, S = 4, 10 ** 6
    gen = torch.Generator().manual_seed(5)
    x = _data(C, S, 1, torch.float32, 0, gen)
    post = _posterior_empirical(x, C)
    xs = x.double().cpu().numpy()[:, :, 0].T
    iters, res = diagnostics.gelman_rubin(post)
    _same(res[0]['rhat'], odiag.r_hats(xs, iters), 1e-9)
    lags, res = diagnostics.autocorrelation(post)
    _same(res[0]['autocorrelation'], odiag.autocorrelation(xs, lags), 1e-9, 1.0)


# ---- forms, views and determinism ---------------------------------------------------------------------------------------

def test_list_and_single_forms_are_bit_identical_and_repeatable():
    C, S, V = 33, 1000, 3
    gen = torch.Generator().manual_seed(11)
    x = _data(C, S, V, torch.float32, 0, gen)
    post = _posterior_empirical(x, C)
    chains = [Empirical(x[:, c].contiguous(), None) for c in range(C)]
    _, a = diagnostics.gelman_rubin(post)
    _, b = diagnostics.gelman_rubin(chains)
    _, a2 = diagnostics.gelman_rubin(post)
    for j in range(V):
        np.testing.assert_array_equal(a[j]['rhat'].view(np.int64), b[j]['rhat'].view(np.int64))
        np.testing.assert_array_equal(a[j]['rhat'].view(np.int64), a2[j]['rhat'].view(np.int64))
        assert torch.equal(a[j]['values'], b[j]['values'])
        # the single form's values are a view of the Empirical's: no copy
        assert a[j]['values'].data_ptr() == post.values.data_ptr() + j * post.values.element_size()
    _, r1 = diagnostics.autocorrelation(post)
    _, r2 = diagnostics.autocorrelation(post)
    for j in range(V):
        np.testing.assert_array_equal(r1[j]['autocorrelation'].view(np.int64), r2[j]['autocorrelation'].view(np.int64))
    # a slice that starts at a multiple of C keeps the chains; num_chains= overrides the metadata
    _, s = diagnostics.gelman_rubin(post[100 * C:], iters=[S - 100])
    _, t = diagnostics.gelman_rubin(Empirical(post.values[100 * C:], None), num_chains=C, iters=[S - 100])
    _, u = diagnostics.gelman_rubin(_posterior_empirical(x[100:].contiguous(), C), iters=[S - 100])
    for j in range(V):
        np.testing.assert_array_equal(s[j]['rhat'], t[j]['rhat'])
        np.testing.assert_array_equal(s[j]['rhat'], u[j]['rhat'])


class GUM(Model):
    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)), name='mu')
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


def test_lmh_end_to_end():
    """GUM under LMH, 1024 chains of 2000 steps, burn-in 500: the kernels on the posterior equal the oracle on its values.
    LMH proposes from the prior Normal(1, sqrt 5), far from the posterior N(7.25, 0.91): few proposals are accepted and a
    chain that reached the posterior's upper tail stays there for long, so R-hat approaches 1 slowly (a numpy
    independence sampler of the same law gives 1.13 at 1500 kept steps, 1.04 at 5000 and 1.01 at 19500).  The test
    asserts that decline here, and R-hat < 1.01 on i.i.d. draws of the posterior laid out the same way."""
    C = 1024
    pyprob.seed(3)
    post = GUM().posterior(2000, inference_engine=InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS, num_chains=C,
                           observe={'obs0': 8, 'obs1': 9}, map_func=lambda t: t.named_variables['mu'].value)
    kept = post[500 * C:]
    iters, res = diagnostics.gelman_rubin(kept, names=['mu'])
    rhat = res['mu']['rhat']
    assert 1.0 < rhat[-1] < 1.25 and (np.diff(rhat[-8:]) < 0).all(), rhat[-8:]
    xs = kept.values.double().reshape(-1, C).t().cpu().numpy()
    _same(rhat, odiag.r_hats(xs, iters), 1e-9)
    lags, res = diagnostics.autocorrelation(kept, names=['mu'])
    _same(res['mu']['autocorrelation'], odiag.autocorrelation(xs, lags), 1e-9, 1.0)
    iid = _posterior_empirical(7.25 + math.sqrt(1 / 1.2) * torch.randn(1500, C, device='cuda'), C)
    _, res = diagnostics.gelman_rubin(iid, names=['mu'])
    assert res['mu']['rhat'][-1] < 1.01


def test_ar1_autocorrelation():
    """AR(1) chains x_t = rho x_{t-1} + e_t started in the stationary law.  Per chain, E r_k = rho^k (S - k) / S up to
    the bias of subtracting the sample mean from numerator and denominator, each O(Var(mean) / gamma_0) =
    O((1 + rho) / ((1 - rho) S)); 4 (1 + rho) / ((1 - rho) S) bounds both.  r_k has standard deviation at most
    sqrt((1 + rho^2) / ((1 - rho^2) S)) (Bartlett), so the mean over C chains is within 5 / sqrt(C) of that."""
    rho, C, S = 0.9, 1024, 10000
    rng = np.random.default_rng(17)
    x = np.empty((S, C))
    x[0] = rng.standard_normal(C) / math.sqrt(1 - rho * rho)
    e = rng.standard_normal((S, C))
    for t in range(1, S):
        x[t] = rho * x[t - 1] + e[t]
    post = _posterior_empirical(torch.from_numpy(x).cuda(), C)
    lags = np.arange(21)
    _, res = diagnostics.autocorrelation(post, lags=lags)
    mean_r = res[0]['autocorrelation'].mean(axis=0)
    want = rho ** lags * (S - lags) / S
    bound = 4 * (1 + rho) / ((1 - rho) * S) + 5 * math.sqrt((1 + rho * rho) / ((1 - rho * rho) * S * C))
    assert np.abs(mean_r - want).max() <= bound, (np.abs(mean_r - want).max(), bound)


# ---- errors ---------------------------------------------------------------------------------------------------------------

def test_errors():
    C, S = 4, 50
    x = torch.randn(S, C, dtype=torch.float64, device='cuda')
    post = _posterior_empirical(x, C)
    with pytest.raises(ValueError, match='at least two chains'):
        diagnostics.gelman_rubin(Empirical(x[:, 0].contiguous(), None))
    with pytest.raises(ValueError, match='at least two chains'):
        diagnostics.gelman_rubin([Empirical(x[:, 0].contiguous(), None)])
    with pytest.raises(ValueError, match='multiple of num_chains'):
        diagnostics.gelman_rubin(post[3:])
    with pytest.raises(ValueError, match='multiple of num_chains'):
        diagnostics.autocorrelation(post, num_chains=7)
    with pytest.raises(ValueError, match='lags'):
        diagnostics.autocorrelation(post, lags=[0, S + 1])
    with pytest.raises(ValueError, match='lags'):
        diagnostics.autocorrelation(post, lags=[-1, 2])
    with pytest.raises(ValueError, match='iters'):
        diagnostics.gelman_rubin(post, iters=[0, 5])
    with pytest.raises(ValueError, match='names'):
        diagnostics.gelman_rubin(post, names=['a', 'b'])
    with pytest.raises(ValueError, match='names'):
        diagnostics.autocorrelation(post, names=['a', 'b'])
    with pytest.raises(NotImplementedError, match='reference'):
        diagnostics.gelman_rubin(post, plot=True)
    with pytest.raises(NotImplementedError, match='reference'):
        diagnostics.autocorrelation(post, plot=True)
    # lag S is allowed (an empty numerator), iters above S mean S
    _, r = diagnostics.autocorrelation(post, lags=[S])
    assert (r[0]['autocorrelation'] == 0).all()
    _, a = diagnostics.gelman_rubin(post, iters=[S, S + 10])
    assert a[0]['rhat'][0] == a[0]['rhat'][1]
