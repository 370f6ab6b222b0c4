"""GPU: Exponential, Gamma, LogNormal, Weibull, Beta, Binomial and VonMises end to end: scoring and sampling kernels,
importance sampling with these families as priors and likelihoods, and inference compilation with them as uncontrolled
sites and observations.  References: the UNMODIFIED reference (tests/golden/families_golden.npz), torch.distributions,
scipy.stats, quadrature and the oracle in tests/families_oracle.py."""
import math
import warnings

import numpy as np
import pytest
import scipy.integrate
import scipy.special
import scipy.stats
import torch

import pyprob_b200 as pyprob
from pyprob_b200 import InferenceEngine, InferenceNetwork, Model, ops
from pyprob_b200.distributions import (Beta, Binomial, Exponential, Gamma, LogNormal, Normal, Poisson,
                                       TruncatedNormal, Uniform, VonMises, Weibull)
from pyprob_b200.util import TraceMode
from tests import families_oracle as fo
from tests.test_oracle_families import load

pytestmark = pytest.mark.gpu

gammaln = scipy.special.gammaln


# ---- scoring: reference fixture ------------------------------------------------------------------------------------------
def _scale(family, g):
    """Magnitude of the largest terms of each log_prob: fp32 rounding of those terms bounds how closely any fp32
    implementation (the reference's included) can agree."""
    v = g['value'].astype(np.float64)
    with np.errstate(all='ignore'):
        if family == 'exponential':
            r = g['rate']
            return np.abs(np.log(r)) + np.abs(r * v)
        if family == 'gamma':
            c, r = g['concentration'], g['rate']
            return np.abs(c * np.log(r)) + np.abs((c - 1) * np.log(v)) + np.abs(r * v) + np.abs(gammaln(c))
        if family == 'lognormal':
            m, s = g['loc'], g['scale']
            return (np.log(v) - m) ** 2 / (2 * s * s) + np.abs(np.log(s)) + np.abs(np.log(v))
        if family == 'weibull':
            x1 = v / g['scale']
            return np.abs(np.log(g['scale'])) + np.abs(g['concentration'] * np.log(x1)) + x1 ** g['concentration']
        if family in ('beta', 'beta_lowhigh'):
            a, b = g['concentration1'], g['concentration0']
            u = (v - g.get('low', 0.0)) / (g.get('high', 1.0) - g.get('low', 0.0))
            return (np.abs((a - 1) * np.log(u)) + np.abs((b - 1) * np.log1p(-u)) + np.abs(gammaln(a + b)) +
                    np.abs(gammaln(a)) + np.abs(gammaln(b)))
        if family == 'binomial':
            n, p = g['total_count'], np.clip(g['probs'], 1.2e-7, 1 - 1.2e-7)
            lg = np.abs(np.log(p) - np.log1p(-p))
            return (np.abs(v) + n) * lg + gammaln(v + 1) + gammaln(n - v + 1) + gammaln(n + 1)
        if family == 'von_mises':
            return g['concentration'] + np.abs(np.log(np.abs(scipy.special.i0e(g['concentration'])))) + 2.0
    raise KeyError(family)


def _close(got, want, scale, rtol=1e-5, stol=2e-6):
    got = got.detach().cpu().double().numpy() if torch.is_tensor(got) else np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    for f in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(f(got), f(want)), (f.__name__, np.nonzero(f(got) != f(want))[0][:10])
    fin = np.isfinite(want)
    scale = np.where(np.isfinite(scale), scale, 0.0)
    with np.errstate(invalid='ignore'):
        err = np.abs(got - want)[fin]
    tol = (rtol * np.abs(want) + stol * scale + 1e-6)[fin]
    assert (err <= tol).all(), (np.max(err - tol), np.nonzero(err > tol)[0][:10])


SCORE = {   # fixture family -> (kernel wrapper, parameter names in argument order)
    'exponential': (ops.exponential_log_prob, ['rate']),
    'gamma': (ops.gamma_log_prob, ['concentration', 'rate']),
    'lognormal': (ops.lognormal_log_prob, ['loc', 'scale']),
    'weibull': (ops.weibull_log_prob, ['scale', 'concentration']),
    'beta': (ops.beta_log_prob, ['concentration1', 'concentration0']),
    'beta_lowhigh': (ops.beta_log_prob, ['concentration1', 'concentration0', 'low', 'high']),
    'binomial': (ops.binomial_log_prob, ['total_count', 'probs']),
    'von_mises': (ops.von_mises_log_prob, ['loc', 'concentration']),
}


@pytest.mark.parametrize('family', sorted(SCORE))
def test_log_prob_vs_reference_fixture(cuda, family):
    """Every grid row, including values outside the support and invalid parameters (NaN where the reference raises)."""
    g = load(family)
    fn, names = SCORE[family]
    scale = _scale(family, g)
    v = torch.from_numpy(g['value']).to(cuda)
    params = [torch.from_numpy(g[k]).to(cuda) for k in names]
    _close(fn(v, *params), g['lp'], scale)
    _close(fn(v[1:], *[p[1:] for p in params]), g['lp'][1:], scale[1:])     # unaligned pointers: the scalar path


def test_binomial_from_logits_vs_reference_fixture(cuda):
    """Binomial(logits=) is scored from sigmoid(logits) in fp32.  The round trip through probs costs the logit a relative
    error of about 6e-8 exp(|logits|), which log_prob multiplies by up to total_count: at total_count = 1000 the values
    agree with the reference's raw-logits form for |logits| <= 5 and drift apart above (8.9 at logits = 12)."""
    g = load('binomial_logits')
    ok = np.abs(g['logits']) <= 5
    d = Binomial(torch.from_numpy(g['total_count']), logits=torch.from_numpy(g['logits']))
    lp = d.log_prob(torch.from_numpy(g['value']).to(cuda)).cpu().numpy()
    _close(lp[ok], g['lp'][ok], _scale('binomial', {'value': g['value'][ok], 'total_count': g['total_count'][ok],
                                                    'probs': 1 / (1 + np.exp(-g['logits'][ok]))}), rtol=1e-4)
    assert np.isfinite(lp[~ok]).all()


@pytest.mark.parametrize('family', sorted(SCORE))
def test_moments_vs_reference_fixture(cuda, family):
    g = load(family)
    _, names = SCORE[family]
    ok = np.isfinite(g['mean'])
    cls = {'exponential': Exponential, 'gamma': Gamma, 'lognormal': LogNormal, 'weibull': Weibull, 'beta': Beta,
           'beta_lowhigh': Beta, 'binomial': Binomial, 'von_mises': VonMises}[family]
    d = cls(*[torch.from_numpy(g[k][ok]) for k in names])
    for what in ('mean', 'variance'):
        got = getattr(d, what)
        got = got.cpu().double().numpy() if torch.is_tensor(got) else np.full(ok.sum(), got)
        want = g[what][ok].astype(np.float64)
        fin = np.isfinite(want)
        assert np.array_equal(np.isfinite(got), fin), what
        # LogNormal's variance (exp(s^2) - 1) exp(2 m + s^2) cancels in fp32 at small s: one ulp of exp is 6e-4 of it at
        # s = 0.01, so GPU and CPU exp differ there by up to 1e-3 relative
        rtol = 1e-3 if (family, what) == ('lognormal', 'variance') else 2e-5
        np.testing.assert_allclose(got[fin], want[fin], rtol=rtol, atol=1e-6, err_msg=what)
    m = cls(*[float(g[k][ok][0]) for k in names]).mean          # scalar parameters give Python floats
    assert isinstance(m, float) and abs(m - float(g['mean'][ok][0])) <= 2e-5 * abs(m) + 1e-6


# ---- scoring: sizes, scalar / per-particle parameters, acc form, against torch.distributions -----------------------------
def _random_case(family, n, gen):
    """(kernel, torch-CPU reference log_prob, value [n], params) with valid parameters and values inside the support."""
    def u(lo, hi):
        return lo + (hi - lo) * torch.rand(n, generator=gen)
    D = torch.distributions
    if family == 'exponential':
        r = u(0.2, 5)
        return ops.exponential_log_prob, lambda v, r: D.Exponential(r, validate_args=False).log_prob(v), \
            D.Exponential(r).sample(), [r]
    if family == 'gamma':
        c, r = u(0.2, 6), u(0.3, 3)
        return ops.gamma_log_prob, lambda v, c, r: D.Gamma(c, r, validate_args=False).log_prob(v), \
            D.Gamma(c, r).sample().clamp(min=1e-20), [c, r]
    if family == 'lognormal':
        m, s = u(-1, 1), u(0.2, 1.5)
        return ops.lognormal_log_prob, lambda v, m, s: D.LogNormal(m, s, validate_args=False).log_prob(v), \
            D.LogNormal(m, s).sample(), [m, s]
    if family == 'weibull':
        lam, k = u(0.5, 3), u(0.5, 4)
        return ops.weibull_log_prob, lambda v, lam, k: D.Weibull(lam, k, validate_args=False).log_prob(v), \
            D.Weibull(lam, k).sample().clamp(min=1e-20), [lam, k]
    if family == 'beta':
        a, b, lo = u(0.3, 6), u(0.3, 6), u(-2, 0)
        hi = lo + u(0.5, 4)
        x = lo + (hi - lo) * D.Beta(a, b).sample().clamp(1e-6, 1 - 1e-6)
        return ops.beta_log_prob, fo.beta_log_prob, x, [a, b, lo, hi]
    if family == 'binomial':
        nt = torch.randint(0, 60, (n,), generator=gen).float()
        p = u(0, 1)
        return ops.binomial_log_prob, lambda v, nt, p: D.Binomial(nt, probs=p, validate_args=False).log_prob(v), \
            D.Binomial(nt, probs=p).sample(), [nt, p]
    if family == 'von_mises':
        m, k = u(-3, 3), u(0.01, 40)
        return ops.von_mises_log_prob, lambda v, m, k: D.VonMises(m, k, validate_args=False).log_prob(v), \
            u(-10, 10), [m, k]
    raise KeyError(family)


FAMILIES = ['exponential', 'gamma', 'lognormal', 'weibull', 'beta', 'binomial', 'von_mises']


@pytest.mark.parametrize('n', [1, 7, 4096, 100003])
@pytest.mark.parametrize('family', FAMILIES)
def test_log_prob_vs_torch_sizes_and_acc(cuda, family, n):
    gen = torch.Generator().manual_seed(n + 17 * FAMILIES.index(family))
    fn, ref, v, params = _random_case(family, n, gen)
    tol = dict(rtol=1e-4, atol=1e-4, equal_nan=True)
    # per-particle parameters (vectorised path), then unaligned pointers (scalar path)
    want = ref(v, *params)
    torch.testing.assert_close(fn(v.to(cuda), *[p.to(cuda) for p in params]).cpu(), want, **tol)
    if n > 1:
        torch.testing.assert_close(fn(v.to(cuda)[1:], *[p.to(cuda)[1:] for p in params]).cpu(), want[1:], **tol)
    # shared (stride-0) parameters: the per-thread constant path
    scal = [float(p[0]) for p in params]
    if family == 'binomial':
        v = torch.minimum(v, torch.tensor(scal[0]))
    want = ref(v, *[torch.tensor(s) for s in scal])
    torch.testing.assert_close(fn(v.to(cuda), *scal).cpu(), want, **tol)
    # acc form: fp64 running sum of the fp32 terms
    acc = torch.full((n,), 0.25, dtype=torch.float64, device=cuda)
    fn(v.to(cuda), *scal, acc=acc, acc_scale=-1.0)
    lp = fn(v.to(cuda), *scal)
    assert torch.equal(acc.nan_to_num(), (0.25 - lp.double()).nan_to_num())


def test_outside_support_and_invalid_parameters_are_nan(cuda):
    def nan(t):
        return np.isnan(t.cpu().numpy())
    v = torch.tensor([-1.0, -1e-30, float('nan'), 1.0], device=cuda)
    assert nan(ops.exponential_log_prob(v, 2.0)).tolist() == [True, True, True, False]
    assert nan(ops.gamma_log_prob(v, 2.0, 1.0)).tolist() == [True, True, True, False]
    assert nan(ops.gamma_log_prob(v[3:], 0.0, 1.0)).all() and nan(ops.gamma_log_prob(v[3:], 1.0, -1.0)).all()
    w = torch.tensor([0.0, -1.0, 1.0], device=cuda)
    assert nan(ops.lognormal_log_prob(w, 0.0, 1.0)).tolist() == [True, True, False]
    assert nan(ops.weibull_log_prob(w, 1.0, 2.0)).tolist() == [True, True, False]
    assert nan(ops.lognormal_log_prob(w[2:], 0.0, 0.0)).all() and nan(ops.weibull_log_prob(w[2:], 1.0, 0.0)).all()
    b = torch.tensor([-2.1, -2.0, 5.0, 5.1], device=cuda)
    assert nan(ops.beta_log_prob(b, 2.0, 3.0, -2.0, 5.0)).tolist() == [True, False, False, True]
    assert nan(ops.beta_log_prob(b[1:2], 0.0, 3.0, -2.0, 5.0)).all()
    k = torch.tensor([-1.0, 0.0, 2.5, 10.0, 11.0], device=cuda)
    assert nan(ops.binomial_log_prob(k, 10.0, 0.3)).tolist() == [True, False, True, False, True]
    assert nan(ops.binomial_log_prob(k[1:2], 10.5, 0.3)).all() and nan(ops.binomial_log_prob(k[1:2], 10.0, 1.5)).all()
    assert nan(ops.von_mises_log_prob(k, 0.0, 0.0)).all() and not nan(ops.von_mises_log_prob(k, 0.0, 1.0)).any()


# ---- sampling -------------------------------------------------------------------------------------------------------------
# (id, sampler, log_prob kernel, parameters, scipy distribution, KS window (lo, hi) or None, support check)
def _pos(x):
    return (x > 0).all()


SAMPLERS = [('exponential-1.5', ops.exponential_sample, ops.exponential_log_prob, (1.5,), scipy.stats.expon(scale=1 / 1.5),
             None, lambda x: (x >= 0).all())]
for c in (0.05, 0.5, 1.0, 2.7, 100.0):
    SAMPLERS.append(('gamma-{}'.format(c), ops.gamma_sample, ops.gamma_log_prob, (c, 2.0),
                     scipy.stats.gamma(c, scale=0.5), (1e-30, math.inf) if c < 0.1 else None, _pos))
for m, s in ((0.5, 0.2), (-1.0, 0.8)):
    SAMPLERS.append(('lognormal-{}-{}'.format(m, s), ops.lognormal_sample, ops.lognormal_log_prob, (m, s),
                     scipy.stats.lognorm(s, scale=math.exp(m)), None, _pos))
for k in (0.5, 1.1, 3.0):
    SAMPLERS.append(('weibull-{}'.format(k), ops.weibull_sample, ops.weibull_log_prob, (1.1, k),
                     scipy.stats.weibull_min(k, scale=1.1), None, _pos))
for a, b, lo, hi in ((0.1, 0.1, 0.0, 1.0), (0.5, 1.0, 0.0, 1.0), (2.0, 5.0, 0.0, 1.0), (50.0, 50.0, 0.0, 1.0),
                     (2.0, 5.0, -2.0, 5.0)):
    SAMPLERS.append(('beta-{}-{}-{}-{}'.format(a, b, lo, hi), ops.beta_sample, ops.beta_log_prob, (a, b, lo, hi),
                     scipy.stats.beta(a, b, loc=lo, scale=hi - lo), (1e-6, 1 - 1e-5) if a < 0.5 else None,
                     lambda x, lo=lo, hi=hi: ((x >= lo) & (x <= hi)).all()))
for nt in (1.0, 10.0, 1000.0):
    for p in (0.01, 0.5, 0.97):
        SAMPLERS.append(('binomial-{}-{}'.format(nt, p), ops.binomial_sample, ops.binomial_log_prob, (nt, p),
                         scipy.stats.binom(int(nt), p), None,
                         lambda x, nt=nt: ((x >= 0) & (x <= nt) & (x == torch.floor(x))).all()))
for k in (1e-3, 1.1, 50.0):
    SAMPLERS.append(('von_mises-{}'.format(k), ops.von_mises_sample, ops.von_mises_log_prob, (0.5, k),
                     scipy.stats.vonmises(k), None, lambda x: ((x >= -math.pi - 1e-6) & (x <= math.pi + 1e-6)).all()))
SAMPLER_IDS = [s[0] for s in SAMPLERS]


def _wrap(x):
    return (x + np.pi) % (2 * np.pi) - np.pi


def _distribution_test(case, x):
    """KS (continuous) or chi-square (Binomial) against scipy: p-value above 1e-4 at a fixed seed.  A KS window (lo, hi)
    compares the draws inside it with the conditional CDF, and the fraction inside with its probability: outside the
    window fp32 cannot resolve the distribution (Gamma(0.05) below 1e-30, Beta(0.1, 0.1) within 1e-5 of 1)."""
    name, dist, window = case[0], case[4], case[5]
    x = x.cpu().double().numpy()
    if name.startswith('von_mises'):
        x = _wrap(x - 0.5)
    if name.startswith('binomial'):
        nt = int(case[3][0])
        counts = np.bincount(x.astype(np.int64), minlength=nt + 1)
        expect = dist.pmf(np.arange(nt + 1)) * x.size
        keep = np.nonzero(expect >= 5)[0]          # bins expected to hold 5 or more; the rest pooled
        f_obs, f_exp = counts[keep].astype(np.float64), expect[keep].copy()
        rest_o, rest_e = x.size - f_obs.sum(), x.size - f_exp.sum()
        if rest_e >= 5:
            f_obs, f_exp = np.append(f_obs, rest_o), np.append(f_exp, rest_e)
        else:
            j = int(np.argmin(f_exp))
            f_obs[j] += rest_o
            f_exp[j] += rest_e
        assert scipy.stats.chisquare(f_obs, f_exp).pvalue > 1e-4, name
        return
    if window is None:
        assert scipy.stats.kstest(x, dist.cdf).pvalue > 1e-4, name
        return
    lo, hi = window
    if name.startswith('beta'):
        lo, hi = case[3][2] + lo * (case[3][3] - case[3][2]), case[3][2] + hi * (case[3][3] - case[3][2])
    Flo, Fhi = dist.cdf(lo), dist.cdf(hi)
    inside = x[(x > lo) & (x < hi)]
    q = Fhi - Flo
    assert abs(inside.size - q * x.size) <= 5 * math.sqrt(x.size * q * (1 - q)) + 1, name
    assert scipy.stats.kstest(inside, lambda t: (dist.cdf(t) - Flo) / q).pvalue > 1e-4, name


@pytest.mark.parametrize('i', range(len(SAMPLERS)), ids=SAMPLER_IDS)
def test_sampler_distribution_support_and_fused_log_prob(cuda, i):
    case = SAMPLERS[i]
    name, draw, score, params, dist, _, support = case
    n = 100000
    x, lp = draw(*params, n, 20240 + i, 3, with_log_prob=True)
    assert support(x), name
    _distribution_test(case, x)
    # lp_out is the log_prob kernel's value at the drawn value, bit for bit
    want = score(x, *params)
    assert torch.isfinite(lp).all() or name.startswith('beta-0.1'), name
    assert torch.equal(torch.nan_to_num(lp), torch.nan_to_num(want)), (name, float((lp - want).abs().max()))


@pytest.mark.parametrize('i', range(len(SAMPLERS)), ids=SAMPLER_IDS)
def test_sampler_moments_and_sharding(cuda, i):
    name, draw, score, params, dist, _, _ = SAMPLERS[i]
    n = 1000000
    x = draw(*params, n, 777 + i, 11).double()
    if name.startswith('von_mises'):
        # circular moments: E cos(x - loc) = I1(k) / I0(k) = 1 - torch's circular variance, E sin(x - loc) = 0
        c, s = torch.cos(x - 0.5), torch.sin(x - 0.5)
        k = params[1]
        want = float(scipy.special.i1e(k) / scipy.special.i0e(k))
        assert abs(c.mean().item() - want) <= 5 * c.std().item() / math.sqrt(n), name
        assert abs(s.mean().item()) <= 5 * s.std().item() / math.sqrt(n), name
        assert abs((1 - want) - VonMises(0.5, k).variance) < 1e-4
    else:
        mean, var, kurt = (float(t) for t in dist.stats(moments='mvk'))
        assert abs(x.mean().item() - mean) <= 5 * math.sqrt(var / n), (name, x.mean().item(), mean)
        se_var = var * math.sqrt(kurt / n + 2 / (n - 1))       # exact sd of the sample variance (kurt: excess)
        assert abs(x.var().item() - var) <= 5 * se_var + 1e-12, (name, x.var().item(), var)
    # two first_index shards reproduce the unsharded draw bit for bit
    m = 30011
    full = draw(*params, m, 5, 9, first_index=100)
    a = draw(*params, m // 3, 5, 9, first_index=100)
    b = draw(*params, m - m // 3, 5, 9, first_index=100 + m // 3)
    assert torch.equal(torch.cat([a, b]), full), name


def test_per_particle_parameter_samplers(cuda):
    n = 300000
    nt = torch.tensor([5.0, 50.0, 500.0], device=cuda).repeat(n // 3)
    x, lp = ops.binomial_sample(nt, 0.3, n, 4, 2, with_log_prob=True)
    assert torch.equal(lp, ops.binomial_log_prob(x, nt, 0.3))
    for j, m in enumerate((5, 50, 500)):
        xs = x[j::3].double()
        assert ((xs >= 0) & (xs <= m)).all()
        assert abs(xs.mean().item() - 0.3 * m) <= 5 * math.sqrt(0.21 * m / xs.numel())
    c = torch.linspace(0.05, 20.0, n, device=cuda)
    g, lp = ops.gamma_sample(c, 1.0, n, 6, 2, with_log_prob=True)
    assert (g > 0).all() and torch.equal(lp, ops.gamma_log_prob(g, c, 1.0))
    z = (g.double() - c.double()) / c.double().sqrt()       # standardised: mean 0, variance 1
    assert abs(z.mean().item()) < 5 / math.sqrt(n) and abs(z.var().item() - 1) < 0.05


def test_invalid_parameters_draw_nan(cuda):
    assert torch.isnan(ops.gamma_sample(-1.0, 1.0, 8, 1, 1)).all()
    assert torch.isnan(ops.binomial_sample(2.5, 0.5, 8, 1, 1)).all()
    assert torch.isnan(ops.von_mises_sample(0.0, 0.0, 8, 1, 1)).all()
    assert torch.isnan(ops.beta_sample(0.0, 1.0, 0.0, 1.0, 8, 1, 1)).all()
    assert (ops.binomial_sample(7.0, 1.0, 8, 1, 1) == 7).all() and (ops.binomial_sample(7.0, 0.0, 8, 1, 1) == 0).all()


# ---- importance sampling --------------------------------------------------------------------------------------------------
def _posterior(model, observe, n=1 << 18, seed=3):
    pyprob.seed(seed)
    post = model.posterior_results(n, InferenceEngine.IMPORTANCE_SAMPLING, observe=observe)
    return float(post.mean), float(post.effective_sample_size)


def _check(mean, ess, want_mean, want_sd):
    assert abs(mean - want_mean) <= 5 * want_sd / math.sqrt(ess), (mean, want_mean, want_sd, ess)


def _quad_moments(density, lo, hi):
    z = scipy.integrate.quad(density, lo, hi, limit=200)[0]
    m = scipy.integrate.quad(lambda t: t * density(t), lo, hi, limit=200)[0] / z
    v = scipy.integrate.quad(lambda t: (t - m) ** 2 * density(t), lo, hi, limit=200)[0] / z
    return m, math.sqrt(v)


class BetaBinomial(Model):
    def forward(self):
        p = pyprob.sample(Beta(2.0, 3.0))
        pyprob.observe(Binomial(20, probs=p), name='k')
        return p


class GammaPoisson(Model):
    def forward(self):
        lam = pyprob.sample(Gamma(3.0, 2.0))
        for i in range(3):
            pyprob.observe(Poisson(lam), name='c{}'.format(i))
        return lam


class GammaExponential(Model):
    def forward(self):
        lam = pyprob.sample(Gamma(2.0, 1.0))
        pyprob.observe(Exponential(lam), name='t0')
        pyprob.observe(Exponential(lam), name='t1')
        return lam


class NormalLogNormal(Model):
    def forward(self):
        mu = pyprob.sample(Normal(0.0, 1.0))
        pyprob.observe(LogNormal(mu, 0.5), name='y0')
        pyprob.observe(LogNormal(mu, 0.5), name='y1')
        return mu


class BetaLowHigh(Model):
    def forward(self):
        theta = pyprob.sample(Beta(2.0, 2.0, low=-1.0, high=3.0))
        pyprob.observe(Normal(theta, 1.0), name='x')
        return theta


class WeibullScale(Model):
    def forward(self):
        lam = pyprob.sample(Uniform(0.5, 3.0))
        for i in range(3):
            pyprob.observe(Weibull(lam, 1.5), name='w{}'.format(i))
        return lam


class VonMisesLocation(Model):
    def forward(self):
        loc = pyprob.sample(Uniform(-math.pi, math.pi))
        pyprob.observe(VonMises(loc, 2.0), name='a0')
        pyprob.observe(VonMises(loc, 2.0), name='a1')
        return loc


def test_is_conjugate_posteriors(cuda):
    mean, ess = _posterior(BetaBinomial(), {'k': 14})                    # Beta(16, 9)
    _check(mean, ess, 16 / 25, math.sqrt(16 * 9 / (25 ** 2 * 26)))
    mean, ess = _posterior(GammaPoisson(), {'c0': 4, 'c1': 6, 'c2': 5})  # Gamma(18, 5)
    _check(mean, ess, 18 / 5, math.sqrt(18) / 5)
    mean, ess = _posterior(GammaExponential(), {'t0': 0.5, 't1': 1.2})  # Gamma(4, 2.7)
    _check(mean, ess, 4 / 2.7, 2 / 2.7)
    ly = math.log(2.0) + math.log(3.0)                                   # log y ~ Normal(mu, 0.5): precision 1 + 8
    mean, ess = _posterior(NormalLogNormal(), {'y0': 2.0, 'y1': 3.0})
    _check(mean, ess, 4 * ly / 9, 1 / 3)


def test_is_quadrature_posteriors(cuda):
    dens = (lambda t: scipy.stats.beta.pdf((t + 1) / 4, 2, 2) * scipy.stats.norm.pdf(1.5, t, 1))
    mean, ess = _posterior(BetaLowHigh(), {'x': 1.5})
    _check(mean, ess, *_quad_moments(dens, -1, 3))
    obs = (0.8, 1.7, 2.4)
    dens = (lambda t: np.prod([scipy.stats.weibull_min.pdf(w, 1.5, scale=t) for w in obs]))
    mean, ess = _posterior(WeibullScale(), {'w{}'.format(i): w for i, w in enumerate(obs)})
    _check(mean, ess, *_quad_moments(dens, 0.5, 3.0))
    dens = (lambda t: scipy.stats.vonmises.pdf(0.3, 2.0, loc=t) * scipy.stats.vonmises.pdf(0.9, 2.0, loc=t))
    mean, ess = _posterior(VonMisesLocation(), {'a0': 0.3, 'a1': 0.9})
    _check(mean, ess, *_quad_moments(dens, -math.pi, math.pi))


def test_is_log_weights_vs_oracle(cuda):
    """One seeded run, particle by particle: the log-weight of a prior proposal is the sum of the observe terms."""
    pyprob.seed(5)
    n = 50000
    tr = BetaBinomial()._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe={'k': 14})
    p = tr.result.cpu()
    want = fo.binomial_log_prob(torch.tensor(14.0), 20.0, p).double()
    np.testing.assert_allclose(tr.log_w.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)
    pyprob.seed(6)
    tr = WeibullScale()._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe={'w0': 0.8, 'w1': 1.7, 'w2': 2.4})
    lam = tr.result.cpu()
    want = sum(fo.weibull_log_prob(torch.tensor(w), lam, 1.5).double() for w in (0.8, 1.7, 2.4))
    np.testing.assert_allclose(tr.log_w.cpu().numpy(), want.numpy(), rtol=1e-5, atol=1e-5)


class RenewalCount(Model):
    """Exponential inter-arrival times drawn inside a while_loop: lanes leave the loop at different iterations."""

    def forward(self):
        rate = pyprob.sample(Gamma(2.0, 1.0), name='rate')

        def body(s):
            t = pyprob.sample(Exponential(rate))
            return {'t': s['t'] + t, 'k': s['k'] + 1}
        st = pyprob.while_loop(lambda s: s['t'] < 1.0, body, {'t': 0.0, 'k': 0.0})
        pyprob.observe(Normal(st['k'], 0.5), name='x')
        return rate


def test_is_while_loop_with_exponential(cuda):
    """k - 1 = arrivals of a rate-r Poisson process in [0, 1]: p(r | x) is proportional to
    Gamma(r; 2, 1) sum_j Poisson(j; r) Normal(x; j + 1, 0.5)."""
    pyprob.seed(8)
    n = 1 << 17
    tr = RenewalCount()._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe={'x': 4.0})
    k = None
    for s in tr.sites:
        if s.distribution is not None and s.distribution.name == 'Exponential':
            assert s.mask is not None
            k = s.mask.long() if k is None else k + s.mask.long()
    assert k is not None and 0 < float((k == k.max()).float().mean()) < 1       # lanes left at different iterations
    want = scipy.stats.norm.logpdf(4.0, k.cpu().double().numpy(), 0.5)
    np.testing.assert_allclose(tr.log_w.cpu().numpy(), want, rtol=1e-5, atol=1e-5)
    js = np.arange(60)
    dens = (lambda r: scipy.stats.gamma.pdf(r, 2.0) * np.sum(scipy.stats.poisson.pmf(js, r) *
                                                             scipy.stats.norm.pdf(4.0, js + 1, 0.5)))
    mean, ess = _posterior(RenewalCount(), {'x': 4.0}, n=n)
    _check(mean, ess, *_quad_moments(dens, 0.0, 40.0))


class TruncatedObserve(Model):
    def forward(self):
        mu = pyprob.sample(Normal(0.0, 1.0))
        pyprob.observe(TruncatedNormal(mu, 1.0, -1.0, 2.0), name='x')
        return mu


def test_is_observe_truncated_normal(cuda):
    from oracle import scoring
    pyprob.seed(9)
    n = 1 << 16
    tr = TruncatedObserve()._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe={'x': 0.5})
    mu = tr.result.cpu()
    want = scoring.truncated_normal_log_prob(torch.tensor(0.5), mu, torch.tensor(1.0), torch.tensor(-1.0),
                                             torch.tensor(2.0))
    np.testing.assert_allclose(tr.log_w.cpu().numpy(), want.double().numpy(), rtol=1e-4, atol=1e-4)

    def dens(t):
        z = scipy.stats.norm.cdf(2.0 - t) - scipy.stats.norm.cdf(-1.0 - t)
        return scipy.stats.norm.pdf(t) * scipy.stats.norm.pdf(0.5, t, 1) / z
    mean, ess = _posterior(TruncatedObserve(), {'x': 0.5}, n=n)
    _check(mean, ess, *_quad_moments(dens, -8, 8))


# ---- inference compilation ------------------------------------------------------------------------------------------------
class ICFamilies(Model):
    """A controlled Normal latent, an uncontrolled Gamma site and Binomial / LogNormal observations.  With `extra` it also
    has a controlled Gamma site and an uncontrolled Weibull site after everything else, which the network never saw."""

    def __init__(self, extra=False):
        super().__init__('IC families')
        self.extra = extra

    def forward(self):
        z = pyprob.sample(Normal(0.0, 1.0), name='z')
        g = pyprob.sample(Gamma(2.0, 4.0), name='g', control=False)
        pyprob.observe(Binomial(20, probs=torch.sigmoid(z)), name='k')
        pyprob.observe(LogNormal(z, 0.3 + g), name='y')
        if self.extra:
            pyprob.sample(Gamma(2.0, 1.0), name='h')
            pyprob.sample(Weibull(1.0, 2.0), name='u', control=False)
        return z


class ControlledGamma(Model):
    def forward(self):
        a = pyprob.sample(Gamma(2.0, 1.0))
        pyprob.observe(Normal(a, 1.0), name='x')
        return a


OBS = {'k': 13.0, 'y': 1.8}


@pytest.mark.parametrize('network', [InferenceNetwork.LSTM, InferenceNetwork.FEEDFORWARD])
def test_ic_log_weights_vs_oracle(cuda, network):
    from unittest import mock
    from oracle import network as onet
    from tests import ff_oracle
    from tests.ic_replay import site_weight_terms
    pyprob.seed(21)
    pyprob.set_verbosity(0)
    model = ICFamilies()
    model.learn_inference_network(num_traces=4 * 256, batch_size=256, inference_network=network, lstm_dim=32,
                                  observe_embeddings={'k': {'dim': 8}, 'y': {'dim': 8}})
    net = model._inference_network
    n = 4000
    with torch.no_grad():
        pyprob.seed(22)
        trace = model._run_batched(n, trace_mode=TraceMode.POSTERIOR,
                                   inference_engine=InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                   inference_network=net, observe=OBS)
    assert [s.name for s in trace.variables_controlled] == ['z']
    patch = ff_oracle.infer_sequence if network == InferenceNetwork.FEEDFORWARD else onet.infer_sequence
    with mock.patch.object(onet, 'infer_sequence', patch):
        want, covered = site_weight_terms(trace, net, torch.tensor([OBS['k'], OBS['y']]))
    assert covered.all()
    z = trace.result.cpu()
    g = trace.named_variables['g'].value.cpu()
    assert (g > 0).all()
    want = want + fo.binomial_log_prob(torch.tensor(OBS['k']), 20.0, torch.sigmoid(z)).double().numpy()
    want = want + fo.lognormal_log_prob(torch.tensor(OBS['y']), z, 0.3 + g).double().numpy()
    np.testing.assert_allclose(trace.log_w.cpu().numpy(), want, rtol=1e-4, atol=2e-4)

    # a controlled site of a new family is unknown to the network: the prior proposes there and its weight term is 0, so
    # with the new sites last the log-weights equal those of the run without them; an uncontrolled one is drawn from its
    # prior as always
    model.extra = True
    with torch.no_grad(), warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter('always')
        pyprob.seed(22)
        trace2 = model._run_batched(n, trace_mode=TraceMode.POSTERIOR,
                                    inference_engine=InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                    inference_network=net, observe=OBS)
    assert any('Address unknown' in str(w.message) for w in caught)
    assert (trace2.named_variables['h'].value > 0).all() and (trace2.named_variables['u'].value > 0).all()
    assert torch.equal(trace2.log_w, trace.log_w)


@pytest.mark.parametrize('network', [InferenceNetwork.LSTM, InferenceNetwork.FEEDFORWARD])
def test_ic_controlled_new_family_is_unsupported(cuda, network):
    pyprob.set_verbosity(0)
    with pytest.raises(RuntimeError, match='Distribution currently unsupported: Gamma'):
        ControlledGamma().learn_inference_network(num_traces=256, batch_size=128, inference_network=network,
                                                  lstm_dim=32, observe_embeddings={'x': {'dim': 8}})
