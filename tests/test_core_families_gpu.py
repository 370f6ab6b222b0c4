"""GPU: the samplers and log_prob kernels of Normal, Uniform, Poisson, Categorical, the Normal mixture and the truncated-
Normal mixture against plain fp64 references (scipy, numpy float64 applied to the same fp32 inputs the kernels see), and the
importance-weight reduction combined from partials as ranks combine them.

Conventions (as tests/test_families_gpu.py): fixed seeds; KS or chi-square p-values above 1e-4, chi-square bins expected to
hold fewer than 5 draws pooled; moments within 5 standard errors; two first_index shards of m = 30011 split at m // 3
reproduce the unsharded draw bit for bit.

Error bounds are counted in eps = 2^-23 (one ulp of 1): a correctly rounded fp32 operation is off by at most eps/2 of its
result, libm logf / expf by 1 / 2 ulp, lgammaf by 6 ulp (CUDA C Programming Guide, mathematical functions), and the MUFU
approximations the scoring kernels use (rcp / ex2 / lg2.approx) by about 2 ulp, lg2 by 2^-22 absolute."""
import math

import numpy as np
import pytest
import scipy.special
import scipy.stats
import torch

from pyprob_b200 import _lib, ops

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -23
EPS32 = float(np.finfo(np.float32).eps)          # clamp_probs bound, = EPS
LOG_SQRT_2PI = 0.5 * math.log(2 * math.pi)
P_MIN = 1e-4
SHARD_M = 30011


def f32(x):
    """the fp64 value of the fp32 number a kernel sees for x"""
    return np.asarray(x, np.float32).astype(np.float64)


def host(t):
    return t.detach().cpu().double().numpy()


# ---- statistics helpers ---------------------------------------------------------------------------------------------------
def chi2(counts, probs, n, name):
    """chi-square of observed counts against cell probabilities over n draws.  The probabilities may sum to less than 1:
    the remainder is one more cell, observed = the draws outside the listed cells.  Cells expected to hold fewer than 5
    draws are pooled into the remainder, or into the smallest cell when the remainder expects fewer than 5 too."""
    counts, probs = np.asarray(counts, np.float64), np.asarray(probs, np.float64)
    expect = probs * n
    keep = expect >= 5
    f_obs, f_exp = counts[keep], expect[keep]
    rest_o, rest_e = n - f_obs.sum(), max(n - f_exp.sum(), 0.0)
    if rest_e >= 5:
        f_obs, f_exp = np.append(f_obs, rest_o), np.append(f_exp, rest_e)
    elif f_obs.size:
        j = int(np.argmin(f_exp))
        f_obs[j] += rest_o
        f_exp[j] += rest_e
    if f_obs.size < 2:                 # one cell holds (nearly) everything: nothing to test beyond the support checks
        assert rest_o <= max(5 * rest_e, 0) + 5, (name, rest_o, rest_e)
        return
    f_exp *= f_obs.sum() / f_exp.sum()          # remove the last-bit mismatch chisquare refuses
    p = scipy.stats.chisquare(f_obs, f_exp).pvalue
    assert p > P_MIN, (name, p)


def chi2_draws(x, n_total, pmf_cells, name):
    """chi-square of integer draws x against pmf_cells = (k0, probabilities of k0, k0 + 1, ...)"""
    k0, probs = pmf_cells
    k = x.astype(np.int64) - k0
    inside = (k >= 0) & (k < probs.size)
    counts = np.bincount(k[inside], minlength=probs.size)
    chi2(counts, probs, n_total, name)


def ks(x, cdf, name):
    p = scipy.stats.kstest(x, cdf).pvalue
    assert p > P_MIN, (name, p)


def lattice_chi2(x, cdf, name):
    """Draws that fp32 rounding puts on a lattice coarse against the distribution's scale (Normal(-1e3, 1e-3): spacing
    6.1e-5 = 0.06 sd) defeat KS against the continuous CDF.  Each observed float takes the mass of its round-to-nearest
    cell, [midpoint to the float below, midpoint to the float above), under the fp64 CDF; the rest of the mass is one cell."""
    v, counts = np.unique(x.astype(np.float32), return_counts=True)
    below = np.nextafter(v, np.float32(-np.inf)).astype(np.float64)
    above = np.nextafter(v, np.float32(np.inf)).astype(np.float64)
    v = v.astype(np.float64)
    probs = cdf((v + above) / 2) - cdf((v + below) / 2)
    chi2(counts, probs, x.size, name)


def moments(x, mean, var, kurt, name):
    """sample mean and variance within 5 standard errors; kurt is the excess kurtosis"""
    n = x.size
    assert abs(x.mean() - mean) <= 5 * math.sqrt(var / n) + 1e-12 * abs(mean), (name, x.mean(), mean)
    se_var = var * math.sqrt(max(kurt, -2.0) / n + 2 / (n - 1))
    assert abs(x.var(ddof=1) - var) <= 5 * se_var, (name, x.var(ddof=1), var)


def sharded(draw, name):
    """draw(m, first_index) -> tensor"""
    full = draw(SHARD_M, 100)
    a = draw(SHARD_M // 3, 100)
    b = draw(SHARD_M - SHARD_M // 3, 100 + SHARD_M // 3)
    assert torch.equal(torch.cat([a, b]), full), name


# ---- Normal ---------------------------------------------------------------------------------------------------------------
# Box-Muller from a 24-bit uniform cannot go beyond sqrt(-2 log 2^-24) = 5.77 sd (probability 8e-9 per draw): far below
# what a test at these sizes can see, so it is not tested.
@pytest.mark.parametrize('mu,sd', [(0.0, 1.0), (2.0, 3.0), (-1e3, 1e-3), (0.0, 1e4)])
def test_normal_sampler(cuda, mu, sd):
    name = 'Normal({}, {})'.format(mu, sd)
    n = 1000000
    x, lp = ops.normal_sample(mu, sd, n, 1101, 3, with_log_prob=True)
    m, s = float(f32(mu)), float(f32(sd))
    xs = host(x)
    assert np.isfinite(xs).all() and torch.isfinite(lp).all(), name
    cdf = scipy.stats.norm(m, s).cdf
    if np.spacing(np.float32(abs(m) + 6 * s)) > 1e-4 * s:
        lattice_chi2(xs, cdf, name)
    else:
        ks(xs, cdf, name)
    moments(xs, m, s * s, 0.0, name)
    # lp_out and the scorer evaluate the same expression
    assert torch.equal(lp, ops.normal_log_prob(x, mu, sd)), name
    sharded(lambda k, f: ops.normal_sample(mu, sd, k, 5, 9, first_index=f), name)


def test_normal_sampler_per_particle(cuda):
    pars = [(0.0, 1.0), (-1e3, 1e-3), (5.0, 20.0)]
    n = 3 * 100000
    mu = torch.tensor([p[0] for p in pars], device=cuda).repeat(n // 3)
    sd = torch.tensor([p[1] for p in pars], device=cuda).repeat(n // 3)
    x, lp = ops.normal_sample(mu, sd, n, 1102, 4, with_log_prob=True)
    assert torch.equal(lp, ops.normal_log_prob(x, mu, sd))
    xs = host(x)
    for j, (m, s) in enumerate(pars):
        m, s = float(f32(m)), float(f32(s))
        name = 'Normal({}, {}) class {}'.format(m, s, j)
        c = xs[j::3]
        cdf = scipy.stats.norm(m, s).cdf
        (lattice_chi2 if np.spacing(np.float32(abs(m) + 6 * s)) > 1e-4 * s else ks)(c, cdf, name)
        moments(c, m, s * s, 0.0, name)


# ---- Uniform --------------------------------------------------------------------------------------------------------------
UNIFORM = [(-1.0, 3.0), (1000.0, 1001.0), (0.0, 1e-6), (-5.0, -4.99)]


@pytest.mark.parametrize('lo,hi', UNIFORM)
def test_uniform_sampler(cuda, lo, hi):
    """Every draw in [low, high) and scored finite: fp32 lo + u (hi - lo) rounds onto hi for u near 1 when the spacing at
    hi is coarse against hi - lo (Uniform(1000, 1001): every u above 1 - 3.05e-5, about 30 draws per million)."""
    name = 'Uniform({}, {})'.format(lo, hi)
    n = 1000000
    x, lp = ops.uniform_sample(lo, hi, n, 1201, 3, with_log_prob=True)
    a, b = float(f32(lo)), float(f32(hi))
    xs = host(x)
    assert (xs >= a).all() and (xs < b).all(), (name, int((xs >= b).sum()), int((xs < a).sum()))
    assert torch.isfinite(lp).all(), (name, int((~torch.isfinite(lp)).sum()))
    # lp_out and the scorer evaluate the same expression: (lo <= v < hi ? 0 : -inf) - logf(hi - lo)
    assert torch.equal(lp, ops.uniform_log_prob(x, lo, hi)), name
    ks(xs, scipy.stats.uniform(a, b - a).cdf, name)
    moments(xs, (a + b) / 2, (b - a) ** 2 / 12, -1.2, name)
    sharded(lambda k, f: ops.uniform_sample(lo, hi, k, 5, 9, first_index=f), name)


def test_uniform_sampler_per_particle(cuda):
    pars = UNIFORM[:3]
    n = 3 * 200000
    lo = torch.tensor([p[0] for p in pars], device=cuda).repeat(n // 3)
    hi = torch.tensor([p[1] for p in pars], device=cuda).repeat(n // 3)
    x, lp = ops.uniform_sample(lo, hi, n, 1202, 4, with_log_prob=True)
    assert torch.equal(lp, ops.uniform_log_prob(x, lo, hi)) and torch.isfinite(lp).all()
    xs = host(x)
    for j, (a, b) in enumerate(pars):
        a, b = float(f32(a)), float(f32(b))
        c = xs[j::3]
        name = 'Uniform({}, {}) class {}'.format(a, b, j)
        assert (c >= a).all() and (c < b).all(), name
        ks(c, scipy.stats.uniform(a, b - a).cdf, name)
        moments(c, (a + b) / 2, (b - a) ** 2 / 12, -1.2, name)


# ---- Poisson --------------------------------------------------------------------------------------------------------------
POISSON_RATES = [0.0, 1e-3, 0.7, 4.0, 9.99, 10.0, 10.01, 37.0, 1e3, 1e5, 1e6]


def poisson_cells(rate):
    """(k0, pmf of k0 .. k1) covering all but about 1e-12 of the mass"""
    d = scipy.stats.poisson(rate)
    k0, k1 = int(d.ppf(1e-12)), int(d.ppf(1 - 1e-12)) + 1
    return k0, d.pmf(np.arange(k0, k1 + 1))


def check_poisson_draws(x, rate, name):
    assert (x == np.floor(x)).all() and (x >= 0).all(), name
    if rate == 0:
        assert (x == 0).all(), name
        return
    chi2_draws(x, x.size, poisson_cells(rate), name)
    moments(x, rate, rate, 1.0 / rate, name)


@pytest.mark.parametrize('rate', POISSON_RATES)
def test_poisson_sampler(cuda, rate):
    """Rates 9.99 / 10 / 10.01 straddle the switch from inversion to PTRS; 1e5 and 1e6 are where an fp32 acceptance test
    (terms near rate log rate, spacing 0.125 at 1e6) visibly skews the distribution."""
    name = 'Poisson({})'.format(rate)
    n = 1000000
    x, lp = ops.poisson_sample(rate, n, 1301, 3, with_log_prob=True)
    r = float(f32(rate))
    xs = host(x)
    check_poisson_draws(xs, r, name)
    assert torch.isfinite(lp).all(), name
    assert torch.equal(lp, ops.poisson_log_prob(x, rate)), name
    sharded(lambda k, f: ops.poisson_sample(rate, k, 5, 9, first_index=f), name)


def test_poisson_sampler_per_particle(cuda):
    rates = [4.0, 37.0, 1e5]
    n = 3 * 200000
    rt = torch.tensor(rates, device=cuda).repeat(n // 3)
    x, lp = ops.poisson_sample(rt, n, 1302, 4, with_log_prob=True)
    xs = host(x)
    assert torch.equal(lp, ops.poisson_log_prob(x, rt))
    for j, r in enumerate(rates):
        c = xs[j::3]
        check_poisson_draws(c, r, 'Poisson({}) class {}'.format(r, j))


# ---- Categorical ----------------------------------------------------------------------------------------------------------
def categorical_probs(C, kind):
    """'spread': unnormalised (sum 7.3) with zero-probability categories first, in the middle and last (C >= 4; the first
    only for C = 2, 3); 'peaked': one category at 1 - 1e-6, the rest sharing 1e-6"""
    if kind == 'spread':
        p = 1.0 + (np.arange(C) * 7) % 5
        zeros = [0, C // 2, C - 1] if C >= 4 else ([0] if C >= 2 else [])
        p[zeros] = 0.0
        return (p * (7.3 / p.sum())).astype(np.float32)
    p = np.full(C, 1e-6 / (C - 1))
    p[C // 3] = 1 - 1e-6
    return p.astype(np.float32)


CAT_CASES = [(C, kind, layout) for C in (1, 2, 3, 7, 16, 33) for kind in ('spread', 'peaked')
             for layout in ('shared', 'rows', 'block') if not (C == 1 and kind == 'peaked')]


def categorical_layout(P, n, layout, cuda):
    """P: [2, C] parameter sets -> (probs argument, set index per particle).  'shared': set 0 as a [C] tensor; 'rows': a
    contiguous [n, C] tensor, particle i holding set i % 2; 'block': the same rows as a column block of a wider tensor"""
    C = P.shape[1]
    if layout == 'shared':
        return torch.from_numpy(P[0]).to(cuda), np.zeros(n, np.int64)
    which = np.arange(n) % 2
    rows = torch.from_numpy(P[which]).to(cuda)
    if layout == 'rows':
        return rows, which
    wide = torch.full((n, C + 5), 3.0, device=cuda)
    wide[:, 2:2 + C] = rows
    return wide[:, 2:2 + C], which


@pytest.mark.parametrize('C,kind,layout', CAT_CASES)
def test_categorical_sampler(cuda, C, kind, layout):
    name = 'C={} {} {}'.format(C, kind, layout)
    n = 200000
    p0 = categorical_probs(C, kind)
    P = np.stack([p0, p0[::-1].copy()])
    probs, which = categorical_layout(P, n, layout, cuda)
    x, lp = ops.categorical_sample(probs, n, 1401 + C, 3, with_log_prob=True)
    xs = host(x)
    assert ((xs == np.floor(xs)) & (xs >= 0) & (xs < C)).all(), name
    # lp_out and the scorer both compute logf(clamp(p[v] / sum p)) with the sum in category order
    assert torch.equal(lp, ops.categorical_log_prob(x, probs)), name
    for s in np.unique(which):
        c = xs[which == s].astype(np.int64)
        w = P[s].astype(np.float64) / P[s].astype(np.float64).sum()
        assert (w[c] > 0).all(), (name, 'zero-probability category drawn')
        chi2(np.bincount(c, minlength=C), w, c.size, name)
        k = np.arange(C)
        mean = (w * k).sum()
        var = (w * (k - mean) ** 2).sum()
        if kind == 'spread' and var > 0:        # 'peaked' draws its rare categories ~0.1 times: no normal limit
            moments(c.astype(np.float64), mean, var, (w * (k - mean) ** 4).sum() / var ** 2 - 3, name)
    sharded(lambda m, f: ops.categorical_sample(probs if layout == 'shared' else probs[f - 100:f - 100 + m], m, 5, 9,
                                                first_index=f), name)


# ---- mixtures: fp64 reference and error bound -----------------------------------------------------------------------------
def mixture_lp64(v, m, s, p, lo=None, hi=None):
    """fp64 log_prob of the reference's Mixture (weights clamp(p / sum p)) of Normal or TruncatedNormal components at the
    fp32 inputs (v [n], m / s / p [n, K], lo / hi [n]), with an error bound for an fp32 evaluation.

    To first order the fp32 logsumexp is off by the responsibility-weighted mean of the errors of its terms
    t_j = log w_j + log N(v; mu_j, sigma_j) (r_j = exp(t_j - lp)), plus its own roundings.  A term carries the quadratic
    z^2 / 2 within about 7 eps (z from a division or an rcp and a product, squared, scaled), log w_j within (K + 3) eps
    (the fp32 sum of K weights, the division, the clamp) and log sigma_j within 2 eps; the exponentials (expf 2 ulp /
    ex2.approx), the fp32 sum of K terms (K eps), the final log and the additions of max and constant add
    (K + 6) eps + 3 eps |lp|.  Bound: 8 eps (sum_j r_j S_j + |lp|) + (2K + 10) eps, S_j = z_j^2 / 2 + |log sigma_j|
    + |log w_j| + 1.  A truncated component's mass Z_j = Phi(beta) - Phi(alpha) is a difference of two fp32 CDFs, each
    within about 4 x 6e-8 absolute (erff's 2 ulp, the rounding of its argument and of 1 + erf): sum_j r_j 8 x 6e-8 / Z_j
    more."""
    v = v[:, None]
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        w = np.clip(p / p.sum(-1, keepdims=True), EPS32, 1 - EPS32)
        z = (v - m) / s
        t = np.log(w) - 0.5 * z * z - np.log(s) - LOG_SQRT_2PI
        extra = 0.0
        if lo is not None:
            lo, hi = lo[:, None], hi[:, None]
            Z = scipy.special.ndtr((hi - m) / s) - scipy.special.ndtr((lo - m) / s)
            t = t - np.log(Z)
            t = np.where((v >= lo) & (v <= hi), t, -np.inf)
            extra = 8 * 6e-8 / Z
        lp = scipy.special.logsumexp(t, axis=1)
        r = np.exp(t - lp[:, None])
        r = np.where(np.isfinite(r), r, 0.0)
        S = 0.5 * z * z + np.abs(np.log(s)) + np.abs(np.log(w)) + 1
        bound = 8 * EPS * ((r * S).sum(1) + np.abs(lp)) + (2 * m.shape[1] + 10) * EPS + (r * extra).sum(1)
    return lp, bound


def expand_rows(x, n):
    x = host(x) if torch.is_tensor(x) else np.asarray(x, np.float64)
    return np.broadcast_to(x, (n, x.shape[-1])) if x.ndim == 1 else x


def expand_param(x, n):
    x = host(x) if torch.is_tensor(x) else f32(x)
    return np.broadcast_to(x.reshape(-1), (n,)) if x.size == 1 else x.reshape(-1)


def same_classes(got, want, name):
    for f in (np.isnan, np.isposinf, np.isneginf):
        assert np.array_equal(f(got), f(want)), (name, f.__name__, np.nonzero(f(got) != f(want))[0][:10])


def within(got, want, bound, name):
    same_classes(got, want, name)
    fin = np.isfinite(want)
    err = np.abs(got[fin] - want[fin])
    assert (err <= bound[fin]).all(), (name, float((err - bound[fin]).max()), np.nonzero(err > bound[fin])[0][:10])


def mixture_layout(sets, n, layout, cuda):
    """sets: list of (means [K], stddevs [K], probs [K]) -> (means, stddevs, probs arguments, set index per particle).
    'shared': set 0 as [K] tensors; 'blocks': per-particle rows taken as the three column blocks of one [n, 3K] tensor
    (the layout of the proposal head's output), particle i holding set i % len(sets)"""
    if layout == 'shared':
        return [torch.tensor(a, dtype=torch.float32, device=cuda) for a in sets[0]] + [np.zeros(n, np.int64)]
    K = len(sets[0][0])
    which = np.arange(n) % len(sets)
    T = torch.from_numpy(np.stack([np.concatenate(st) for st in sets])[which].astype(np.float32)).to(cuda)
    return [T[:, :K], T[:, K:2 * K], T[:, 2 * K:], which]


def mixture_moments(m, s, w):
    """mean, variance, excess kurtosis of a Normal mixture"""
    mean = (w * m).sum()
    d = m - mean
    var = (w * (s * s + d * d)).sum()
    m4 = (w * (d ** 4 + 6 * d * d * s * s + 3 * s ** 4)).sum()
    return mean, var, m4 / var ** 2 - 3


def normal_mixture_sets(K):
    a = (np.linspace(-6, 6, K) + 0.3, 0.3 + 0.4 * (np.arange(K) % 4), 1.0 + (np.arange(K) * 5) % 7)
    b = (-0.5 * a[0][::-1] + 2, 1.5 * a[1], a[2][::-1].copy())
    if K >= 3:
        a[2][K // 2] = 0.0
    for st in (a, b):
        st[2][:] *= 7.3 / st[2].sum()
    return [tuple(f32(x) for x in st) for st in (a, b)]


@pytest.mark.parametrize('layout', ['shared', 'blocks'])
@pytest.mark.parametrize('K', [1, 3, 10, 32])
def test_mixture_normal_sampler(cuda, K, layout):
    name = 'K={} {}'.format(K, layout)
    n = 400000
    sets = normal_mixture_sets(K)
    means, stddevs, probs, which = mixture_layout(sets, n, layout, cuda)
    x, lp = ops.mixture_normal_sample(means, stddevs, probs, n, 1501 + K, 3, with_log_prob=True)
    xs = host(x)
    assert np.isfinite(xs).all(), name
    for j in np.unique(which):
        m, s, p = sets[j]
        w = p / p.sum()
        c = xs[which == j]
        ks(c, lambda t: (w * scipy.special.ndtr((t[:, None] - m) / s)).sum(1), name)
        moments(c, *mixture_moments(m, s, w), name=name)
    # both lp_out and the scorer within the fp64 bound of the exact value: within twice the bound of each other
    want = host(ops.mixture_normal_log_prob(x, means, stddevs, probs))
    _, bound = mixture_lp64(xs, expand_rows(means, n), expand_rows(stddevs, n), expand_rows(probs, n))
    within(host(lp), want, 2 * bound, name)
    if layout == 'shared':
        sharded(lambda k, f: ops.mixture_normal_sample(means, stddevs, probs, k, 5, 9, first_index=f), name)
    else:
        sharded(lambda k, f: ops.mixture_normal_sample(means[f - 100:f - 100 + k], stddevs[f - 100:f - 100 + k],
                                                       probs[f - 100:f - 100 + k], k, 5, 9, first_index=f), name)


def trunc_sets(K, window):
    """list of (means, stddevs, probs, low, high) parameter sets; every component keeps at least 1e-3 of its mass inside
    the window, so that fp32 resolves it"""
    k = np.arange(K)
    p = 1.0 + (k * 5) % 7
    if window == 'central':
        return [(np.linspace(-1, 1.5, K), 0.5 + 1.5 * k / max(K - 1, 1), p, -1.5, 2.0)]
    if window == 'tail':          # N(0, 1) on [2.5, 40]: mass 6.2e-3; the widest alpha (2.5 / 0.9) leaves 2.7e-3
        return [(np.linspace(0, 0.5, K), np.linspace(0.9, 1.1, K), p, 2.5, 40.0)]
    if window == 'poisson':       # the Poisson proposal window, means spread over [-2, 45]: mass >= 0.16
        return [(np.linspace(-2, 45, K), np.linspace(2, 5, K), p, 0.0, 40.0)]
    # per-particle low / high, as proposals for Uniform priors: three windows, the last where fp32 is coarse near high
    return [(np.linspace(-0.5, 2.5, K), np.full(K, 1.0), p, -1.0, 3.0),
            (np.linspace(-2, 45, K), np.linspace(2, 5, K), p[::-1].copy(), 0.0, 40.0),
            (1000.8 + np.linspace(-0.3, 0.1, K), np.full(K, 0.5), p, 1000.0, 1001.0)]


def trunc_mixture_cdf(m, s, w, lo, hi):
    comps = [scipy.stats.truncnorm((lo - mk) / sk, (hi - mk) / sk, loc=mk, scale=sk) for mk, sk in zip(m, s)]
    return lambda t: sum(wk * c.cdf(t) for wk, c in zip(w, comps))


def trunc_mixture_moments(m, s, w, lo, hi):
    """mean, variance, excess kurtosis; raw moments taken about the window's centre c, so that they do not cancel at
    [1000, 1001]"""
    c = (lo + hi) / 2
    raw = np.zeros(5)
    for mk, sk, wk in zip(m, s, w):
        d = scipy.stats.truncnorm((lo - mk) / sk, (hi - mk) / sk, loc=mk - c, scale=sk)
        raw += wk * np.array([1.0] + [d.moment(j) for j in range(1, 5)])
    mean = raw[1]
    var = raw[2] - mean ** 2
    m4 = raw[4] - 4 * mean * raw[3] + 6 * mean ** 2 * raw[2] - 3 * mean ** 4
    return mean + c, var, m4 / var ** 2 - 3


@pytest.mark.parametrize('window', ['central', 'tail', 'poisson', 'per-particle'])
@pytest.mark.parametrize('K', [1, 3, 10])
def test_mixture_truncated_normal_sampler(cuda, K, window):
    name = 'K={} {}'.format(K, window)
    n = 300000
    raw = trunc_sets(K, window)
    sets = [tuple(f32(x) for x in st[:3]) for st in raw]
    bounds = [(float(f32(st[3])), float(f32(st[4]))) for st in raw]
    means, stddevs, probs, which = mixture_layout(sets, n, 'shared' if len(sets) == 1 else 'blocks', cuda)
    if len(sets) == 1:
        low, high = bounds[0]
    else:
        low = torch.tensor([b[0] for b in bounds], device=cuda)[torch.from_numpy(which).to(cuda)]
        high = torch.tensor([b[1] for b in bounds], device=cuda)[torch.from_numpy(which).to(cuda)]
    x, lp = ops.mixture_truncated_normal_sample(means, stddevs, probs, low, high, n, 1601 + K, 3, with_log_prob=True)
    xs = host(x)
    for j in np.unique(which):
        (m, s, p), (a, b) = sets[j], bounds[j]
        c = xs[which == j]
        assert ((c >= a) & (c < b)).all(), (name, j, c.min(), c.max())
        w = p / p.sum()
        ks(c, trunc_mixture_cdf(m, s, w, a, b), name)
        moments(c, *trunc_mixture_moments(m, s, w, a, b), name=name)
    want = host(ops.mixture_truncated_normal_log_prob(x, means, stddevs, probs, low, high))
    _, bound = mixture_lp64(xs, expand_rows(means, n), expand_rows(stddevs, n), expand_rows(probs, n),
                            expand_param(low, n), expand_param(high, n))
    assert np.isfinite(want).all(), name
    within(host(lp), want, 2 * bound, name)
    if len(sets) == 1:
        sharded(lambda k, f: ops.mixture_truncated_normal_sample(means, stddevs, probs, low, high, k, 5, 9,
                                                                 first_index=f), name)
    else:
        def draw(k, f):
            sl = slice(f - 100, f - 100 + k)
            return ops.mixture_truncated_normal_sample(means[sl], stddevs[sl], probs[sl], low[sl], high[sl], k, 5, 9,
                                                       first_index=f)
        sharded(draw, name)


@pytest.mark.parametrize('mean,low,high', [(0.0, 6.0, 7.0), (-20.0, 0.0, 40.0)])
def test_mixture_truncated_normal_sampler_deep_tail(cuda, mean, low, high):
    """Windows whose mass fp32 CDF differences cannot resolve (N(0, 1) on [6, 7]: 1e-9; mean -20 on [0, 40]: 3e-89).
    Phi(alpha) and Phi(beta) both round to 1, the inverse-CDF argument is clamped to 1 - 6e-8 (5.3 sd) and the clamp into
    the window then puts every draw on low: the draws are valid values of the support, not draws from the distribution.
    Only that is asserted."""
    x = ops.mixture_truncated_normal_sample(torch.tensor([mean, mean + 0.5], device=cuda),
                                            torch.tensor([1.0, 1.0], device=cuda), torch.tensor([0.5, 0.5], device=cuda),
                                            low, high, 100000, 1701, 3)
    assert torch.isfinite(x).all() and (x >= low).all() and (x < high).all()


# ---- mixture scoring against fp64 -------------------------------------------------------------------------------------------
# every launch_mixture instantiation: KMAX 4 (K = 1, 2, 4), KMAX 10 with a runtime K (5, 9), K == 10 exact, KMAX 32 (11..32)
MIX_K = [1, 2, 4, 5, 9, 10, 11, 31, 32]


def mixture_score_case(K, trunc, layout, n, gen):
    """value, means, stddevs, probs ([n, K] or [K]), low, high ([n]) with unnormalised weights, a zero weight, and (rows /
    blocks) special rows: values outside [low, high], components far apart where the one with the largest exponent has
    zero weight, a negative sigma."""
    k = np.arange(K)
    v = gen.standard_normal(n) * 2
    if layout == 'shared':
        m = np.broadcast_to(np.linspace(-1.5, 1.5, K), (n, K)).copy()
        s = np.broadcast_to(0.4 + 1.6 * ((k * 3) % 5) / 4, (n, K)).copy()
        p = np.broadcast_to(1.0 + (k * 5) % 7, (n, K)).copy()
        lo, hi = np.full(n, -2.0), np.full(n, 2.0)
    else:
        m = v[:, None] + 0.75 * (2 * gen.random((n, K)) - 1)
        s = 0.4 + 1.6 * gen.random((n, K))
        p = 7.3 * gen.random((n, K)) / K
        lo, hi = v - 0.5 - gen.random(n), v + 0.5 + gen.random(n)
    if K >= 2:
        p[:, K // 2] = 0.0
    if layout != 'shared':
        v[1], v[2] = lo[1] - 0.25, hi[2] + 0.25          # outside the window (truncated: -inf)
        v[3], v[4] = lo[3], hi[4]                        # on its edges (inside)
        s[5, K - 1] = -1.0                               # negative sigma: NaN
        if not trunc and K >= 2:                         # far apart; the nearest component has weight 0
            for i in range(6, 12):
                m[i] = v[i] + 30.0 * (k + 1) * (i - 5)
                m[i, 0] = v[i]
                p[i, 0] = 0.0
                p[i, 1:] = 1.0
                s[i] = 1.0
    m, s, p = f32(m), f32(s), f32(p)
    return f32(v), m, s, p, f32(lo), f32(hi)


def mixture_args(m, s, p, layout, cuda):
    n, K = m.shape
    if layout == 'shared':
        return [torch.tensor(a[0], dtype=torch.float32, device=cuda) for a in (m, s, p)]
    if layout == 'rows':
        return [torch.tensor(a, dtype=torch.float32, device=cuda) for a in (m, s, p)]
    T = torch.tensor(np.concatenate([m, s, p], 1), dtype=torch.float32, device=cuda)
    return [T[:, :K], T[:, K:2 * K], T[:, 2 * K:]]


@pytest.mark.parametrize('layout', ['shared', 'rows', 'blocks'])
@pytest.mark.parametrize('trunc', [False, True], ids=['normal', 'truncated'])
@pytest.mark.parametrize('K', MIX_K)
def test_mixture_log_prob_vs_fp64(cuda, K, trunc, layout):
    name = 'K={} {} {}'.format(K, 'truncated' if trunc else 'normal', layout)
    n = 2053
    gen = np.random.default_rng(1000 * K + 10 * trunc + len(layout))
    v, m, s, p, lo, hi = mixture_score_case(K, trunc, layout, n, gen)
    args = mixture_args(m, s, p, layout, cuda)
    vt = torch.tensor(v, dtype=torch.float32, device=cuda)
    if trunc:
        low, high = ((-2.0, 2.0) if layout == 'shared' else
                     (torch.tensor(lo, dtype=torch.float32, device=cuda), torch.tensor(hi, dtype=torch.float32, device=cuda)))
        fn = lambda **kw: ops.mixture_truncated_normal_log_prob(vt, *args, low, high, **kw)   # noqa: E731
        want, bound = mixture_lp64(v, m, s, p, lo, hi)
        with np.errstate(invalid='ignore'):
            Z = scipy.special.ndtr((hi[:, None] - m) / s) - scipy.special.ndtr((lo[:, None] - m) / s)
        assert (Z[s > 0] >= 0.05).all()                  # the windows keep mass >= 0.05 in every component
    else:
        fn = lambda **kw: ops.mixture_normal_log_prob(vt, *args, **kw)                         # noqa: E731
        want, bound = mixture_lp64(v, m, s, p)
    with np.errstate(invalid='ignore'):
        want = np.where((s < 0).any(1), np.nan, want)    # log of a negative sigma poisons the row
    got = fn()
    within(host(got), want, bound, name)
    if layout != 'shared':
        assert np.isnan(host(got)[5])
        if trunc:
            assert np.isneginf(host(got)[1:3]).all() and np.isfinite(host(got)[3:5]).all()
    # acc form: fp64 running sum of the fp32 terms, with either sign
    acc = torch.full((n,), 0.25, dtype=torch.float64, device=cuda)
    fn(acc=acc, acc_scale=1.0)
    assert torch.equal(acc.nan_to_num(), (0.25 + got.double()).nan_to_num()), name
    fn(acc=acc, acc_scale=-1.0)
    assert torch.equal(acc.nan_to_num(), (0.25 + got.double() - got.double()).nan_to_num()), name


@pytest.mark.parametrize('trunc', [False, True], ids=['normal', 'truncated'])
def test_mixture_log_prob_k33_not_supported(cuda, trunc):
    n, K = 64, 33
    m, s, p = (torch.full((K,), c, device=cuda) for c in (0.0, 1.0, 1.0))
    v = torch.zeros(n, device=cuda)
    lp = torch.full((n,), 7.0, device=cuda)
    torch.cuda.synchronize()
    before = _lib.call('ppb_launch_count')
    with pytest.raises(RuntimeError, match='K=33 > 32 not supported'):
        if trunc:
            ops.mixture_truncated_normal_log_prob(v, m, s, p, -1.0, 1.0, lp_out=lp)
        else:
            ops.mixture_normal_log_prob(v, m, s, p, lp_out=lp)
    assert _lib.call('ppb_launch_count') == before
    assert (lp == 7.0).all()


# ---- Categorical scoring ----------------------------------------------------------------------------------------------------
def test_categorical_log_prob_paths_vs_fp64(cuda):
    """The vectorised path (C % 4 == 0, 16-byte aligned rows) and the scalar path agree bit for bit: both sum the row in
    category order.  Against fp64: the sum of C terms is within (C - 1) eps / 2 relative, the division and clamp eps / 2,
    logf 1 ulp: |diff| <= (C + 2) eps + eps |lp|."""
    n = 5003
    gen = np.random.default_rng(3)
    for C in (16, 7):
        p = f32(gen.random((n, C)) * 7.3 / C)
        p[:, C // 2] = 0.0
        p[::7, 0] = 1e-9                                   # below clamp_probs' eps after normalising
        v = f32(gen.integers(0, C, n))
        vt = torch.tensor(v, dtype=torch.float32, device=cuda)
        aligned = torch.tensor(p, dtype=torch.float32, device=cuda)
        buf = torch.empty(n * C + 1, device=cuda)
        offset = buf[1:].view(n, C)                       # every row one float off 16-byte alignment: scalar path
        offset.copy_(aligned)
        got = ops.categorical_log_prob(vt, aligned)
        assert torch.equal(got, ops.categorical_log_prob(vt, offset)), C
        shared = ops.categorical_log_prob(vt, aligned[0])
        w = np.clip(p / p.sum(1, keepdims=True), EPS32, 1 - EPS32)
        want = np.log(w[np.arange(n), v.astype(np.int64)])
        within(host(got), want, (C + 2) * EPS + EPS * np.abs(want), 'C={}'.format(C))
        want0 = np.log(w[0][v.astype(np.int64)])
        within(host(shared), want0, (C + 2) * EPS + EPS * np.abs(want0), 'C={} shared'.format(C))
        bad = torch.tensor([-1.0, float(C)], device=cuda)
        assert torch.isnan(ops.categorical_log_prob(bad, aligned[:2])).all()
        assert torch.isnan(ops.categorical_log_prob(bad, offset[:2])).all()


# ---- Poisson scoring --------------------------------------------------------------------------------------------------------
def test_poisson_log_prob_vs_fp64(cuda):
    """k = 62..65 cross from the log-factorial table to lgammaf.  fp64 reference xlogy(k, rate) - rate - lgamma(k + 1) at
    the fp32 rate; the fp32 formula cancels, so the bound is relative to its terms: the kernel's k lg2(rate) ln2 is within
    k 2^-22 ln2 + 2 eps |k log rate|, log k! within eps / 2 (table) or 6 ulp (lgammaf), and two subtractions add eps each
    of the partial sums: 8 eps T + 2^-22 k, T = |k log rate| + rate + lgamma(k + 1)."""
    ks_ = np.array([0, 1, 62, 63, 64, 65, 1000], np.float64)
    rates = np.array([1e-3, 0.5, 37.0, 1e5])
    kk, rr = [a.reshape(-1) for a in np.meshgrid(ks_, f32(rates))]
    kk, rr = np.tile(kk, 3), np.tile(rr, 3)                  # 84 values: both paths see full float4 groups and a tail
    want = scipy.special.xlogy(kk, rr) - rr - scipy.special.gammaln(kk + 1)
    bound = 8 * EPS * (np.abs(scipy.special.xlogy(kk, rr)) + rr + scipy.special.gammaln(kk + 1)) + 2.0 ** -22 * kk
    v = torch.tensor(kk, dtype=torch.float32, device=cuda)
    r = torch.tensor(rr, dtype=torch.float32, device=cuda)
    within(host(ops.poisson_log_prob(v, r)), want, bound, 'aligned')
    within(host(ops.poisson_log_prob(v[1:], r[1:])), want[1:], bound[1:], 'unaligned')
    for rate in f32(rates):
        sel = rr == rate
        within(host(ops.poisson_log_prob(v[torch.from_numpy(sel).to(cuda)], float(rate))), want[sel], bound[sel],
               'shared {}'.format(rate))
    # rate 1: lg2(1) = 0, so lp = -1 - log k!.  The table side (k < 64) is the correctly rounded log k! and one more
    # rounding: within 1 ulp of lp; lgammaf (k >= 64) within 6 ulp of log k! and one rounding
    k = np.arange(0, 200, dtype=np.float64)
    want = -1.0 - scipy.special.gammaln(k + 1)
    got = host(ops.poisson_log_prob(torch.tensor(k, dtype=torch.float32, device=cuda), 1.0))
    ulp = np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
    err = np.abs(got - want)
    assert (err[:64] <= ulp[:64]).all(), np.nonzero(err[:64] > ulp[:64])[0]
    assert (err[64:] <= 7 * ulp[64:]).all(), np.nonzero(err[64:] > 7 * ulp[64:])[0]


# ---- Uniform scoring --------------------------------------------------------------------------------------------------------
def test_uniform_log_prob_edges(cuda):
    """low scores -log(high - low) (hi - lo is exact in fp32 for these pairs, logf within 1 ulp), high scores -inf, at the
    vectorised (aligned), scalar (unaligned) and shared-parameter paths."""
    for lo, hi in UNIFORM:
        a, b = np.float32(lo), np.float32(hi)
        vals = np.array([a, b, (a + b) / 2, np.nextafter(a, np.float32(-np.inf)), np.nextafter(b, a), b, a, a],
                        np.float32)
        inside = np.array([1, 0, 1, 0, 1, 0, 1, 1], bool)
        ref = -math.log(float(b) - float(a))
        want = np.where(inside, ref, -np.inf)
        tol = np.full(want.size, float(np.spacing(np.float32(abs(ref)))))
        v = torch.tensor(np.tile(vals, 2), device=cuda)
        lo_t = torch.full((v.numel(),), float(a), device=cuda)
        hi_t = torch.full((v.numel(),), float(b), device=cuda)
        w2, t2 = np.tile(want, 2), np.tile(tol, 2)
        name = 'Uniform({}, {})'.format(lo, hi)
        within(host(ops.uniform_log_prob(v, lo_t, hi_t)), w2, t2, name + ' aligned')
        within(host(ops.uniform_log_prob(v[1:], lo_t[1:], hi_t[1:])), w2[1:], t2[1:], name + ' unaligned')
        within(host(ops.uniform_log_prob(v, float(a), float(b))), w2, t2, name + ' shared')


# ---- importance weights -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dead_half', ['first', 'second'])
def test_weights_finalize_from_two_ranks_partials(cuda, dead_half):
    """ppb_weights_finalize over the partials of two disjoint halves, concatenated as parallel.gather_weight_partials
    concatenates ranks', one half all -inf.  n = 3,000,001 is past the 4 x SM partial cap, so the partials kernel runs its
    grid-stride loop.  The result equals the single pass and the fp64 oracle up to the rounding of fp64 sums in a different
    order."""
    n = 3000001
    h = n // 2
    gen = torch.Generator().manual_seed(11)
    lw = (torch.randn(n, generator=gen) * 5 - 40).float()
    if dead_half == 'first':
        lw[:h] = -math.inf
    else:
        lw[h:] = -math.inf
    assert h > 4 * 132 * 256 * 8             # more 2048-element tiles than partials in each half
    d = lw.to(cuda)
    part = torch.cat([ops.weights_partials(d[:h]), ops.weights_partials(d[h:])])
    stats2, logits2 = ops.weights_finalize(d, partials=part)
    stats1, logits1 = ops.weights_finalize(d)
    x = lw.double().numpy()
    lse = scipy.special.logsumexp(x)
    p = np.exp(x - lse)
    ess = 1.0 / (p * p).sum()
    for stats, logits in ((stats1, logits1), (stats2, logits2)):
        st = host(stats)
        np.testing.assert_allclose(st[0], lse, rtol=1e-13)
        np.testing.assert_allclose(st[1], ess, rtol=1e-10)
        got = host(logits)
        fin = np.isfinite(x)
        assert np.isneginf(got[~fin]).all()
        np.testing.assert_allclose(got[fin], x[fin] - lse, rtol=1e-13, atol=1e-12)
    np.testing.assert_allclose(host(stats2), host(stats1), rtol=1e-13)
