"""Event-shaped observations: the event log_prob kernel against the per-particle kernels and an fp64 sum, the event
samplers (element 0, sharding, distributions, counter independence, lp_out), and the engines end to end (IS, LMH / RMH,
IC training and posterior) on models that observe a vector in one statement."""
import math

import numpy as np
import pytest
import scipy.stats
import torch

import pyprob_b200 as pyprob
from pyprob_b200 import InferenceEngine, InferenceNetwork, Model, ops
from pyprob_b200.distributions import (Bernoulli, Beta, Binomial, Categorical, Exponential, Gamma, LogNormal, Normal,
                                       Poisson, TruncatedNormal, Uniform, VonMises, Weibull)
from pyprob_b200.util import TraceMode

pytestmark = pytest.mark.gpu

FAMILIES = list(ops.EVENT_FAMILIES)
SCALAR = {'Normal': ops.normal_log_prob, 'Uniform': ops.uniform_log_prob, 'Poisson': ops.poisson_log_prob,
          'Bernoulli': ops.bernoulli_log_prob, 'Exponential': ops.exponential_log_prob, 'Gamma': ops.gamma_log_prob,
          'LogNormal': ops.lognormal_log_prob, 'Weibull': ops.weibull_log_prob, 'Beta': ops.beta_log_prob,
          'Binomial': ops.binomial_log_prob, 'VonMises': ops.von_mises_log_prob}
SAMPLE = {'Normal': ops.normal_sample, 'Uniform': ops.uniform_sample, 'Poisson': ops.poisson_sample,
          'Bernoulli': ops.bernoulli_sample, 'Exponential': ops.exponential_sample, 'Gamma': ops.gamma_sample,
          'LogNormal': ops.lognormal_sample, 'Weibull': ops.weibull_sample, 'Beta': ops.beta_sample,
          'Binomial': ops.binomial_sample, 'VonMises': ops.von_mises_sample}


def _case(family, shape, g):
    """(value, [parameters]) of `shape`, inside the support (Uniform also outside), as CUDA fp32 tensors."""
    def u(lo=0.0, hi=1.0):
        return lo + (hi - lo) * torch.rand(shape, generator=g, device='cuda')
    if family == 'Normal':
        return torch.randn(shape, generator=g, device='cuda'), [u(-1, 1), u(0.5, 2)]
    if family == 'Uniform':
        lo = u(-2, -1)
        hi = lo + u(1, 2)
        return lo + (hi - lo) * u(-0.1, 1.1), [lo, hi]
    if family == 'Poisson':
        rate = u(0.1, 70)
        return torch.poisson(rate, generator=g), [rate]
    if family == 'Bernoulli':
        return (u() < 0.5).float(), [u()]
    if family == 'Exponential':
        return u(0, 3), [u(0.5, 2)]
    if family == 'Gamma':
        return u(0.01, 3), [u(0.5, 4), u(0.5, 2)]
    if family == 'LogNormal':
        return u(0.01, 3), [u(-0.5, 0.5), u(0.5, 1.5)]
    if family == 'Weibull':
        return u(0.01, 3), [u(0.5, 2), u(0.5, 3)]
    if family == 'Beta':
        return u(-1, 2), [u(0.5, 3), u(0.5, 3), torch.full(shape, -1.0, device='cuda'),
                          torch.full(shape, 2.0, device='cuda')]
    if family == 'Binomial':
        N = torch.floor(u(1, 30))
        return torch.floor(u() * (N + 1)).clamp(max=N), [N, u()]
    return u(-4, 4), [u(-3, 3), u(0.1, 6)]


LAYOUTS = ['scalar', 'particle', 'shared', 'event']


def _operand(full, layout):
    """The layout's operand from a full [n, D] tensor, and the [n, D] tensor it stands for."""
    n, D = full.shape
    if layout == 'scalar':
        x = full[0, 0].reshape(1)
        return x, x.reshape(1, 1).expand(n, D)
    if layout == 'particle':
        x = full[:, :1].contiguous()
        return x, x.expand(n, D)
    if layout == 'shared':
        x = full[:1].contiguous()
        return x, x.expand(n, D)
    return full, full


def _offset(full):
    """The same values in a view whose rows start 4 bytes off a 16-byte boundary."""
    buf = torch.empty(full.numel() + 1, device='cuda')
    v = buf[1:].view(full.shape)
    v.copy_(full)
    return v


def _check_layouts(family, n, D, seed, offset=False):
    g = torch.Generator(device='cuda').manual_seed(seed)
    fid = ops.EVENT_FAMILIES[family]
    value, params = _case(family, (n, D), g)
    # values: shared event (0, 1), event per particle (D, 1), scalar (0, 0), one per particle (1, 0)
    combos = [(vl, L) for vl in ('shared', 'event', 'scalar', 'particle') for L in LAYOUTS] + [('event', 'mixed')]
    for vl, pl in combos:
        layouts = [LAYOUTS[(k + 1) % 4] for k in range(len(params))] if pl == 'mixed' else [pl] * len(params)
        if family == 'Beta':
            layouts[2:] = ['scalar', 'scalar'] if pl != 'mixed' else ['shared', 'particle']
        v_op, v_full = _operand(value, {'shared': 'shared', 'event': 'event', 'scalar': 'scalar',
                                        'particle': 'particle'}[vl])
        ops_full = [_operand(p, L) for p, L in zip(params, layouts)]
        p_ops = [o for o, _ in ops_full]
        if offset:
            v_op = _offset(v_op) if v_op.dim() == 2 and v_op.size(0) == n and n > 1 else v_op
            p_ops = [_offset(o) if o.dim() == 2 and o.size(1) == D and o.size(0) == n and n > 1 else o for o in p_ops]
        # element-wise: the per-particle kernel over the flattened operands, bit for bit
        want = SCALAR[family](v_full.reshape(-1).contiguous(), *[f.reshape(-1).contiguous() for _, f in ops_full])
        lp = ops.event_log_prob(fid, v_op, p_ops, n, D)
        assert torch.equal(lp.view(-1).isnan(), want.isnan()), (family, vl, layouts)
        ok = ~want.isnan()
        assert torch.equal(lp.view(-1)[ok], want[ok]), (family, vl, layouts)
        # the accumulator: acc0 + 0.75 * (fp64 row sum), to summation-order rounding
        acc0 = torch.randn(n, dtype=torch.float64, generator=g, device='cuda')
        acc = acc0.clone()
        lp2 = torch.full((n, D), float('nan'), device='cuda')
        ops.event_log_prob(fid, v_op, p_ops, n, D, lp_out=lp2, acc=acc, acc_scale=0.75)   # both outputs in one call
        assert torch.equal(lp2.view(-1)[ok], want[ok])
        rows = want.view(n, D).double()
        exp = acc0 + 0.75 * rows.sum(1)
        bound = 1e-13 * (rows.abs().sum(1) + acc0.abs()) + 1e-300
        fin = torch.isfinite(exp)
        assert ((acc - exp).abs()[fin] <= bound[fin]).all(), (family, vl, layouts)
        assert torch.equal(acc[~fin].isnan(), exp[~fin].isnan())
        # repeated calls: the same bits
        acc2 = acc0.clone()
        ops.event_log_prob(fid, v_op, p_ops, n, D, acc=acc2, acc_scale=0.75)
        assert torch.equal(acc.view(torch.int64), acc2.view(torch.int64))


@pytest.mark.parametrize('family', FAMILIES)
@pytest.mark.parametrize('n,D', [(1, d) for d in (1, 2, 3, 31, 32, 33, 784, 4097)] +
                         [(3, d) for d in (1, 2, 3, 31, 32, 33, 784, 4097)] +
                         [(1000, d) for d in (1, 2, 3, 31, 32, 33, 784, 4097)] +
                         [(65537, d) for d in (1, 3, 33)])
def test_event_log_prob_every_layout(cuda, family, n, D):
    _check_layouts(family, n, D, seed=sum(map(ord, family)) + 7 * n + D)


@pytest.mark.parametrize('family', ['Normal', 'Poisson', 'Gamma', 'Beta'])
@pytest.mark.parametrize('n,D', [(65537, 784), (1000, 4097), (1000, 33)])
def test_event_log_prob_large_and_unaligned(cuda, family, n, D):
    _check_layouts(family, n, D, seed=7, offset=True)


def test_event_log_prob_vs_fp64_normal(cuda):
    """The Normal element term against its fp64 formula (the per-particle kernels have their own fp64 tests)."""
    n, D = 3000, 37
    g = torch.Generator(device='cuda').manual_seed(1)
    v, (mu, sd) = _case('Normal', (n, D), g)
    acc = torch.zeros(n, dtype=torch.float64, device='cuda')
    ops.event_log_prob(0, v[:1], [mu, sd[:, :1].contiguous()], n, D, acc=acc)
    vd, mud, sdd = v[:1].double(), mu.double(), sd[:, :1].double()
    want = (-(vd - mud) ** 2 / (2 * sdd ** 2) - sdd.log() - 0.5 * math.log(2 * math.pi)).sum(1)
    np.testing.assert_allclose(acc.cpu().numpy(), want.cpu().numpy(), rtol=2e-6, atol=2e-5)


@pytest.mark.parametrize('family', FAMILIES)
def test_d1_equals_scalar_accumulator(cuda, family):
    n = 10007
    g = torch.Generator(device='cuda').manual_seed(3)
    v, params = _case(family, (n, 1), g)
    a1 = torch.randn(n, dtype=torch.float64, generator=g, device='cuda')
    a2 = a1.clone()
    SCALAR[family](v.reshape(-1), *[p.reshape(-1) for p in params], acc=a1, acc_scale=1.3)
    ops.event_log_prob(ops.EVENT_FAMILIES[family], v, [p.reshape(n, 1) for p in params], n, 1, acc=a2, acc_scale=1.3)
    assert torch.equal(a1.view(torch.int64), a2.view(torch.int64))

    # every D = 1 layout is a flat stride: (1, 1) is (1, 0), and a shared (0, 1) or (0, 0) operand is (1, 0) over its
    # expanded copy, for the value and every parameter, accumulator and lp_out bit for bit
    def run(operands):
        acc, lp = a1.clone(), torch.empty(n, device='cuda')
        slots = [a for t, ps, es in operands[1:] for a in (ops.ptr(t), ps, es)] + [None, 0, 0] * (5 - len(operands))
        t, ps, es = operands[0]
        ops._lib.call('ppb_event_log_prob', ops.EVENT_FAMILIES[family], ops.ptr(t), ps, es, *slots, n, 1, ops.ptr(lp),
                      ops.ptr(acc), 1.3, ops.stream())
        return acc.view(torch.int64), lp
    flat = [t.reshape(n).contiguous() for t in [v] + params]
    want = run([(t, 1, 0) for t in flat])
    got = run([(t, 1, 1) for t in flat])
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    for k in range(len(flat)):
        shared = [t[:1].clone() if j == k else t for j, t in enumerate(flat)]
        want = run([(t.expand(n).contiguous(), 1, 0) for t in shared])
        for es in (0, 1):
            got = run([(t, 0, es) if j == k else (t, 1, 0) for j, t in enumerate(shared)])
            assert torch.equal(got[0], want[0]) and torch.equal(got[1].isnan(), want[1].isnan()), (family, k, es)
            ok = ~want[1].isnan()
            assert torch.equal(got[1][ok], want[1][ok]), (family, k, es)


def test_beyond_2_31_elements(cuda):
    """n D = 2^32 with a shared value row and scalar parameters: nothing large is allocated."""
    n, D = 1 << 22, 1 << 10
    row = torch.full((1, D), 0.3, device='cuda')
    acc = torch.zeros(n, dtype=torch.float64, device='cuda')
    ops.event_log_prob(0, row, [0.1, 1.7], n, D, acc=acc)
    one = ops.normal_log_prob(torch.full((1,), 0.3, device='cuda'), 0.1, 1.7).double()
    assert torch.equal(acc, (D * one).expand(n))


def test_errors_before_launch(cuda):
    row = torch.zeros(1, 4, device='cuda')
    with pytest.raises(RuntimeError, match='D > 0'):
        ops._lib.call('ppb_event_log_prob', 0, ops.ptr(row), 0, 1, ops.ptr(row), 0, 0, ops.ptr(row), 0, 0, None, 0, 0,
                      None, 0, 0, 4, 0, None, None, 1.0, ops.stream())
    with pytest.raises(RuntimeError, match='strides'):
        ops._lib.call('ppb_event_log_prob', 0, ops.ptr(row), 2, 1, ops.ptr(row), 0, 0, ops.ptr(row), 0, 0, None, 0, 0,
                      None, 0, 0, 4, 4, None, None, 1.0, ops.stream())
    with pytest.raises(RuntimeError, match='null'):
        ops._lib.call('ppb_event_log_prob', 0, ops.ptr(row), 0, 1, None, 0, 0, ops.ptr(row), 0, 0, None, 0, 0,
                      None, 0, 0, 4, 4, None, None, 1.0, ops.stream())
    with pytest.raises(RuntimeError, match='unknown family'):
        ops._lib.call('ppb_event_log_prob', 11, ops.ptr(row), 0, 1, ops.ptr(row), 0, 0, ops.ptr(row), 0, 0, None, 0, 0,
                      None, 0, 0, 4, 4, None, None, 1.0, ops.stream())
    with pytest.raises(RuntimeError, match='2\\^40'):
        ops._lib.call('ppb_event_sample', 0, ops.ptr(row), 0, 0, ops.ptr(row), 0, 0, None, 0, 0, None, 0, 0,
                      ops.ptr(row), None, 4, 1, 1, 0, (1 << 40) - 2, ops.stream())


# ---- samplers ---------------------------------------------------------------------------------------------------------------
SAMPLER_PARAMS = {'Normal': [[-1.0, 0.0, 2.0, 5.0], [0.5, 1.0, 2.0, 0.1]], 'Uniform': [[-1.0, 0.0, 2.0, 1000.0],
                                                                                       [1.0, 0.5, 5.0, 1001.0]],
                  'Poisson': [[0.5, 3.0, 12.0, 80.0]], 'Bernoulli': [[0.1, 0.5, 0.9, 0.3]],
                  'Exponential': [[0.5, 1.0, 2.0, 7.0]], 'Gamma': [[0.3, 1.0, 2.5, 9.0], [1.0, 2.0, 0.5, 3.0]],
                  'LogNormal': [[0.0, -1.0, 1.0, 0.5], [0.5, 1.0, 0.2, 1.5]],
                  'Weibull': [[1.0, 2.0, 0.5, 3.0], [0.7, 1.5, 3.0, 1.0]],
                  'Beta': [[0.5, 2.0, 5.0, 1.0], [0.5, 3.0, 1.0, 1.0], [0.0, -1.0, 0.0, 2.0], [1.0, 1.0, 1.0, 5.0]],
                  'Binomial': [[1.0, 10.0, 40.0, 100.0], [0.3, 0.5, 0.9, 0.2]],
                  'VonMises': [[0.0, 1.0, -2.0, 3.0], [0.5, 2.0, 8.0, 40.0]]}


def _scipy(family, p):
    if family == 'Normal':
        return scipy.stats.norm(p[0], p[1])
    if family == 'Uniform':
        return scipy.stats.uniform(p[0], p[1] - p[0])
    if family == 'Poisson':
        return scipy.stats.poisson(p[0])
    if family == 'Bernoulli':
        return scipy.stats.bernoulli(p[0])
    if family == 'Exponential':
        return scipy.stats.expon(scale=1 / p[0])
    if family == 'Gamma':
        return scipy.stats.gamma(p[0], scale=1 / p[1])
    if family == 'LogNormal':
        return scipy.stats.lognorm(p[1], scale=math.exp(p[0]))
    if family == 'Weibull':
        return scipy.stats.weibull_min(p[1], scale=p[0])
    if family == 'Beta':
        return scipy.stats.beta(p[0], p[1], loc=p[2], scale=p[3] - p[2])
    if family == 'Binomial':
        return scipy.stats.binom(int(p[0]), p[1])
    return scipy.stats.vonmises(p[1], loc=p[0])


DISCRETE = {'Poisson', 'Bernoulli', 'Binomial'}


@pytest.mark.parametrize('family', FAMILIES)
def test_event_sampler(cuda, family):
    fid = ops.EVENT_FAMILIES[family]
    P = SAMPLER_PARAMS[family]
    D = len(P[0])
    shared = [torch.tensor([row], device='cuda') for row in P]
    n = 40000
    v, lp = ops.event_sample(fid, shared, n, D, 11, 5, 0, with_log_prob=True)
    # element 0 is the per-particle draw bit for bit
    assert torch.equal(v[:, 0], SAMPLE[family](*[row[0] for row in P], n, 11, 5))
    # per-particle parameters: element 0 again, and a shard draws the rows of the full run
    g = torch.Generator(device='cuda').manual_seed(2)
    per = [t.expand(n, D) * (1 + 0.01 * torch.rand(n, 1, generator=g, device='cuda')) for t in shared]
    if family == 'Binomial':
        per[0] = shared[0].expand(n, D).contiguous()
    if family == 'Beta':
        per[2:] = [shared[2].expand(n, D).contiguous(), shared[3].expand(n, D).contiguous()]
    vp = ops.event_sample(fid, [p[:, :1].contiguous() for p in per], n, D, 12, 6, 0)
    assert torch.equal(vp[:, 0], SAMPLE[family](*[p[:, 0].contiguous() for p in per], n, 12, 6))
    full = ops.event_sample(fid, per, n, D, 13, 7, 0)
    a, b = 12345, 23456
    shard = ops.event_sample(fid, [p[a:b] for p in per], b - a, D, 13, 7, a)
    assert torch.equal(full[a:b], shard)
    # lp_out: the scoring kernel's row sums of the drawn rows
    acc = torch.zeros(n, dtype=torch.float64, device='cuda')
    ops.event_log_prob(fid, v, shared, n, D, acc=acc)
    assert torch.equal(lp, acc.float())
    # each element against scipy, with its own parameters
    x = v.cpu().double().numpy()
    for j in range(D):
        dist = _scipy(family, [row[j] for row in P])
        if family in DISCRETE:
            ks = np.arange(0, int(x[:, j].max()) + 1)
            pmf = dist.pmf(ks)
            keep = pmf * n >= 5
            obs = np.array([(x[:, j] == k).sum() for k in ks])
            o = np.append(obs[keep], obs[~keep].sum())
            e = np.append(pmf[keep], 1 - pmf[keep].sum()) * n
            if e[-1] < 5:
                o, e = o[:-1], e[:-1] * (n / e[:-1].sum())
                o = o * (n / o.sum())
            p = scipy.stats.chisquare(o, e).pvalue if len(o) > 1 else 1.0
        else:
            xj = x[:, j]
            if family == 'VonMises':    # draws lie in [-pi, pi); scipy's support is [loc - pi, loc + pi)
                loc = P[0][j]
                xj = np.mod(xj - loc + math.pi, 2 * math.pi) - math.pi + loc
            p = scipy.stats.kstest(xj, dist.cdf).pvalue
        assert p > 1e-5, (family, j, p)
    # neighbouring elements are independent across particles: no reused counters
    for j in range(D - 1):
        c = np.corrcoef(x[:, j], x[:, j + 1])[0, 1]
        if np.isfinite(c):
            assert abs(c) < 5 / math.sqrt(n), (family, j, c)
    # the same parameter at every element: rows of identical parameters are still independent
    same = ops.event_sample(fid, [row[0] for row in P], n, 8, 14, 8, 0).cpu().double().numpy()
    for j in range(7):
        c = np.corrcoef(same[:, j], same[:, j + 1])[0, 1]
        if np.isfinite(c):
            assert abs(c) < 5 / math.sqrt(n), (family, j, c)


def test_sampler_limits(cuda):
    with pytest.raises(ValueError, match='2\\^24'):
        ops.event_sample(0, [0.0, 1.0], 2, (1 << 24) + 1, 1, 1)
    with pytest.raises(ValueError, match='2\\^40'):
        ops.event_sample(0, [0.0, 1.0], 4, 2, 1, 1, first_index=(1 << 40) - 2)


# ---- engines ------------------------------------------------------------------------------------------------------------
D50 = 50
OBS50 = torch.linspace(-1, 3, D50)


class IIDVector(Model):
    def forward(self):
        mu = pyprob.sample(Normal(0.0, 2.0), name='mu')
        pyprob.observe(Normal(mu, 1.5), name='y')
        return mu


class IIDScalars(Model):
    def forward(self):
        mu = pyprob.sample(Normal(0.0, 2.0), name='mu')
        for j in range(D50):
            pyprob.observe(Normal(mu, 1.5), name='y{}'.format(j))
        return mu


def _normal_posterior(obs, prior_sd=2.0, sd=1.5):
    prec = 1 / prior_sd ** 2 + len(obs) / sd ** 2
    return float(obs.sum()) / sd ** 2 / prec, math.sqrt(1 / prec)


def test_is_vector_observe_equals_scalar_observes(cuda):
    n = 65536
    pyprob.seed(4)
    t1 = IIDVector()._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe={'y': OBS50})
    pyprob.seed(4)
    t2 = IIDScalars()._run_batched(n, trace_mode=TraceMode.POSTERIOR,
                                   observe={'y{}'.format(j): float(OBS50[j]) for j in range(D50)})
    assert torch.equal(t1.result, t2.result)
    np.testing.assert_allclose(t1.log_w.cpu().numpy(), t2.log_w.cpu().numpy(), rtol=1e-12, atol=0)
    y = t1.named_variables['y'].value
    assert y.shape == (n, D50) and y.stride(0) == 0
    m, s = _normal_posterior(OBS50)
    post = IIDVector().posterior_results(1 << 18, InferenceEngine.IMPORTANCE_SAMPLING, observe={'y': OBS50})
    assert abs(float(post.mean) - m) < 5 * s / math.sqrt(float(post.effective_sample_size))


class Regression(Model):
    def __init__(self, x):
        super().__init__()
        self.x = x

    def forward(self):
        w = pyprob.sample(Normal(0.0, 1.0), name='w')
        b = pyprob.sample(Normal(0.0, 1.0), name='b')
        loc = w.view(-1, 1) * self.x.view(1, -1) + b.view(-1, 1)       # [n, D]: one event per particle
        pyprob.observe(Normal(loc, 0.5), name='y')
        return torch.stack([w, b], 1)


def test_is_bayesian_linear_regression(cuda):
    D = 200
    x = torch.linspace(-1, 1, D, device='cuda')
    g = torch.Generator().manual_seed(0)
    y = (0.7 * x.cpu() - 0.2 + 0.5 * torch.randn(D, generator=g))
    X = np.stack([x.cpu().numpy(), np.ones(D)], 1).astype(np.float64)
    cov = np.linalg.inv(np.eye(2) + X.T @ X / 0.25)
    mean = cov @ (X.T @ y.double().numpy() / 0.25)
    pyprob.seed(9)
    n = 1 << 21
    tr = Regression(x)._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe={'y': y})
    lw = tr.log_w
    w = torch.exp(lw - lw.max())
    w = w / w.sum()
    ess = float(1 / (w ** 2).sum())
    th = tr.result.double()
    m = (w.view(-1, 1) * th).sum(0)
    c = (w.view(-1, 1, 1) * (th - m).unsqueeze(2) * (th - m).unsqueeze(1)).sum(0)
    sd = np.sqrt(np.diag(cov))
    assert ess > 100
    assert np.all(np.abs(m.cpu().numpy() - mean) < 5 * sd / math.sqrt(ess)), (m, mean, ess)
    np.testing.assert_allclose(c.cpu().numpy(), cov, rtol=0.3, atol=0.3 * sd.max() ** 2)


@pytest.mark.parametrize('engine', [InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS,
                                    InferenceEngine.RANDOM_WALK_METROPOLIS_HASTINGS])
def test_mh_vector_observe(cuda, engine):
    obs = OBS50[:10]

    class M(Model):
        def forward(self):
            mu = pyprob.sample(Normal(0.0, 2.0), name='mu')
            pyprob.observe(Normal(mu, 1.5), name='y')
            return mu
    pyprob.seed(5)
    C, S, burn = 4096, 300, 150
    post = M().posterior_results(S, engine, observe={'y': obs}, num_chains=C)
    vals = np.array([float(post[i]) for i in range(burn * C, S * C, 10 * C + 1)])
    m, s = _normal_posterior(obs)
    assert scipy.stats.kstest(vals, scipy.stats.norm(m, s).cdf).pvalue > 1e-4


class Net8(Model):
    def forward(self):
        z = pyprob.sample(Normal(0.0, 1.0), name='z')
        u = pyprob.sample(Uniform(0.0, 2.0), name='u')
        pyprob.observe(Normal(z.view(-1, 1) * torch.linspace(0, 1, 8, device='cuda') + u.view(-1, 1), 0.3),
                       name='x')
        return z


def test_training_trace_draws_event_and_encodes_columns(cuda):
    pyprob.seed(3)
    tr = Net8()._run_batched(512, trace_mode=TraceMode.PRIOR_FOR_INFERENCE_NETWORK)
    x = tr.named_variables['x'].value
    assert x.shape == (512, 8)
    z, u = tr.named_variables['z'].value, tr.named_variables['u'].value
    resid = (x - z.view(-1, 1) * torch.linspace(0, 1, 8, device='cuda') - u.view(-1, 1)) / 0.3
    assert abs(float(resid.mean())) < 0.05 and abs(float(resid.std()) - 1) < 0.05


@pytest.mark.parametrize('network', [InferenceNetwork.LSTM, InferenceNetwork.FEEDFORWARD])
def test_ic_training_and_posterior(cuda, network):
    from unittest import mock
    from oracle import network as onet
    from pyprob_b200.dataset import OnlineDataset
    from tests import ff_oracle
    from tests.ic_replay import site_weight_terms
    pyprob.seed(21)
    pyprob.set_verbosity(0)
    model = Net8()
    model.learn_inference_network(num_traces=4 * 256, batch_size=256, inference_network=network, lstm_dim=32,
                                  observe_embeddings={'x': {'dim': 16}})
    net = model._inference_network
    assert net._observe_in_dims == [8]
    # loss and every gradient on a fresh batch against the oracle, through TraceBatch.encode's D columns
    batch = OnlineDataset(model).next_batch(256)
    subs = batch.to_sub_batches(['x'])
    assert subs[0]['obs'].shape == (256, 8)
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
    K = net._proposal_mixture_components
    oracle = ff_oracle if network == InferenceNetwork.FEEDFORWARD else onet
    want_loss, want_grads, _ = oracle.loss_and_grads(params, tsubs, ['x'], [8], K)
    for p in net.parameters():
        p.grad = None if p.grad is None else p.grad.zero_()
    ok, loss = net._loss(batch)
    assert ok
    assert abs(float(loss.detach()) - float(want_loss)) <= 1e-4 * abs(float(want_loss))
    loss.backward()
    for k, gw in want_grads.items():
        got = net.grad_view(k).cpu()
        scale = max(float(gw.abs().max()), 1e-6)
        assert float((got - gw).abs().max()) <= 1e-4 * scale + 1e-7, k
    # IC posterior: log-weights particle by particle against the replay
    obs = torch.linspace(0, 1, 8) * 0.4 + 1.1
    n = 4000
    with torch.no_grad():
        pyprob.seed(22)
        trace = model._run_batched(n, trace_mode=TraceMode.POSTERIOR,
                                   inference_engine=InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                   inference_network=net, observe={'x': obs})
    patch = ff_oracle.infer_sequence if network == InferenceNetwork.FEEDFORWARD else onet.infer_sequence
    with mock.patch.object(onet, 'infer_sequence', patch):
        want, covered = site_weight_terms(trace, net, obs)
    assert covered.all()
    z, u = trace.named_variables['z'].value.cpu().double(), trace.named_variables['u'].value.cpu().double()
    loc = z.view(-1, 1) * torch.linspace(0, 1, 8).double() + u.view(-1, 1)
    lik = (-(obs.double() - loc) ** 2 / (2 * 0.09) - math.log(0.3) - 0.5 * math.log(2 * math.pi)).sum(1)
    np.testing.assert_allclose(trace.log_w.cpu().numpy(), want + lik.numpy(), rtol=1e-4, atol=2e-4)


def test_offline_dataset_round_trip(cuda, tmp_path):
    from pyprob_b200.offline import OfflineDataset
    pyprob.seed(6)
    pyprob.set_verbosity(0)
    model = Net8()
    model.save_dataset(str(tmp_path), num_traces=512, num_traces_per_file=256, observe_names=['x'])
    ds = OfflineDataset(str(tmp_path))
    assert ds.observe_dims == [8]
    b = ds.next_batch(64)
    assert b.size == 64
    model.learn_inference_network(num_traces=512, batch_size=128, dataset_dir=str(tmp_path),
                                  inference_network=InferenceNetwork.LSTM, lstm_dim=32,
                                  observe_embeddings={'x': {'dim': 16}})
    assert model._inference_network._observe_in_dims == [8]


def test_errors(cuda):
    n = 16
    with pytest.raises(ValueError, match='broadcast'):
        Normal(torch.zeros(1, 5), 1.0).event_site(n, torch.zeros(4))
    with pytest.raises(ValueError, match='broadcast'):
        Normal(torch.zeros(1, 5), torch.ones(1, 4)).event_site(n)
    for d in (Categorical(torch.tensor([0.5, 0.5])), TruncatedNormal(0.0, 1.0, -1.0, 1.0)):
        with pytest.raises(NotImplementedError, match='reference'):
            d.event_site(n, torch.zeros(3, 2))

    class Latent(Model):
        def forward(self):
            return pyprob.sample(Normal(torch.zeros(1, 3), 1.0), name='v')
    with pytest.raises(NotImplementedError, match='reference'):
        Latent()._run_batched(8, trace_mode=TraceMode.POSTERIOR)
    with pytest.raises(NotImplementedError, match='reference'):
        Latent().posterior_results(4, InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS)


def test_shape_rules_on_device(cuda):
    n = 8
    ev = Normal(0.0, 1.0).event_site(n, torch.arange(8.0).view(1, 8))      # a shared 1-D event of length n
    assert ev.shape == (1, 8) and ev.site_value.shape == (n, 1, 8)
    assert Normal(0.0, 1.0).event_site(n, torch.arange(8.0)) is None        # [n]: one value per particle
    ev = Normal(torch.zeros(28, 1), 1.0).event_site(n, torch.zeros(28, 28))  # a parameter that broadcasts
    assert ev.shape == (28, 28) and ev.params[0].shape == (1, 784)
    ev = Normal(torch.zeros(n, 3), 1.0).event_site(n, torch.zeros(3))
    assert ev.params[0].shape == (n, 3)
    # outside a trace the particle count is the length of the 1-D parameters (1 here), so an [8, 3] parameter is one
    # shared event: the element-wise values keep torch's layout behind a particle axis of 1
    lp = Normal(torch.zeros(n, 3), 1.0).log_prob(torch.zeros(3))
    assert lp.shape == (1, n, 3)
    x = Normal(torch.zeros(1, 2, 3), 1.0).sample(5)
    assert x.shape == (5, 2, 3)
    np.testing.assert_allclose(float(Normal(torch.zeros(1, 3), 2.0).log_prob(torch.ones(3), sum=True)),
                               float(torch.distributions.Normal(0.0, 2.0).log_prob(torch.ones(3)).sum()), rtol=1e-6)


# ---- the per-particle path stays where no parameter has an event shape -------------------------------------------------
def test_scalar_parameter_log_prob_keeps_shape_and_kernel(cuda):
    from torch.profiler import ProfilerActivity, profile
    x = torch.randn(65536, device='cuda')
    lp = Normal(0.0, 2.0).log_prob(x)
    assert lp.shape == (65536,)
    assert torch.equal(lp, ops.normal_log_prob(x, 0.0, 2.0))
    assert Normal(torch.zeros(65536, 1, device='cuda'), 2.0).log_prob(x).shape == (65536,)

    class M(Model):
        def forward(self):
            mu = pyprob.sample(Normal(0.0, 2.0), name='mu')
            pyprob.sample(Gamma(2.0, 1.0), name='g')
            pyprob.observe(Normal(mu, 1.5), name='y')
            return mu
    pyprob.seed(2)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        M().posterior_results(20, InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS, observe={'y': OBS50[:10]},
                              num_chains=65536)
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages()]
    # the prior rescoring of every step runs the per-particle kernels; only the vector observe runs k_event
    assert any('k_score2' in k and 'NormalOp' in k for k in names)
    assert any('k_score2' in k and 'GammaOp' in k for k in names)
    assert not any('k_event' in k and 'GammaOp' in k for k in names)
    ev = [e for e in prof.key_averages() if 'k_event' in e.key]
    assert all('NormalOp' in e.key for e in ev)


# ---- against the reference fixture (tests/golden/event_golden.npz) --------------------------------------------------------
def _reference_case_model(case):
    fam = {'Normal': Normal, 'Uniform': Uniform, 'Poisson': Poisson, 'Bernoulli': Bernoulli, 'Exponential': Exponential,
           'Gamma': Gamma, 'LogNormal': LogNormal, 'Weibull': Weibull, 'Beta': Beta,
           'Binomial': lambda n, p: Binomial(n, probs=p), 'VonMises': VonMises}[case['family']]
    params = [p if isinstance(p, float) else torch.from_numpy(p).cuda() for p in case['params']]

    class M(Model):
        def forward(self):
            ps = list(params)
            if case['z'] is not None:
                z = pyprob.sample(Normal(0.0, 1.0), name='z')
                p0 = ps[0]
                ps[0] = z + p0 if isinstance(p0, float) else z.view(-1, *([1] * p0.dim())) + p0.unsqueeze(0)
            pyprob.observe(fam(*ps), name='x')
            return 0
    return M()


def test_log_weights_vs_reference_fixture(cuda):
    """Every family and broadcasting form: the log-weight of each particle is the reference's log_prob_observed."""
    from tests.test_oracle_event import load_cases
    n = 5      # no parameter or value here has a leading dimension of 5
    for case in load_cases():
        observe = {'x': torch.from_numpy(case['value'])}
        if case['z'] is not None:
            observe['z'] = case['z']
        tr = _reference_case_model(case)._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe=observe)
        lw = tr.log_w.cpu().numpy()
        np.testing.assert_allclose(lw, np.full(n, case['lpo']), rtol=2e-6, atol=2e-5,
                                   err_msg='{} {}'.format(case['family'], case['form']))


NET_TOL = {0: (1e-4, 1e-4), 1: (2e-3, 5e-2), 2: (1e-4, 1e-4)}


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('tag', ['lstm', 'ff'])
def test_network_loss_and_grads_vs_reference_fixture(cuda, tag, precision):
    """The reference's _loss and every gradient with a D = 8 observable, after load_reference_state_dict."""
    from pyprob_b200 import synthetic
    from tests import ff_oracle
    from tests.test_oracle_event import load_network
    fx = load_network(tag)
    depth = {nm: sum(1 for k in fx['params'] if k.startswith('_layers_observe_embedding.{}.'.format(nm))
                     and k.endswith('.weight')) for nm in fx['observe_names']}
    emb = {nm: {'dim': int(fx['params']['_layers_observe_embedding.{}._layers.{}.weight'.format(nm, d - 1)].shape[0]),
                'depth': d} for nm, d in depth.items()}
    kw = {'inference_network': InferenceNetwork.FEEDFORWARD} if tag == 'ff' else {'lstm_dim': fx['lstm_dim']}
    net = synthetic.build_network(emb, fx['observe_in_dims'], ff_oracle.address_table(fx), mixture_components=fx['K'],
                                  precision=precision, **kw)
    net.load_reference_state_dict(fx['params'])
    subs = [{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in sb.items()} for sb in fx['subs']]
    net._arena.grad = None
    ok, loss = net._loss(synthetic.ArrayBatch(subs))
    ltol, gtol = NET_TOL[precision]
    assert ok and abs(float(loss.detach()) - fx['loss']) <= ltol * abs(fx['loss'])
    loss.backward()
    for k, g in fx['grads'].items():
        scale = max(float(g.abs().max()), 1e-6)
        err = float((net.grad_view(k).cpu() - g).abs().max())
        assert err <= gtol * scale + 1e-6, (k, err, scale)
