"""Oracle: log_prob of the Exponential, Gamma, LogNormal, Weibull, Beta, Binomial and VonMises families, restated with
torch-CPU tensor ops (TEST INFRASTRUCTURE ONLY).

The reference wraps torch.distributions (pyprob/distributions/{exponential,gamma,log_normal,weibull,beta,binomial,
von_mises}.py), which validates its arguments and raises on a value outside the support or an invalid parameter.  These
functions score element-wise instead and give NaN there, the value the kernels give.  Inputs broadcast; every operation is
fp32, in torch's order, so the values equal the reference's to the last bit or nearly.
"""
import math

import torch

EPS32 = torch.finfo(torch.float32).eps
LOG_SQRT_2PI = math.log(math.sqrt(2 * math.pi))

# Abramowitz & Stegun 9.8.1 / 9.8.2, the coefficients torch.distributions.von_mises uses for log I0
_I0_SMALL = [1.0, 3.5156229, 3.0899424, 1.2067492, 0.2659732, 0.360768e-1, 0.45813e-2]
_I0_LARGE = [0.39894228, 0.1328592e-1, 0.225319e-2, -0.157565e-2, 0.916281e-2, -0.2057706e-1, 0.2635537e-1,
             -0.1647633e-1, 0.392377e-2]


def _t(*xs):
    return torch.broadcast_tensors(*(torch.as_tensor(x, dtype=torch.float32) for x in xs))


def _nan_unless(ok, lp):
    return torch.where(ok, lp, torch.full_like(lp, float('nan')))


def exponential_log_prob(value, rate):
    v, r = _t(value, rate)
    return _nan_unless((r > 0) & (v >= 0), r.log() - r * v)


def gamma_log_prob(value, concentration, rate):
    v, c, r = _t(value, concentration, rate)
    lp = torch.xlogy(c, r) + torch.xlogy(c - 1, v) - r * v - torch.lgamma(c)
    return _nan_unless((c > 0) & (r > 0) & (v >= 0), lp)


def lognormal_log_prob(value, loc, scale):
    v, m, s = _t(value, loc, scale)
    x = v.log()
    normal = -((x - m) ** 2) / (2 * s ** 2) - s.log() - LOG_SQRT_2PI
    return _nan_unless((s > 0) & (v > 0), -x + normal)


def weibull_log_prob(value, scale, concentration):
    """torch's TransformedDistribution(Exponential(1), [PowerTransform(1/k), AffineTransform(0, scale)]) step by step."""
    v, lam, k = _t(value, scale, concentration)
    e = k.reciprocal()
    x1 = v / lam
    x0 = x1.pow(1 / e)
    lp = (0.0 - lam.abs().log()) - (e * x1 / x0).abs().log()
    lp = lp + (-x0)
    return _nan_unless((lam > 0) & (k > 0) & (v > 0), lp)


def beta_log_prob(value, concentration1, concentration0, low=0.0, high=1.0):
    """pyprob/distributions/beta.py:38-40: torch Beta(c1, c0).log_prob((x - low) / (high - low)), no Jacobian term."""
    v, a, b, lo, hi = _t(value, concentration1, concentration0, low, high)
    u = (v - lo) / (hi - lo)
    lp = (torch.xlogy(a - 1.0, u) + torch.xlogy(b - 1.0, 1.0 - u)) + torch.lgamma(a + b) - (torch.lgamma(a) + torch.lgamma(b))
    return _nan_unless((a > 0) & (b > 0) & (u >= 0) & (u <= 1), lp)


def binomial_log_prob(value, total_count, probs=None, logits=None):
    """torch Binomial: from probs, logits = log(pc) - log1p(-pc) with pc = clamp(probs, eps, 1 - eps); from logits, the
    raw logits."""
    if logits is None:
        v, n, p = _t(value, total_count, probs)
        pc = p.clamp(min=EPS32, max=1 - EPS32)
        lg = torch.log(pc) - torch.log1p(-pc)
        ok_p = (p >= 0) & (p <= 1)
    else:
        v, n, lg = _t(value, total_count, logits)
        ok_p = ~torch.isnan(lg)
    cz = (lg.clamp(min=0) + lg - lg.clamp(max=0)) / 2
    norm = n * cz + n * torch.log1p(torch.exp(-lg.abs())) - torch.lgamma(n + 1)
    lp = v * lg - torch.lgamma(v + 1) - torch.lgamma(n - v + 1) - norm
    ok_n = (n >= 0) & (torch.remainder(n, 1) == 0)
    ok_v = (v >= 0) & (v <= n) & (torch.remainder(v, 1) == 0)
    return _nan_unless(ok_n & ok_p & ok_v, lp)


def _poly(y, coef):
    result = torch.full_like(y, coef[-1])
    for c in reversed(coef[:-1]):
        result = c + y * result
    return result


def log_i0(x):
    """torch.distributions.von_mises._log_modified_bessel_fn(x, order=0)."""
    x = torch.as_tensor(x, dtype=torch.float32)
    y = x / 3.75
    small = _poly(y * y, _I0_SMALL).log()
    large = x - 0.5 * x.log() + _poly(3.75 / x, _I0_LARGE).log()
    return torch.where(x < 3.75, small, large)


def von_mises_log_prob(value, loc, concentration):
    v, m, k = _t(value, loc, concentration)
    lp = k * torch.cos(v - m)
    lp = lp - math.log(2 * math.pi) - log_i0(k)
    return _nan_unless((k > 0) & ~torch.isnan(v) & ~torch.isnan(m), lp)
