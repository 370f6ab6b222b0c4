"""The proposal heads restated in plain torch with autograd, at any precision (TEST INFRASTRUCTURE ONLY).

For one row given by its raw head output x (the output of the last head layer), its value v and its prior parameters,
`head` returns log q(v), d(-log q)/dx and the proposal parameters, written straight from the reference's formulas:

* transforms      pyprob/nn/proposal_normal_normal_mixture.py, proposal_uniform_truncated_normal_mixture.py,
                  proposal_poisson_truncated_normal_mixture.py ([0, 40] window), proposal_categorical_categorical.py
                  (softmax + 1e-8), proposal_bernoulli_bernoulli.py (sigmoid + 1e-8)
* Mixture         pyprob/distributions/mixture.py: renormalise, clamp_probs, log, logsumexp
* TruncatedNormal pyprob/distributions/truncated_normal.py
* Categorical     torch Categorical(probs): normalise, clamp_probs, log, gather
* Bernoulli       torch Bernoulli(probs): clamp_probs, logits, -BCE-with-logits

The reference runs in fp32, so its probability clamps sit at the fp32 epsilon whatever `dtype` computes them: at
dtype=float64 this is the same function as the reference's, evaluated without its rounding, and at dtype=float32 it is the
reference's own arithmetic.  A log q of -inf is replaced by log(1e-8) with a zero gradient (util.replace_negative_inf, as
the CUDA training path applies it); a NaN or +inf log q is returned as it is, with a NaN gradient, because the reference
aborts such a batch.  A value outside the support of a Categorical or Bernoulli head scores NaN, as the CUDA path does.
"""
import math

import numpy as np
import torch

EPS32 = float(torch.finfo(torch.float32).eps)
LOG_EPSILON = math.log(1e-8)
LOG_SQRT_2PI = math.log(math.sqrt(2 * math.pi))
MIXTURES = ('Normal', 'Uniform', 'Poisson')


def _clamp_probs(p):
    return p.clamp(min=EPS32, max=1 - EPS32)


def _ulps32(t, n):
    return n * torch.from_numpy(np.spacing(np.abs(t.detach().float().numpy()))).to(t.dtype)


def _std_normal_cdf(x):
    return 0.5 * (1 + torch.erf(x / math.sqrt(2)))


def _normal_lp(v, mean, sd, std_nudge=0):
    d = v - mean
    if std_nudge:   # v - mean one fp32 ulp off, on its own
        d = d + _ulps32(d, std_nudge)
    return -(d ** 2) / (2 * sd ** 2) - sd.log() - LOG_SQRT_2PI


def _truncated_normal_lp(v, mean, sd, lo, hi, cdf_nudge=0, std_nudge=0):
    alpha, beta = (lo - mean) / sd, (hi - mean) / sd
    z = (v - mean) / sd
    if std_nudge:   # the three standardised values each one fp32 ulp off on its own: z and beta up, alpha down
        z, alpha, beta = z + _ulps32(z, std_nudge), alpha - _ulps32(alpha, std_nudge), beta + _ulps32(beta, std_nudge)
    ca, cb = _std_normal_cdf(alpha), _std_normal_cdf(beta)
    if cdf_nudge:
        # Phi(beta) and Phi(alpha) moved apart (or together) by three fp32 ulps each (erff's two, and one for the product and
        # sum around it), and the densities phi(alpha), phi(beta) that are their derivatives moved in opposite directions by
        # three ulps each (expf's two, one for the product): the value of Z is kept, only its slope moves
        pa, pb = (torch.exp(-0.5 * a.detach() ** 2) / math.sqrt(2 * math.pi) for a in (alpha, beta))
        ca = ca - _ulps32(ca, 3 * cdf_nudge) - _ulps32(pa, 3 * cdf_nudge) * (alpha - alpha.detach())
        cb = cb + _ulps32(cb, 3 * cdf_nudge) + _ulps32(pb, 3 * cdf_nudge) * (beta - beta.detach())
    Z = cb - ca
    inside = ((v >= lo) & (v <= hi)).to(mean.dtype)
    return torch.log(inside) + (-(z ** 2) / 2 - LOG_SQRT_2PI) - torch.log(sd * Z)


def window(family, p0, p1):
    """Truncation window of a truncated-normal head (None for Normal)."""
    if family == 'Uniform':
        return p0, p1
    if family == 'Poisson':
        return 0.0, 40.0
    return None


def proposal(family, x, K, p0, p1):
    """x [n] (one row, any dtype) or [rows, n] -> (means, stddevs, probs) of a mixture head, (probs,) of a Categorical or
    Bernoulli head: the tensors the reference's proposal layer hands to its distribution.  With rows, p0 and p1 are
    [rows, 1] (or scalars)."""
    if family == 'Categorical':
        return (torch.softmax(x, dim=-1) + 1e-8,)
    if family == 'Bernoulli':
        return (torch.sigmoid(x) + 1e-8,)
    means, stddevs, coeffs = x[..., :K], x[..., K:2 * K], torch.softmax(x[..., 2 * K:3 * K], dim=-1)
    if family == 'Normal':
        return p0 + means * p1, torch.exp(stddevs) * p1, coeffs
    if family == 'Uniform':
        rng = p1 - p0
        return p0 + torch.sigmoid(means) * rng, rng / 1000 + torch.sigmoid(stddevs) * rng * 10, coeffs
    if family == 'Poisson':
        return torch.sigmoid(means) * 40.0, torch.exp(stddevs), coeffs
    raise ValueError(family)


def log_prob(family, params, v, p0, p1, num_categories=0, cdf_nudge=0, comp_nudge=0, std_nudge=0):
    """log q(v) of the proposal distribution built from `params` (0-d tensor)."""
    if family == 'Categorical':
        if not (0 <= v < num_categories) or v != int(v):
            return params[0].sum() * float('nan')
        probs = params[0] / params[0].sum()
        return torch.log(_clamp_probs(probs))[int(v)]
    if family == 'Bernoulli':
        if v not in (0.0, 1.0):
            return params[0].sum() * float('nan')
        pc = _clamp_probs(params[0][0])
        logits = torch.log(pc) - torch.log1p(-pc)
        return -torch.nn.functional.binary_cross_entropy_with_logits(logits, logits.new_tensor(v))
    means, stddevs, coeffs = params
    v = means.new_tensor(v)
    w = window(family, p0, p1)
    comp = _normal_lp(v, means, stddevs, std_nudge) if w is None else \
        _truncated_normal_lp(v, means, stddevs, w[0], w[1], cdf_nudge, std_nudge)
    if comp_nudge:  # each component's log density moved by two fp32 ulps of its parts, alternately up and down
        mag = comp.detach().abs() + stddevs.detach().log().abs() + 1
        sign = comp_nudge * (1 - 2 * (torch.arange(len(comp)) % 2)).to(comp.dtype)
        comp = comp + sign * _ulps32(mag, 2)
    probs = coeffs / coeffs.sum()
    return torch.logsumexp(torch.log(_clamp_probs(probs)) + comp, dim=0)


def head(family, x, v, p0=0.0, p1=0.0, K=None, num_categories=0, dtype=torch.float64, round_params=False, nudge=None):
    """One row: x = raw head output (fp32 values, promoted to `dtype`), v, prior0, prior1 (fp32 values).

    round_params: round the proposal parameters (means, stddevs, probs) to fp32 before log q, keeping the unrounded
    derivative of the transform.  The result is the log q of the distribution an fp32 head actually proposes, which can
    differ from the exact one by far more than fp32 rounding (sigmoid(30) * 40 is 40 in fp32: a mean exactly on the
    Poisson window's edge).
    nudge: one sign per proposal parameter tensor (+1, -1 or 0): move every entry of it by one fp32 ulp that way, again
    keeping the unrounded derivative; an optional further sign moves the truncated normal's Phi(beta) and Phi(alpha) apart
    by three fp32 ulps each and the densities in their slopes by three ulps (erff's and expf's error bounds plus one
    rounding), a next one each component's log density by two ulps of its parts, and a last one the standardised values
    z, alpha and beta (v - mean for Normal) by one ulp each.  How far that moves log q and its
    gradient is how much one rounding of these quantities, which any fp32 evaluation makes, can cost: the conditioning of
    the expression.

    Returns {'lp': float, 'grad': float64 [len(x)] = d(-log q)/dx, 'params': tuple of float64 arrays,
    'repaired': log q was -inf and is log(1e-8)}."""
    x32 = np.asarray(x, np.float32)
    xt = torch.tensor(x32, dtype=dtype, requires_grad=True)
    v = float(np.float32(v))
    p0, p1 = (torch.tensor(float(np.float32(a)), dtype=dtype) for a in (p0, p1))
    if family in MIXTURES:
        K = len(x32) // 3 if K is None else K
        assert len(x32) == 3 * K
    params = proposal(family, xt, K, p0, p1)
    if round_params:
        params = tuple(p + (p.float().to(dtype) - p).detach() for p in params)
    if nudge is not None:
        params = tuple(p + _ulps32(p, sg) for p, sg in zip(params, nudge))
    lp = log_prob(family, params, v, p0, p1, num_categories or len(x32),
                  *(nudge[3:6] if nudge is not None else ()))
    out = {'params': tuple(p.detach().double().numpy() for p in params), 'repaired': False}
    lpv = float(lp.detach())
    if lpv == -math.inf:
        out.update(lp=LOG_EPSILON, grad=np.zeros(len(x32)), repaired=True)
    elif not math.isfinite(lpv):
        out.update(lp=lpv, grad=np.full(len(x32), np.nan))
    else:
        (-lp).backward()
        out.update(lp=lpv, grad=xt.grad.double().numpy())
    return out
