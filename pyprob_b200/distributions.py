"""Particle-batched distributions backed by the CUDA scoring / sampling kernels.

Public protocol follows the reference (pyprob/distributions/distribution.py:9-95): ``name``,
``_address_suffix``, ``sample()``, ``log_prob(value, sum=False)``, ``mean/stddev/variance``.  Parameters may
be Python scalars (shared by all particles) or length-n CUDA tensors (one per particle).  There is no CPU
path: every sample/log_prob is a kernel launch over the particle axis.

Event shapes (observations only).  A site over n particles has an event shape E (D = prod(E) elements) formed as torch's
``log_prob`` broadcasts the value against the parameters:
  * a parameter that is a Python scalar or a 1-D [n] tensor keeps its meaning (shared, one per particle), and so does
    an [n, 1, ...] tensor of n elements (``w.view(-1, 1)``); a tensor with at least 2 dims and leading size n is one
    event per particle, [n, *E]; [1, *E] or any other shape (a 1-D tensor of another length included) is one event
    shared by all particles.  A parameter that only broadcasts to E (a [28, 1] against a [28, 28] value) is expanded;
  * an observed value is data, the same for every particle: a scalar, or a 1-D [n] tensor under a distribution whose
    parameters have no event shape, keeps today's per-particle meaning; any other shape is one shared event.  So a
    shared 1-D event of length n must be passed as [1, n];
  * parameters and value that do not broadcast raise ValueError.
The site's weight term is likelihood_importance * sum_j log p(v_j), the reference's log_prob(value, sum=True) for one
particle (pyprob/state.py:147); ``log_prob(value)`` returns the element-wise [n, *E] values and ``sample(n)`` draws
[n, *E].  Categorical, Mixture and TruncatedNormal have no event form (NotImplementedError).
"""
import math

import torch

from . import ops, util

_shard_first_index = 0  # global index of particle 0 on this rank (set by the engine for sharded runs)


def set_shard_first_index(i):
    global _shard_first_index
    _shard_first_index = int(i)


def _as_param(x):
    if torch.is_tensor(x):
        return x.to(device='cuda', dtype=torch.float32).reshape(-1) if x.numel() > 1 else float(x)
    return float(x)


def _params(*xs):
    """-> (parameters as _as_param gives them, parameters with their shape kept (for event sites))"""
    shaped = []
    for x in xs:
        if torch.is_tensor(x) and x.numel() > 1 and x.dim() >= 2:
            shaped.append(x.to(device='cuda', dtype=torch.float32))
        else:
            shaped.append(_as_param(x))
    return tuple(p.reshape(-1) if torch.is_tensor(p) else p for p in shaped), tuple(shaped)


class EventSite:
    """A site with an event shape, resolved against n particles: event operands for ops.event_log_prob /
    ops.event_sample ([n, 1] per particle, [1, D] shared event, [n, D] event per particle, or a scalar)."""

    def __init__(self, family, shape, n, params, value=None):
        self.family, self.shape, self.n = family, tuple(shape), int(n)
        self.D = int(math.prod(self.shape))
        self.params, self.value = params, value

    @property
    def site_value(self):
        """The observed value as the trace holds it: an [n, *E] view of the one shared row (row stride 0, no copy)."""
        v = self.value
        if not torch.is_tensor(v):
            v = torch.full((1,), float(v), device='cuda')
        return (v.reshape(1) if v.numel() == 1 else v.reshape(self.shape)).expand(self.n, *self.shape)

    def score_into(self, acc, scale):
        ops.event_log_prob(self.family, self.value, self.params, self.n, self.D, acc=acc, acc_scale=scale)

    def log_prob(self):
        return ops.event_log_prob(self.family, self.value, self.params, self.n, self.D).view(self.n, *self.shape)

    def sample(self, with_log_prob=False):
        s, o, f = util._seed, util.next_draw_offset(), _shard_first_index
        out = ops.event_sample(self.family, self.params, self.n, self.D, s, o, f, with_log_prob)
        if with_log_prob:
            return out[0].view(self.n, *self.shape), out[1]
        return out.view(self.n, *self.shape)


_NO_VALUE = object()
_REFERENCE_NOTE = ('(the reference scores and draws such sites with torch, pyprob/state.py:118-219; pyprob_b200 supports '
                   'tensor-valued observations of the families with an element-wise log_prob)')


def _broadcast_events(shapes):
    try:
        return tuple(torch.broadcast_shapes(*shapes))
    except RuntimeError as e:
        raise ValueError('event shapes do not broadcast: {} ({})'.format(
            ', '.join(str(tuple(s)) for s in shapes), e)) from None


def _param_form(p, n):
    """(kind, event shape) of a parameter over n particles: a scalar; one per particle (a 1-D [n] tensor, or [n, 1, ...]);
    one event per particle ([n, *E], at least 2 dims); or one shared event ([1, *E], or any other shape)."""
    if not torch.is_tensor(p):
        return 'scalar', ()
    if p.dim() >= 1 and p.size(0) == n and p.numel() == n:
        return 'particle', ()
    if p.dim() <= 1:
        return 'event', tuple(p.shape)
    if p.size(0) == n:
        return 'particle_event', tuple(p.shape[1:])
    if p.size(0) == 1:
        return 'event', tuple(p.shape[1:])
    return 'event', tuple(p.shape)


def _event_layout(shaped, n, value=_NO_VALUE, per_particle_value=False):
    """The shape rules (module docstring), host-side only: -> None when the site is scalar (today's path), else
    (E, [(kind, event shape)] per parameter, value form, value), kind / form one of 'scalar', 'particle',
    'particle_event', 'event' (shared)."""
    param_event = any(_param_form(p, n)[0] == 'event' or _param_form(p, n)[0] == 'particle_event' for p in shaped)
    if value is _NO_VALUE or value is None:
        vform = None
    elif isinstance(value, (int, float)):
        vform = 'scalar'
    else:
        if not torch.is_tensor(value):
            value = torch.as_tensor(value, dtype=torch.float32)
        if value.numel() == 1:
            vform = 'scalar'
        elif per_particle_value and value.dim() >= 2 and value.size(0) == n:
            vform = 'particle_event'
        elif value.dim() <= 1 and value.numel() == n and not param_event:
            return None
        else:
            vform = 'event'
    if not param_event and vform in (None, 'scalar'):
        return None
    forms = [_param_form(p, n) for p in shaped]
    shapes = [e for _, e in forms]
    if vform in ('event', 'particle_event'):
        shapes.append(tuple(value.shape[1:]) if vform == 'particle_event' else tuple(value.shape))
    E = _broadcast_events(shapes)
    if math.prod(E) <= 1 and vform in (None, 'scalar'):
        return None                     # [n, 1, ...] parameters: one value per particle, today's path
    return E, forms, vform, value


def _resolve_event(dist, n, value=_NO_VALUE, per_particle_value=False):
    """The EventSite of `dist` over n particles observing `value`, or None when the site is scalar (today's path)."""
    shaped = dist._shaped
    layout = _event_layout(shaped, n, value, per_particle_value)
    if layout is None:
        return None
    E, forms, vform, value = layout
    D = math.prod(E)

    def particle_rows(t, e):
        t = t.reshape(n, *([1] * (len(E) - len(e))), *e)
        return t.expand(n, *E).reshape(n, D)

    def shared_row(t, e):
        return t.reshape(e).expand(E).reshape(1, D)
    params = []
    for p, (kind, e) in zip(shaped, forms):
        if kind == 'scalar':
            params.append(p)
        elif kind == 'particle':
            params.append(p.reshape(n, 1))
        elif kind == 'particle_event':
            params.append(particle_rows(p, e))
        else:
            params.append(shared_row(p, e))
    if vform is None:
        v = None
    elif vform == 'scalar':
        v = float(value) if not torch.is_tensor(value) else value.to(device='cuda', dtype=torch.float32).reshape(1)
    else:
        t = value.to(device='cuda', dtype=torch.float32)
        v = particle_rows(t, tuple(t.shape[1:])) if vform == 'particle_event' else shared_row(t, tuple(t.shape))
    return EventSite(dist.family, E, n, params, v)


def _length(*params):
    n = 1
    for p in params:
        if torch.is_tensor(p):
            n = max(n, p.numel())
    return n


def _value(v, n=None):
    if not torch.is_tensor(v):
        v = torch.tensor(v, dtype=torch.float32)
    v = v.to(device='cuda', dtype=torch.float32).reshape(-1)
    if n is not None and v.numel() == 1 and n > 1:
        v = v.expand(n).contiguous()
    return v


class Distribution:
    _shaped = ()   # the parameters with their shapes (event sites); empty for the families without an event form

    def __init__(self, name, address_suffix):
        self.name = name
        self._address_suffix = address_suffix

    @property
    def batch_length(self):
        return 1

    def _draw(self, n, with_log_prob):
        raise NotImplementedError()

    def _has_event_param(self):
        """A parameter of at least 2 dims that is not one column of values ([n, 1, ...])."""
        return any(torch.is_tensor(p) and p.dim() >= 2 and p.numel() != p.size(0) for p in self._shaped)

    def _standalone_n(self):
        """Particles of a call outside a trace: the length of the one-per-particle parameters (1-D, or [n, 1, ...]);
        event parameters do not count."""
        if self._has_event_param():
            return max([p.size(0) for p in self._shaped if torch.is_tensor(p) and p.numel() == p.size(0)] + [1])
        return self.batch_length

    def event_site(self, n, value=_NO_VALUE):
        """The EventSite of this distribution over n particles observing `value` (a data value, shared by every
        particle), or None when the site is scalar.  Raises ValueError when the shapes do not broadcast and
        NotImplementedError for a family without an event form."""
        if not self._shaped:
            if value is not _NO_VALUE and value is not None and not isinstance(value, (int, float)):
                v = value if torch.is_tensor(value) else torch.as_tensor(value)
                if v.numel() > 1 and not (v.dim() <= 1 and v.numel() == n):
                    raise NotImplementedError('{} observations with an event shape {} {}'.format(
                        self.name, tuple(v.shape), _REFERENCE_NOTE))
            return None
        return _resolve_event(self, n, value)

    def sample(self, n=None, with_log_prob=False):
        n = self._standalone_n() if n is None else n
        if self._shaped:
            ev = _resolve_event(self, n)
            if ev is not None:
                return ev.sample(with_log_prob)
        return self._draw(n, with_log_prob)

    def log_prob(self, value, sum=False):
        ev = None
        if self._has_event_param() and torch.is_tensor(value) and value.numel() > 1:
            # without an event parameter, log_prob is today's element-wise [N] kernel call
            n = self._standalone_n()
            if value.dim() >= 2 and n == 1:
                n = value.size(0)
            ev = _resolve_event(self, n, value, per_particle_value=True)
        lp = ev.log_prob() if ev is not None else self._log_prob(value)
        return lp.sum() if sum else lp

    def prob(self, value):
        return torch.exp(self.log_prob(value))

    @property
    def stddev(self):
        return self.variance ** 0.5 if torch.is_tensor(self.variance) else math.sqrt(self.variance)

    def _prior_params(self):
        """The prior parameters a proposal head takes as inputs: (loc, scale) for Normal, (low, high) for Uniform,
        (None, None) for the other families."""
        return None, None

    def _seed_args(self):
        return util._seed, util.next_draw_offset(), _shard_first_index


class _ElementWise(Distribution):
    """A family with an element-wise log_prob (ops.EVENT_FAMILIES), scored and drawn by the family-id kernels; the
    parameters are kept in the kernels' order (self._params), each a Python scalar or a length-n CUDA tensor."""

    def __init__(self, name, *params):
        super().__init__(name, name)
        self.family = ops.EVENT_FAMILIES[name]
        self._params, self._shaped = _params(*params)

    @property
    def batch_length(self):
        return _length(*self._params)

    def _draw(self, n, with_log_prob):
        s, o, f = self._seed_args()
        return ops._sample(self.family, self._params, n, s, o, f, with_log_prob, 'cuda')

    def _log_prob(self, value):
        return ops._score(self.family, _value(value, self.batch_length), self._params, None, None, 1.0)

    def score_into(self, value, acc, scale):
        ops._score(self.family, value, self._params, None, acc, scale)


class Normal(_ElementWise):
    def __init__(self, loc, scale):
        super().__init__('Normal', loc, scale)
        self.loc, self.scale = self._params

    mean = property(lambda self: self.loc)
    variance = property(lambda self: self.scale ** 2)
    stddev = property(lambda self: self.scale)

    def _prior_params(self):
        return self.loc, self.scale

    def __repr__(self):
        return 'Normal({}, {})'.format(self.loc, self.scale)


class Uniform(_ElementWise):
    def __init__(self, low, high):
        super().__init__('Uniform', low, high)
        self.low, self.high = self._params

    mean = property(lambda self: (self.low + self.high) / 2)
    variance = property(lambda self: (self.high - self.low) ** 2 / 12)

    def _prior_params(self):
        return self.low, self.high

    def __repr__(self):
        return 'Uniform(low={}, high={})'.format(self.low, self.high)


class Poisson(_ElementWise):
    def __init__(self, rate):
        super().__init__('Poisson', rate)
        self.rate, = self._params

    mean = property(lambda self: self.rate)
    variance = property(lambda self: self.rate)

    def __repr__(self):
        return 'Poisson({})'.format(self.rate)


class Bernoulli(_ElementWise):
    """probs (or logits, converted with a sigmoid): a scalar shared by all particles or one per particle (reference:
    bernoulli.py, torch Bernoulli).  Values are 0. / 1.; any other value scores NaN.

    log_prob always works from probs clamped to [eps32, 1 - eps32], so it is at least log(eps32) = -15.9.  Built from
    logits, torch's Bernoulli scores with the raw logits instead and agrees only while |logits| < about 16: at
    logits = -30 it gives -30 for the value 1 where this gives -15.9 (DESIGN.md section 8)."""

    def __init__(self, probs=None, logits=None):
        if probs is None:
            if logits is None:
                raise ValueError('Either probs or logits must be given.')
            probs = torch.sigmoid(torch.as_tensor(logits, dtype=torch.float32))
        super().__init__('Bernoulli', probs)
        self.probs, = self._params

    @property
    def logits(self):
        p = self.probs
        return torch.log(p) - torch.log1p(-p) if torch.is_tensor(p) else math.log(p) - math.log1p(-p)

    mean = property(lambda self: self.probs)
    variance = property(lambda self: self.probs * (1 - self.probs))

    def __repr__(self):
        return 'Bernoulli({})'.format(self.probs)


def _moment(fn, *params):
    """fn over fp32 tensors (the reference's torch moments): a tensor when a parameter is per particle, a Python float when
    every parameter is a scalar, like the moments of the other families."""
    if any(torch.is_tensor(p) for p in params):
        return fn(*(p if torch.is_tensor(p) else torch.tensor(p, dtype=torch.float32, device='cuda') for p in params))
    return float(fn(*(torch.tensor(p, dtype=torch.float32) for p in params)))


class Exponential(_ElementWise):
    """rate: a scalar shared by all particles or one per particle (reference: exponential.py, torch Exponential).  Values
    below 0 and rates that are not positive score NaN."""

    def __init__(self, rate):
        super().__init__('Exponential', rate)
        self.rate, = self._params

    mean = property(lambda self: _moment(lambda r: 1 / r, self.rate))
    variance = property(lambda self: _moment(lambda r: r.pow(-2), self.rate))

    def __repr__(self):
        return 'Exponential({})'.format(self.rate)


class Gamma(_ElementWise):
    """Gamma(concentration, rate) (reference: gamma.py, torch Gamma).  Draws are clamped below at the smallest normal
    float, as torch's are, so no draw is 0."""

    def __init__(self, concentration, rate):
        super().__init__('Gamma', concentration, rate)
        self.concentration, self.rate = self._params

    mean = property(lambda self: _moment(lambda c, r: c / r, self.concentration, self.rate))
    variance = property(lambda self: _moment(lambda c, r: c / r.pow(2), self.concentration, self.rate))

    def __repr__(self):
        return 'Gamma(concentration={}, rate={})'.format(self.concentration, self.rate)


class LogNormal(_ElementWise):
    """LogNormal(loc, scale): exp of a Normal(loc, scale) (reference: log_normal.py, torch LogNormal)."""

    def __init__(self, loc, scale):
        super().__init__('LogNormal', loc, scale)
        self.loc, self.scale = self._params

    mean = property(lambda self: _moment(lambda m, s: (m + s.pow(2) / 2).exp(), self.loc, self.scale))
    variance = property(lambda self: _moment(lambda m, s: (s.pow(2).exp() - 1) * (2 * m + s.pow(2)).exp(),
                                             self.loc, self.scale))

    def __repr__(self):
        return 'LogNormal({}, {})'.format(self.loc, self.scale)


class Weibull(_ElementWise):
    """Weibull(scale, concentration) (reference: weibull.py, torch Weibull)."""

    def __init__(self, scale, concentration):
        super().__init__('Weibull', scale, concentration)
        self.scale, self.concentration = self._params

    mean = property(lambda self: _moment(lambda s, k: s * torch.exp(torch.lgamma(1 + k.reciprocal())),
                                         self.scale, self.concentration))
    variance = property(lambda self: _moment(
        lambda s, k: s.pow(2) * (torch.exp(torch.lgamma(1 + 2 * k.reciprocal())) -
                                 torch.exp(2 * torch.lgamma(1 + k.reciprocal()))), self.scale, self.concentration))

    def __repr__(self):
        return 'Weibull(scale={}, concentration={})'.format(self.scale, self.concentration)


class Beta(_ElementWise):
    """Beta(concentration1, concentration0) on [low, high] (reference: beta.py): a draw is low + (high - low) u with
    u ~ torch Beta(concentration1, concentration0), and log_prob(x) is torch's Beta log_prob of u = (x - low) / (high - low).

    Like the reference, log_prob has no -log(high - low) term, so with low / high other than 0 / 1 it is not the density
    of x (DESIGN.md section 8)."""

    def __init__(self, concentration1, concentration0, low=0, high=1):
        super().__init__('Beta', concentration1, concentration0, low, high)
        self.concentration1, self.concentration0, self.low, self.high = self._params

    @property
    def mean(self):
        return _moment(lambda a, b, lo, hi: lo + a / (a + b) * (hi - lo), self.concentration1, self.concentration0,
                       self.low, self.high)

    @property
    def variance(self):
        def var(a, b, lo, hi):
            total = a + b
            return a * b / (total.pow(2) * (total + 1)) * (hi - lo) * (hi - lo)
        return _moment(var, self.concentration1, self.concentration0, self.low, self.high)

    def __repr__(self):
        return 'Beta(concentration1={}, concentration0={}, low={}, high={})'.format(
            self.concentration1, self.concentration0, self.low, self.high)


class Binomial(_ElementWise):
    """Binomial(total_count, probs) (reference: binomial.py, torch Binomial); total_count and probs are each a scalar or
    one per particle.  Values are the integers 0 .. total_count stored as floats; any other value scores NaN.

    Scored in torch's logits form from probs clamped to [eps32, 1 - eps32], as torch does for a Binomial built from probs.
    Built from logits (converted with a sigmoid), torch's Binomial scores with the raw logits instead.  The fp32 round trip
    through probs costs the logit a relative error of about 6e-8 exp(|logits|) and log_prob multiplies it by up to
    total_count: at total_count = 1000 the two agree to 1e-4 for |logits| <= 5, differ by 9 at logits = 12, and beyond
    |logits| = 16 the clamp takes over (DESIGN.md section 8)."""

    def __init__(self, total_count=1, probs=None, logits=None):
        if probs is None:
            if logits is None:
                raise ValueError('Either probs or logits must be given.')
            probs = torch.sigmoid(torch.as_tensor(logits, dtype=torch.float32))
        super().__init__('Binomial', total_count, probs)
        self.total_count, self.probs = self._params

    @property
    def logits(self):
        p = self.probs
        return torch.log(p) - torch.log1p(-p) if torch.is_tensor(p) else math.log(p) - math.log1p(-p)

    mean = property(lambda self: _moment(lambda n, p: n * p, self.total_count, self.probs))
    variance = property(lambda self: _moment(lambda n, p: n * p * (1 - p), self.total_count, self.probs))

    def __repr__(self):
        return 'Binomial(total_count={}, probs={})'.format(self.total_count, self.probs)


class VonMises(_ElementWise):
    """VonMises(loc, concentration) (reference: von_mises.py, torch VonMises).  Draws lie in [-pi, pi); any real value
    can be scored.  variance is torch's circular variance 1 - I1(concentration) / I0(concentration)."""

    def __init__(self, loc, concentration):
        super().__init__('VonMises', loc, concentration)
        self.loc, self.concentration = self._params

    mean = property(lambda self: self.loc)
    # torch's own fp32 formula, so that the value is the reference's (it loses digits at large concentration)
    variance = property(lambda self: _moment(
        lambda k: torch.distributions.VonMises(torch.zeros_like(k), k, validate_args=False).variance, self.concentration))

    def __repr__(self):
        return 'VonMises(loc={}, concentration={})'.format(self.loc, self.concentration)


class Categorical(Distribution):
    """probs: [C] shared or [n, C] per particle (unnormalised, like the reference: categorical.py:8-21)."""

    def __init__(self, probs=None, logits=None):
        if probs is None:
            probs = torch.softmax(torch.as_tensor(logits, dtype=torch.float32), dim=-1)
        probs = torch.as_tensor(probs, dtype=torch.float32).to('cuda')
        if probs.dim() == 0:
            raise ValueError('probs cannot be a scalar.')
        self._probs = probs.contiguous()
        self._num_categories = probs.size(-1)
        super().__init__('Categorical', 'Categorical(len_probs:{})'.format(self._num_categories))

    @property
    def batch_length(self):
        return self._probs.size(0) if self._probs.dim() == 2 else 1

    num_categories = property(lambda self: self._num_categories)

    @property
    def probs(self):
        return self._probs / self._probs.sum(-1, keepdim=True)

    @property
    def mean(self):
        return (self.probs * torch.arange(self._num_categories, device='cuda')).sum(-1)

    @property
    def variance(self):
        idx = torch.arange(self._num_categories, device='cuda')
        return (self.probs * idx ** 2).sum(-1) - self.mean ** 2

    def _draw(self, n, with_log_prob):
        s, o, f = self._seed_args()
        return ops.categorical_sample(self._probs, n, s, o, f, with_log_prob)

    def _log_prob(self, value):
        return ops.categorical_log_prob(_value(value, self.batch_length), self._probs)

    def score_into(self, value, acc, scale):
        ops.categorical_log_prob(value, self._probs, acc=acc, acc_scale=scale)

    def __repr__(self):
        return 'Categorical(num_categories={})'.format(self._num_categories)


class TruncatedNormal(Distribution):
    """Scored and drawn as a one-component truncated mixture (reference: truncated_normal.py:11-112)."""

    def __init__(self, mean_non_truncated, stddev_non_truncated, low, high):
        super().__init__('TruncatedNormal', 'TruncatedNormal')
        self.mean_non_truncated, self.stddev_non_truncated = _as_param(mean_non_truncated), _as_param(stddev_non_truncated)
        self.low, self.high = _as_param(low), _as_param(high)

    @property
    def batch_length(self):
        return _length(self.mean_non_truncated, self.stddev_non_truncated, self.low, self.high)

    def _rows(self, n):
        def col(p):
            t = p if torch.is_tensor(p) else torch.full((n,), p, device='cuda')
            return t.reshape(-1, 1).expand(n, 1).contiguous()
        return col(self.mean_non_truncated), col(self.stddev_non_truncated), torch.ones(n, 1, device='cuda')

    def _draw(self, n, with_log_prob):
        s, o, f = self._seed_args()
        m, sd, p = self._rows(n)
        return ops.mixture_truncated_normal_sample(m, sd, p, self.low, self.high, n, s, o, f, with_log_prob)

    def _log_prob(self, value):
        v = _value(value, self.batch_length)
        m, sd, p = self._rows(v.numel())
        return ops.mixture_truncated_normal_log_prob(v, m, sd, p, self.low, self.high)

    def score_into(self, value, acc, scale):
        m, sd, p = self._rows(value.numel())
        ops.mixture_truncated_normal_log_prob(value, m, sd, p, self.low, self.high, acc=acc, acc_scale=scale)


class Mixture(Distribution):
    """Mixture of K Normals or K TruncatedNormals with per-particle parameters.

    Either built like the reference (``Mixture([Normal(..), ...], probs)``, mixture.py:8-30) or directly from
    parameter rows with ``Mixture.from_rows``."""

    def __init__(self, distributions, probs=None):
        super().__init__('Mixture', 'Mixture({})'.format(', '.join(d._address_suffix for d in distributions)))
        K = len(distributions)
        n = max(d.batch_length for d in distributions)
        trunc = isinstance(distributions[0], TruncatedNormal)

        def stack(attr):
            cols = []
            for d in distributions:
                p = getattr(d, attr)
                cols.append(p.reshape(-1) if torch.is_tensor(p) else torch.full((n,), p, device='cuda'))
            return torch.stack(cols, dim=1).contiguous()
        self._means = stack('mean_non_truncated' if trunc else 'loc')
        self._stddevs = stack('stddev_non_truncated' if trunc else 'scale')
        if probs is None:
            probs = torch.full((K,), 1.0 / K)
        probs = torch.as_tensor(probs, dtype=torch.float32).to('cuda')
        self._probs = (probs.expand(n, K) if probs.dim() == 1 else probs).contiguous()
        self._low = distributions[0].low if trunc else None
        self._high = distributions[0].high if trunc else None
        self._trunc, self._n, self.length = trunc, n, K

    @classmethod
    def from_rows(cls, means, stddevs, probs, low=None, high=None):
        self = cls.__new__(cls)
        Distribution.__init__(self, 'Mixture', 'Mixture')
        self._means, self._stddevs, self._probs = means, stddevs, probs
        self._low, self._high = low, high
        self._trunc, self._n, self.length = low is not None, means.size(0), means.size(1)
        return self

    @property
    def batch_length(self):
        return self._n

    @property
    def probs(self):
        return self._probs / self._probs.sum(-1, keepdim=True)

    @property
    def mean(self):
        if self._trunc:
            raise NotImplementedError('mean of a truncated mixture')
        return (self.probs * self._means).sum(-1)

    @property
    def variance(self):
        m = self.mean.view(-1, 1)
        return (self.probs * ((self._means - m) ** 2 + self._stddevs ** 2)).sum(-1)

    def _draw(self, n, with_log_prob):
        s, o, f = self._seed_args()
        if self._trunc:
            return ops.mixture_truncated_normal_sample(self._means, self._stddevs, self._probs, self._low, self._high,
                                                       n, s, o, f, with_log_prob)
        return ops.mixture_normal_sample(self._means, self._stddevs, self._probs, n, s, o, f, with_log_prob)

    def _log_prob(self, value):
        v = _value(value, self._n)
        if self._trunc:
            return ops.mixture_truncated_normal_log_prob(v, self._means, self._stddevs, self._probs, self._low,
                                                         self._high)
        return ops.mixture_normal_log_prob(v, self._means, self._stddevs, self._probs)

    def score_into(self, value, acc, scale):
        if self._trunc:
            ops.mixture_truncated_normal_log_prob(value, self._means, self._stddevs, self._probs, self._low, self._high,
                                                  acc=acc, acc_scale=scale)
        else:
            ops.mixture_normal_log_prob(value, self._means, self._stddevs, self._probs, acc=acc, acc_scale=scale)
