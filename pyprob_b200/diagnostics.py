"""MCMC diagnostics computed on the GPU: Gelman-Rubin R-hat against the iteration and per-chain autocorrelation
(reference: pyprob/diagnostics.py:714-873, ``gelman_rubin`` and ``autocorrelation``).

The reference reads named variables out of Empiricals of ``Trace`` objects.  Here a posterior holds ``map_func`` values,
so the diagnostics read those: one Empirical from ``Model.posterior(..., inference_engine=LMH / RMH, num_chains=C)``
(values ``[S * C]`` or ``[S * C, V]`` in step-major order, entry ``k * C + c`` is chain c after recorded step k), or a
list of Empiricals of one chain each (the reference's form; truncated to the shortest).  The V columns of the values are
the variables; ``names`` labels them (default: the column indices).  C is read from the Empirical's metadata
(``op='posterior', num_chains=C``) unless ``num_chains`` is given.  A slice keeps that metadata, but it must start at a
multiple of C to keep every entry on its chain: ``post[burn_in * C:]``.

The statistics are the reference's formulas in fp64 (DESIGN.md section 8), computed by the kernels of
``csrc/diagnostics.cu`` with a fixed number of launches: no Python loop over chains, steps, iterations or lags, and one
device-to-host copy of the result.  Plotting is not implemented.
"""
import numpy as np
import torch

from . import ops
from .empirical import Empirical

_VALUE_DTYPES = (torch.float32, torch.float64, torch.int32, torch.int64)


def _no_plot(plot):
    if plot:
        raise NotImplementedError('pyprob_b200.diagnostics does not plot; plot result[name]["rhat"] or '
                                  '["autocorrelation"] yourself, or use the reference pyprob.diagnostics plots')


def _declared_chains(dist):
    for md in reversed(dist.metadata):
        if md.get('op') == 'posterior' and 'num_chains' in md:
            return int(md['num_chains'])
    return 1


def _columns(dist, length):
    """The first `length` values of an Empirical as a [length, V] CUDA tensor (a view when the values allow one)."""
    v = dist.values
    if not torch.is_tensor(v) or not v.is_cuda:
        raise TypeError('diagnostics need the CUDA tensor values of a posterior (a map_func result), got {}'.format(
            type(v).__name__ if not torch.is_tensor(v) else v.device))
    if v.dtype not in _VALUE_DTYPES:
        raise TypeError('diagnostics read float32, float64, int32 or int64 values, got {}'.format(v.dtype))
    return v[:length].reshape(length, -1)


def _chains(trace_dists, num_chains):
    """-> x [S, C, V] in the values' dtype; for one Empirical a view of its values."""
    if isinstance(trace_dists, Empirical):
        C = _declared_chains(trace_dists) if num_chains is None else int(num_chains)
        N = len(trace_dists)
        if C < 1:
            raise ValueError('num_chains must be positive, got {}'.format(C))
        if N == 0 or N % C:
            raise ValueError('the Empirical holds {} values, which is not a positive multiple of num_chains = {}; '
                             'a slice must start at a multiple of num_chains, e.g. post[burn_in * num_chains:]'.format(
                                 N, C))
        v = _columns(trace_dists, N)
        return v.reshape(N // C, C, v.size(1))
    if not isinstance(trace_dists, (list, tuple)) or not trace_dists or \
            not all(isinstance(d, Empirical) for d in trace_dists):
        raise TypeError('expecting an Empirical from posterior(..., num_chains=C) or a list of Empiricals, '
                        'one chain each')
    if any(_declared_chains(d) != 1 for d in trace_dists):
        raise ValueError('in a list every Empirical is one chain; pass a posterior of several chains on its own')
    if num_chains is not None and int(num_chains) != len(trace_dists):
        raise ValueError('num_chains = {} but the list holds {} chains'.format(num_chains, len(trace_dists)))
    S = min(len(d) for d in trace_dists)      # reference diagnostics.py:804-807
    if S == 0:
        raise ValueError('an Empirical of the list is empty')
    cols = [_columns(d, S) for d in trace_dists]
    if len({c.size(1) for c in cols}) != 1:
        raise ValueError('the chains have different numbers of variables: {}'.format([c.size(1) for c in cols]))
    if len({c.dtype for c in cols}) != 1:
        cols = [c.to(torch.float64) for c in cols]
    return torch.stack(cols, dim=1)


def _names(names, V):
    if names is None:
        return list(range(V))
    names = [names] if isinstance(names, str) else list(names)
    if len(names) != V:
        raise ValueError('names has {} entries but the values have {} variables (columns)'.format(len(names), V))
    return names


def _ints(a, what):
    arr = np.asarray(a)
    out = arr.astype(np.int64).reshape(-1)
    if arr.size == 0 or arr.ndim > 1 or not np.array_equal(out, arr.reshape(-1)):
        raise ValueError('{} must be a non-empty 1-d sequence of integers, got {!r}'.format(what, a))
    return out


def _kernel_input(x):
    # the kernels read fp32 or fp64; integer values are exact in fp64 up to 2^53
    return x if x.dtype in (torch.float32, torch.float64) else x.to(torch.float64)


def gelman_rubin(trace_dists, names=None, iters=None, num_chains=None, plot=False):
    """Gelman-Rubin R-hat of every variable against the number of iterations (reference diagnostics.py:784-873).

    trace_dists: one Empirical of C >= 2 chains in step-major order, or a list of Empiricals of one chain each.
    iters: prefix lengths (any order, >= 1; a value above the chain length S means S); default
    ``np.unique(np.logspace(0, np.log10(S)).astype(int))``.
    -> (iters, {name: {'values': CUDA view [C, S], 'rhat': numpy fp64 [len(iters)]}}).  R-hat is NaN for a one-step
    prefix, and inf (NaN) where every chain is constant (and all chains agree), as numpy gives."""
    _no_plot(plot)
    x = _chains(trace_dists, num_chains)
    S, C, V = x.shape
    keys = _names(names, V)
    if C < 2:
        raise ValueError('Gelman-Rubin diagnostic requires at least two chains')
    if iters is None:
        iters = np.unique(np.logspace(0, np.log10(S)).astype(int))
    it = _ints(iters, 'iters')
    if (it < 1).any():
        raise ValueError('iters must be >= 1, got {}'.format(it[it < 1]))
    rhat = ops.diag_rhat(_kernel_input(x), it).cpu().numpy()
    return iters, {k: {'values': x[:, :, i].t(), 'rhat': rhat[i]} for i, k in enumerate(keys)}


def autocorrelation(trace_dist, names=None, lags=None, num_chains=None, plot=False):
    """Autocorrelation of every chain of every variable at the given lags (reference diagnostics.py:714-781).

    trace_dist: one Empirical of C chains in step-major order (C = 1: the reference's single chain).
    lags: integers in [0, S]; default ``np.unique(np.logspace(0, np.log10(S / 2)).astype(int))``.
    -> (lags, {name: {'values': CUDA view [C, S], 'autocorrelation': numpy fp64 [C, len(lags)], or [len(lags)] for one
    chain}}), with sum_{i < S - lag} (x_i - mu)(x_{i+lag} - mu) / (1e-8 + sum_i (x_i - mu)^2) and mu the chain's mean."""
    _no_plot(plot)
    if not isinstance(trace_dist, Empirical):
        raise TypeError('expecting an Empirical (from posterior(..., num_chains=C))')
    x = _chains(trace_dist, num_chains)
    S, C, V = x.shape
    keys = _names(names, V)
    if lags is None:
        lags = np.unique(np.logspace(0, np.log10(S / 2)).astype(int))
    lg = _ints(lags, 'lags')
    if ((lg < 0) | (lg > S)).any():
        raise ValueError('lags must lie in [0, {}] (the chain length), got {}'.format(S, lg[(lg < 0) | (lg > S)]))
    ac = ops.diag_autocorr(_kernel_input(x), lg).cpu().numpy()
    return lags, {k: {'values': x[:, :, i].t(), 'autocorrelation': ac[i] if C > 1 else ac[i, 0]}
                  for i, k in enumerate(keys)}
