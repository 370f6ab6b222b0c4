"""Oracle: the reference's MCMC diagnostics in numpy fp64 (TEST INFRASTRUCTURE ONLY).

Restates pyprob/diagnostics.py:788-802 (Gelman-Rubin R-hat of every prefix) and :720-736 (autocorrelation of one chain)
over arrays of values instead of Empiricals of traces, vectorised over the chains.
"""
import warnings

import numpy as np

EPSILON = 1e-8       # pyprob/util.py:34


def r_hat(values):
    """values [m, n]: m chains of n steps."""
    values = np.asarray(values, dtype=np.float64)
    m, n = values.shape
    if m < 2:
        raise ValueError('Gelman-Rubin diagnostic requires at least two chains')
    with np.errstate(divide='ignore', invalid='ignore'), warnings.catch_warnings():
        warnings.simplefilter('ignore', RuntimeWarning)   # numpy's NaN / inf are the results
        b = n * np.var(np.mean(values, axis=1), axis=0, ddof=1)        # between-chain variance
        w = np.mean(np.var(values, axis=1, ddof=1), axis=0)           # within-chain variance
        v_hat = ((n - 1) / n) * w + b / n
        return np.sqrt(v_hat / w)


def r_hats(values, iters):
    """R-hat of the prefix values[:, :iter] for every iter (an iter above n takes all n steps)."""
    values = np.asarray(values, dtype=np.float64)
    return np.array([r_hat(values[:, :int(it)]) for it in iters], dtype=np.float64)


def autocorrelation(values, lags):
    """values [S] or [C, S] -> [len(lags)] or [C, len(lags)]: sum_{i < S - lag} d_i d_{i+lag} / (1e-8 + sum_i d_i^2)
    with d = values - the chain's mean; lags in [0, S]."""
    x = np.asarray(values, dtype=np.float64)
    S = x.shape[-1]
    d = x - x.mean(axis=-1, keepdims=True)
    den = EPSILON + (d * d).sum(axis=-1)
    out = []
    for lag in lags:
        lag = int(lag)
        if not 0 <= lag <= S:
            raise ValueError('lag {} outside [0, {}]'.format(lag, S))
        out.append((d[..., :S - lag] * d[..., lag:]).sum(axis=-1) / den)
    return np.stack(out, axis=-1)
