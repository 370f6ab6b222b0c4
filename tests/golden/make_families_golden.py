"""Generate tests/golden/families_golden.npz by running the UNMODIFIED reference (pyprob v1.5.0) on the CPU.

    python tests/golden/make_families_golden.py

Needs the reference checkout on sys.path and the import stubs in oracle/ref_stubs, as make_golden.py does.
For each family, every row of a value / parameter grid holds the reference's log_prob, mean and variance:
  <family>/value, <family>/<parameter>...   the grid (fp32), one row per element
  <family>/lp                               Distribution.log_prob(value); NaN where the reference raises (a value outside
                                            the support or an invalid parameter: torch validates its arguments)
  <family>/mean, <family>/variance          Distribution.mean / .variance; NaN where the constructor raises
The grids include the edges: Gamma and Beta with concentrations below 1 at 0 and near 0, Beta at u = 0 and u = 1 with
and without low / high, Binomial at k = 0 and k = n with p near 0 and 1 and from logits, VonMises at kappa = 1e-3 and
where exp(kappa) overflows fp32, Exponential at 0, LogNormal and Weibull near 0.
"""
import itertools
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402,F401  (puts the reference and its stubs on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pyprob  # noqa: E402  (the reference)
from pyprob.distributions import Beta, Binomial, Exponential, Gamma, LogNormal, VonMises, Weibull  # noqa: E402


def _grid(*axes):
    rows = np.array(list(itertools.product(*axes)), dtype=np.float64).astype(np.float32)
    return [rows[:, j] for j in range(rows.shape[1])]


def _scalar(make, args, what):
    try:
        d = make(*[torch.tensor(float(a)) for a in args[1:]])
        if what == 'lp':
            return float(d.log_prob(torch.tensor(float(args[0]))))
        return float(getattr(d, what))
    except ValueError:        # torch argument validation: invalid parameter or value outside the support
        return float('nan')


def family(name, make, names, columns):
    """Reference log_prob / mean / variance, row by row (each row is its own reference distribution)."""
    out = {'{}/{}'.format(name, k): c for k, c in zip(names, columns)}
    rows = list(zip(*columns))
    for what in ('lp', 'mean', 'variance'):
        out['{}/{}'.format(name, what)] = np.array([_scalar(make, r, what) for r in rows], dtype=np.float32)
    return out


def main():
    pyprob.set_verbosity(0)
    fx = {}
    fx.update(family('exponential', lambda r: Exponential(r), ['value', 'rate'],
                     _grid([0.0, 1e-30, 1e-6, 0.25, 1.0, 5.0, 100.0, -1e-6, -1.0], [1e-3, 0.5, 1.5, 4.0, 100.0, 0.0, -1.0])))
    fx.update(family('gamma', lambda c, r: Gamma(c, r), ['value', 'concentration', 'rate'],
                     _grid([0.0, 1e-30, 1e-8, 1e-3, 0.4167, 1.0, 3.0, 50.0, -0.5], [0.05, 0.5, 1.0, 2.7, 100.0, 0.0, -1.0],
                           [0.1, 1.2, 7.0, 0.0])))
    fx.update(family('lognormal', lambda m, s: LogNormal(m, s), ['value', 'loc', 'scale'],
                     _grid([1e-30, 1e-10, 1e-3, 0.5, 1.682, 10.0, 1e4, 0.0, -1.0], [-2.0, 0.0, 0.5, 3.0],
                           [0.01, 0.2, 1.0, 3.0, 0.0])))
    fx.update(family('weibull', lambda s, k: Weibull(s, k), ['value', 'scale', 'concentration'],
                     _grid([1e-30, 1e-10, 1e-3, 0.5, 2.2, 10.0, 100.0, 0.0, -1.0], [0.1, 1.1, 5.0, 0.0],
                           [0.5, 1.1, 3.0, 10.0, 0.0])))
    fx.update(family('beta', lambda a, b: Beta(a, b), ['value', 'concentration1', 'concentration0'],
                     _grid([0.0, 1e-30, 1e-6, 0.285714, 0.5, 0.999999, 1.0, -0.1, 1.1], [0.1, 0.5, 1.0, 2.0, 50.0, 0.0],
                           [0.1, 1.0, 5.0, 50.0])))
    v, a, b = _grid([-2.0, -1.9999, -1.0, 0.8, 3.0, 4.9999, 5.0, -2.5, 5.5], [0.1, 0.5, 2.0], [0.1, 1.0, 5.0])
    lo, hi = np.full_like(v, -2.0), np.full_like(v, 5.0)
    fx.update(family('beta_lowhigh', lambda a, b, lo, hi: Beta(a, b, low=lo, high=hi),
                     ['value', 'concentration1', 'concentration0', 'low', 'high'], [v, a, b, lo, hi]))
    cols = [[], [], []]
    for n in (0.0, 1.0, 10.0, 1000.0, 2.5, -1.0):
        for p in (0.0, 1e-9, 0.01, 0.2, 0.5, 0.97, 1.0 - 1e-7, 1.0, 1.5):
            for k in sorted({0.0, 1.0, 2.0, n - 1, n, n + 1, 0.5, -1.0}):
                for c, x in zip(cols, (k, n, p)):
                    c.append(x)
    cols = [np.array(c, dtype=np.float32) for c in cols]
    fx.update(family('binomial', lambda n, p: Binomial(total_count=n, probs=p), ['value', 'total_count', 'probs'], cols))
    cols = [[], [], []]
    for n in (1.0, 10.0, 1000.0):
        for lg in (-30.0, -5.0, -0.3, 0.0, 2.0, 12.0, 30.0):
            for k in sorted({0.0, 1.0, n - 1, n}):
                for c, x in zip(cols, (k, n, lg)):
                    c.append(x)
    cols = [np.array(c, dtype=np.float32) for c in cols]
    fx.update(family('binomial_logits', lambda n, lg: Binomial(total_count=n, logits=lg),
                     ['value', 'total_count', 'logits'], cols))
    fx.update(family('von_mises', lambda m, k: VonMises(m, k), ['value', 'loc', 'concentration'],
                     _grid([-math.pi, -1.0, 0.0, 1.0, 3.1415, 10.0, 100.0], [0.0, 3.1415, -2.0],
                           [1e-3, 0.5, 1.1, 3.74, 3.76, 50.0, 100.0, 1e4, 0.0])))
    np.savez_compressed(os.path.join(HERE, 'families_golden.npz'), **fx)
    print('wrote families_golden.npz with', len(fx), 'arrays')


if __name__ == '__main__':
    main()
