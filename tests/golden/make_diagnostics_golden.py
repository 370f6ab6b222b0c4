"""Generate tests/golden/diagnostics_golden.npz by running the UNMODIFIED reference (pyprob v1.5.0) on the CPU.

    python tests/golden/make_diagnostics_golden.py

Needs the reference checkout on sys.path and the import stubs in oracle/ref_stubs, as make_golden.py does.
For two models (GUM with a named `mu`; a two-variable model with named `mu ~ Normal`, `s ~ Uniform(0.5, 3)` observed
through Normal(mu, s)) under LMH and RMH, runs four seeded chains of STEPS steps with the reference's
Model.posterior, then the reference's pyprob.diagnostics.gelman_rubin (n_most_frequent=None) and autocorrelation (on
every chain) with their default iters / lags and with custom ones that hold iter 1, iter S, lag 0 and lag S.  Stores,
per case <model>_<engine>:
  <case>/values/<name>          [4, S] the values the reference extracted, chain by chain
  <case>/rhat/<name>            default iters       <case>/iters
  <case>/rhat_custom/<name>     custom iters        <case>/iters_custom
  <case>/acf/<name>             [4, len(lags)]      <case>/lags
  <case>/acf_custom/<name>      [4, len(lags)]      <case>/lags_custom
"""
import math
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402,F401  (puts the reference and its stubs on sys.path)
import numpy as np  # noqa: E402

import pyprob  # noqa: E402  (the reference)
from pyprob import InferenceEngine, Model, diagnostics, util  # noqa: E402
from pyprob.distributions import Normal, Uniform  # noqa: E402

STEPS = 300
CHAINS = 4


class GUM(Model):
    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)), name='mu')
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


class TwoVariables(Model):
    def forward(self):
        mu = pyprob.sample(Normal(0, 3), name='mu')
        s = pyprob.sample(Uniform(0.5, 3), name='s')
        likelihood = Normal(mu, s)
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        pyprob.observe(likelihood, name='obs2')
        return mu


MODELS = [('gum', GUM, {'obs0': 8, 'obs1': 9}, ['mu']),
          ('two', TwoVariables, {'obs0': 1.5, 'obs1': -0.5, 'obs2': 2.5}, ['mu', 's'])]
ENGINES = [('lmh', InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS),
           ('rmh', InferenceEngine.RANDOM_WALK_METROPOLIS_HASTINGS)]
ITERS_CUSTOM = np.array([STEPS, 7, 1, 150, 2, 40])
LAGS_CUSTOM = np.array([0, STEPS, 1, 3, 299, 100, 17])


def main():
    out = {}
    for mi, (mname, make, observe, names) in enumerate(MODELS):
        for ei, (ename, engine) in enumerate(ENGINES):
            case = '{}_{}'.format(mname, ename)
            model = make()
            chains = []
            for c in range(CHAINS):
                util.seed(1000 + 100 * mi + 10 * ei + c)
                chains.append(model.posterior(num_traces=STEPS, inference_engine=engine, observe=observe))
            iters, vv = diagnostics.gelman_rubin(chains, names=names, n_most_frequent=None)
            _, vv_custom = diagnostics.gelman_rubin(chains, names=names, iters=ITERS_CUSTOM, n_most_frequent=None)
            out[case + '/iters'] = np.asarray(iters)
            out[case + '/iters_custom'] = ITERS_CUSTOM
            by_name = {v['variable'].name: v for v in vv.values()}
            by_name_custom = {v['variable'].name: v for v in vv_custom.values()}
            acf, acf_custom, lags = {n: [] for n in names}, {n: [] for n in names}, None
            for chain in chains:
                lags, av = diagnostics.autocorrelation(chain, names=names)
                _, av_custom = diagnostics.autocorrelation(chain, names=names, lags=LAGS_CUSTOM)
                for v in av.values():
                    acf[v['variable'].name].append(v['autocorrelation'])
                for v in av_custom.values():
                    acf_custom[v['variable'].name].append(v['autocorrelation'])
            out[case + '/lags'] = np.asarray(lags)
            out[case + '/lags_custom'] = LAGS_CUSTOM
            for n in names:
                out['{}/values/{}'.format(case, n)] = np.asarray(by_name[n]['values'], dtype=np.float64)
                out['{}/rhat/{}'.format(case, n)] = np.asarray(by_name[n]['rhat'], dtype=np.float64)
                out['{}/rhat_custom/{}'.format(case, n)] = np.asarray(by_name_custom[n]['rhat'], dtype=np.float64)
                out['{}/acf/{}'.format(case, n)] = np.asarray(acf[n], dtype=np.float64)
                out['{}/acf_custom/{}'.format(case, n)] = np.asarray(acf_custom[n], dtype=np.float64)
    np.savez_compressed(os.path.join(HERE, 'diagnostics_golden.npz'), **out)
    print('wrote {} arrays'.format(len(out)))


if __name__ == '__main__':
    main()
