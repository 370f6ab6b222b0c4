"""Generate tests/golden/mcmc_golden.npz by running the UNMODIFIED reference (pyprob v1.5.0) on the CPU.

    python tests/golden/make_mcmc_golden.py

Needs the reference checkout on sys.path and the import stubs in oracle/ref_stubs, as make_golden.py does.
Runs the reference's LMH and RMH (seeded) on four models: GUM, a Marsaglia-style rejection loop, Branching and a Uniform
prior with a Normal likelihood.  The step loop below is model.py:141-170 with the candidate generation, the acceptance
ratio and the decision left to the reference; it only records, for every step:
  step/*   model, engine, |controlled| and log_prob_observed of the current and the candidate trace, the reference's
           _metropolis_hastings_site_transition_log_prob (NaN when the candidate did not reach the site), the log alpha
           of model.py:151-162, and at the chosen address: its family, the candidate's prior parameters (p0, p1) and
           the current / candidate value and log_prob
  site/*   every controlled site of both traces: step, trace (0 current, 1 candidate), address id, value, log_prob,
           reused
"""
import math
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402,F401  (puts the reference and its stubs on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pyprob  # noqa: E402  (the reference)
from pyprob import InferenceEngine, Model, state, util  # noqa: E402
from pyprob.distributions import Normal, Poisson, Uniform  # noqa: E402
from pyprob.util import TraceMode  # noqa: E402

STEPS = 60
FAMILIES = {'Normal': 0, 'Uniform': 1, 'Poisson': 2}


class GUM(Model):
    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


class Marsaglia(Model):
    def marsaglia(self, mean, stddev):
        uniform = Uniform(-1, 1)
        s = 1
        while float(s) >= 1:
            x = pyprob.sample(uniform)
            y = pyprob.sample(uniform)
            s = x * x + y * y
        return mean + stddev * (x * torch.sqrt(-2 * torch.log(s) / s))

    def forward(self):
        mu = self.marsaglia(1, math.sqrt(5))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


def _fib(n):
    if n < 2:
        return 1
    a = fib = 1
    for _ in range(n - 2):
        a, fib = fib, a + fib
    return fib


class Branching(Model):
    def forward(self):
        count_prior = Poisson(4)
        r = pyprob.sample(count_prior)
        if 4 < float(r):
            lam = 6
        else:
            lam = 1 + _fib(3 * int(r)) + pyprob.sample(count_prior)
        pyprob.observe(Poisson(lam), name='obs')
        return r


class UniformPrior(Model):
    def forward(self):
        x = pyprob.sample(Uniform(0, 10))
        pyprob.observe(Normal(x, 1.0), name='obs')
        return x


MODELS = [(GUM, {'obs0': 8, 'obs1': 9}), (Marsaglia, {'obs0': 8, 'obs1': 9}), (Branching, {'obs': 6}),
          (UniformPrior, {'obs': 7.0})]
ENGINES = [InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS, InferenceEngine.RANDOM_WALK_METROPOLIS_HASTINGS]


def _params(d):
    if isinstance(d, Normal):
        return float(d.mean), float(d.stddev)
    if isinstance(d, Uniform):
        return float(d.low), float(d.high)
    return float('nan'), float('nan')


def main():
    steps, sites, addresses = {k: [] for k in ('model', 'engine', 'cur_n', 'cand_n', 'cur_lpo', 'cand_lpo', 'transition',
                                               'log_alpha', 'family', 'p0', 'p1', 'x_old', 'lp_old', 'x_new',
                                               'lp_new')}, [], {}
    for mi, (make, observe) in enumerate(MODELS):
        for ei, engine in enumerate(ENGINES):
            util.seed(100 + 10 * mi + ei)
            model = make()
            cur = next(model._trace_generator(trace_mode=TraceMode.POSTERIOR, inference_engine=engine, observe=observe))
            for _ in range(STEPS):
                cand = next(model._trace_generator(trace_mode=TraceMode.POSTERIOR, inference_engine=engine,
                                                   metropolis_hastings_trace=cur, observe=observe))
                # model.py:151-162, verbatim
                log_acceptance_ratio = math.log(cur.length_controlled) - math.log(cand.length_controlled) + \
                    cand.log_prob_observed - cur.log_prob_observed
                for variable in cand.variables_controlled:
                    if variable.reused:
                        log_acceptance_ratio += torch.sum(variable.log_prob)
                        log_acceptance_ratio -= torch.sum(cur.variables_dict_address[variable.address].log_prob)
                t = state._metropolis_hastings_site_transition_log_prob
                if t is not None:
                    log_acceptance_ratio += torch.sum(t)
                address = state._metropolis_hastings_site_address
                new = cand.variables_dict_address.get(address)
                old = cur.variables_dict_address[address]
                s = len(steps['model'])
                for k, v in (('model', mi), ('engine', ei), ('cur_n', cur.length_controlled),
                             ('cand_n', cand.length_controlled), ('cur_lpo', float(cur.log_prob_observed)),
                             ('cand_lpo', float(cand.log_prob_observed)),
                             ('transition', float('nan') if t is None else float(t)),
                             ('log_alpha', float(log_acceptance_ratio)),
                             ('family', FAMILIES[old.distribution.name]),
                             ('p0', _params(new.distribution)[0] if new is not None else float('nan')),
                             ('p1', _params(new.distribution)[1] if new is not None else float('nan')),
                             ('x_old', float(old.value)), ('lp_old', float(old.log_prob)),
                             ('x_new', float(new.value) if new is not None else float('nan')),
                             ('lp_new', float(new.log_prob) if new is not None else float('nan'))):
                    steps[k].append(v)
                for which, trace in ((0, cur), (1, cand)):
                    for v in trace.variables_controlled:
                        aid = addresses.setdefault(v.address, len(addresses))
                        sites.append((s, which, aid, float(v.value), float(v.log_prob), bool(v.reused)))
                if math.log(random.random()) < float(log_acceptance_ratio):   # model.py:165-167
                    cur = cand
    out = {'step/' + k: np.asarray(v) for k, v in steps.items()}
    sites = np.array(sites, dtype=np.float64)
    for j, k in enumerate(('step', 'trace', 'address', 'value', 'log_prob', 'reused')):
        out['site/' + k] = sites[:, j]
    np.savez_compressed(os.path.join(HERE, 'mcmc_golden.npz'), **out)
    print('wrote {} steps, {} sites, {} addresses'.format(len(steps['model']), len(sites), len(addresses)))


if __name__ == '__main__':
    main()
