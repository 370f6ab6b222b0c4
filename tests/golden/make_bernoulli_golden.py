"""Generate tests/golden/bernoulli_golden.npz by running the UNMODIFIED reference (pyprob v1.5.0) on the CPU.

    python tests/golden/make_bernoulli_golden.py

Needs the reference checkout on sys.path and the import stubs in oracle/ref_stubs, as make_golden.py does.
  scoring/*   Bernoulli.log_prob over per-particle probs, probs of 0 and 1 included, values 0 and 1.
  bern/*      InferenceNetworkLSTM._loss + backward for a model that mixes Bernoulli with Normal and Categorical
              (two trace types through control flow on a Bernoulli value; prior probs are 1-element tensors, so the
              reference computes the per-row loss), same layout as network_golden.npz.
  quirk/*     the same kind of model with Python-scalar prior probs: the reference's loss of that batch, whose
              Bernoulli terms are the pairwise -sum_b sum_b' log q_b(v_b') (see DESIGN.md section 8).
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the reference and its stubs on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pyprob  # noqa: E402  (the reference)
from pyprob import Model  # noqa: E402
from pyprob.distributions import Bernoulli, Categorical, Normal  # noqa: E402


def scoring_fixture(seed=4321, n=257):
    g = torch.Generator().manual_seed(seed)
    probs = torch.rand(n, generator=g)
    probs[::17] = 0.0
    probs[5::17] = 1.0
    probs[9::17] = 1e-9        # inside the clamp
    v = (torch.rand(n, generator=g) < 0.5).float()
    v[::34] = 1.0              # value 1 at probs 0 and value 0 at probs 1: log(eps)
    v[5::34] = 0.0
    return {'scoring/value': v.numpy(), 'scoring/probs': probs.numpy(),
            'scoring/lp': Bernoulli(probs).log_prob(v).detach().numpy()}


class BernoulliMixed(Model):
    """Bernoulli at t = 0 and as the previous site of a Normal; two trace types through the first Bernoulli value."""

    def __init__(self, scalar_probs=False):
        super().__init__('bernoulli mixed')
        self._p = (lambda p: p) if scalar_probs else (lambda p: torch.tensor([p]))

    def forward(self):
        b = pyprob.sample(Bernoulli(self._p(0.4)))
        if int(b) == 1:
            k = pyprob.sample(Categorical([0.2, 0.3, 0.5]))
            m = float(k) * 0.5
        else:
            m = float(pyprob.sample(Normal(0.5, 1.0)))
        c = pyprob.sample(Bernoulli(self._p(0.7)))
        mu = pyprob.sample(Normal(m + 2.0 * float(c) - 1.0, 1.0))
        pyprob.observe(Normal(mu, 0.5), name='y0')
        pyprob.observe(Normal(float(b), 0.3), name='y1')
        return mu


def main():
    pyprob.set_verbosity(0)
    fx = scoring_fixture()
    fx.update(make_golden.network_fixture(BernoulliMixed(), {'y0': {'dim': 8, 'depth': 2}, 'y1': {'dim': 4, 'depth': 1}},
                                          lstm_dim=32, K=5, batch_size=24, train_traces=96, seed=21, tag='bern'))
    fx.update(make_golden.network_fixture(BernoulliMixed(scalar_probs=True), {'y0': {'dim': 8, 'depth': 2},
                                                                              'y1': {'dim': 4, 'depth': 1}},
                                          lstm_dim=32, K=5, batch_size=24, train_traces=96, seed=22, tag='quirk'))
    np.savez_compressed(os.path.join(HERE, 'bernoulli_golden.npz'), **fx)
    print('wrote bernoulli_golden.npz with', len(fx), 'arrays')


if __name__ == '__main__':
    main()
