"""Generate tests/golden/event_golden.npz by running the UNMODIFIED reference (pyprob v1.5.0) on the CPU: observations
with an event shape.

    python tests/golden/make_event_golden.py

Needs the reference checkout on sys.path and the import stubs in oracle/ref_stubs, as make_golden.py does.
  case<i>/*   one model per (family, broadcasting form): an observe of a vector / matrix value whose parameters are
              scalars, shared events of the value's shape, rows that broadcast against it ([4, 1] against [4, 3]), or a
              value that is a scalar or [1, D] against [D] parameters; Normal cases also carry a latent z ~ Normal(0, 1)
              fixed through `observe` that shifts the loc.  Recorded: the family, the parameters (p0 .. p3, with their
              shapes), the value, z (or NaN) and the reference's trace.log_prob_observed of one posterior trace.
  lstm/*, ff/*  InferenceNetworkLSTM / InferenceNetworkFeedForward _loss + backward on reference traces of a model with a
              D = 8 observable, in the layout of network_golden.npz / ff_golden.npz.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden  # noqa: E402  (puts the reference and its stubs on sys.path)
import numpy as np  # noqa: E402
import torch  # noqa: E402

import pyprob  # noqa: E402  (the reference)
from pyprob import InferenceNetwork, Model  # noqa: E402
from pyprob.distributions import (Bernoulli, Beta, Binomial, Exponential, Gamma, LogNormal, Normal,  # noqa: E402
                                  Poisson, Uniform, VonMises, Weibull)
from pyprob.nn.dataset import Batch, OnlineDataset  # noqa: E402
from pyprob.util import TraceMode  # noqa: E402

CTORS = {'Normal': Normal, 'Uniform': Uniform, 'Poisson': Poisson, 'Bernoulli': Bernoulli, 'Exponential': Exponential,
         'Gamma': Gamma, 'LogNormal': LogNormal, 'Weibull': Weibull, 'Beta': Beta,
         'Binomial': lambda n, p: Binomial(total_count=n, probs=p), 'VonMises': VonMises}


def _draw(family, shape, g):
    """(value, [parameters]) of `shape` inside the support, as float32 tensors."""
    def u(lo=0.0, hi=1.0):
        return lo + (hi - lo) * torch.rand(shape, generator=g)
    if family == 'Normal':
        return torch.randn(shape, generator=g), [u(-1, 1), u(0.5, 2)]
    if family == 'Uniform':
        lo = u(-2, -1)
        return lo + 0.5 * u(), [lo, lo + u(1, 2)]
    if family == 'Poisson':
        rate = u(0.5, 20)
        return torch.poisson(rate, generator=g), [rate]
    if family == 'Bernoulli':
        return (u() < 0.5).float(), [u(0.05, 0.95)]
    if family == 'Exponential':
        return u(0, 3), [u(0.5, 2)]
    if family == 'Gamma':
        return u(0.05, 3), [u(0.5, 4), u(0.5, 2)]
    if family == 'LogNormal':
        return u(0.05, 3), [u(-0.5, 0.5), u(0.5, 1.5)]
    if family == 'Weibull':
        return u(0.05, 3), [u(0.5, 2), u(0.5, 3)]
    if family == 'Beta':
        return u(-0.9, 1.9), [u(0.5, 3), u(0.5, 3), torch.full(shape, -1.0), torch.full(shape, 2.0)]
    if family == 'Binomial':
        n = torch.floor(u(2, 30))
        return torch.minimum(torch.floor(u() * (n + 1)), n), [n, u(0.05, 0.95)]
    return u(-3, 3), [u(-3, 3), u(0.1, 6)]


FORMS = ['scalar_params', 'event_params', 'row_params', 'scalar_value', 'one_by_d_value']


def cases(seed=77):
    """(family, form, parameters (floats or tensors), value) for every family and broadcasting form."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for family in CTORS:
        for form in FORMS:
            shape = (4, 3) if form == 'row_params' else (7,)
            v, ps = _draw(family, shape, g)
            if form == 'scalar_params':
                ps = [float(p.reshape(-1)[0]) for p in ps]
                if family == 'Binomial':
                    v = torch.minimum(v, torch.tensor(ps[0]))
            elif form == 'row_params':
                ps = [p[:, :1].contiguous() for p in ps]
                if family == 'Binomial':
                    v = torch.minimum(v, ps[0].expand(4, 3))
            elif form == 'scalar_value':
                v = v.reshape(-1)[:1].reshape(())
                if family == 'Binomial':
                    v = torch.minimum(v, ps[0].min())
                if family == 'Uniform':
                    v = ps[0].max() + 0.01 * (ps[1].min() - ps[0].max())
            elif form == 'one_by_d_value':
                v = v.reshape(1, -1)
            if family == 'Beta' and form != 'scalar_params':
                ps[2], ps[3] = -1.0, 2.0
            if family == 'Uniform' and form != 'scalar_value':   # inside [low, high) of every element it meets
                lo, hi = (torch.as_tensor(q) for q in ps)
                v = (lo + 0.5 * (hi - lo) * torch.rand(v.shape, generator=g)).reshape(v.shape)
            out.append((family, form, ps, v))
    return out


class EventModel(Model):
    def __init__(self, family, params, latent):
        super().__init__('event ' + family)
        self.family, self.params, self.latent = family, params, latent

    def forward(self):
        ps = list(self.params)
        if self.latent:
            z = pyprob.sample(Normal(0.0, 1.0), name='z')
            ps[0] = ps[0] + z
        pyprob.observe(CTORS[self.family](*ps), name='x')
        return 0


def log_prob_observed(model, observe):
    with make_golden._silence():
        traces = model._traces(1, trace_mode=TraceMode.POSTERIOR, observe=observe, silent=True)
    tr = traces[0] if isinstance(traces, (list, tuple)) else traces.get_values()[0]
    return float(tr.log_prob_observed)


def case_fixture():
    fx = {}
    for i, (family, form, ps, v) in enumerate(cases()):
        latent = family == 'Normal'
        z = 0.37 if latent else float('nan')
        observe = {'x': v}
        if latent:
            observe['z'] = torch.tensor(z)
        p = 'case{}/'.format(i)
        fx[p + 'family'] = np.asarray(family)
        fx[p + 'form'] = np.asarray(form)
        for k, q in enumerate(ps):
            fx[p + 'p{}'.format(k)] = np.asarray(q.numpy() if torch.is_tensor(q) else q, np.float32)
        fx[p + 'value'] = v.numpy().astype(np.float32)
        fx[p + 'z'] = np.asarray(z, np.float64)
        fx[p + 'lpo'] = np.asarray(log_prob_observed(EventModel(family, ps, latent), observe), np.float64)
    fx['num_cases'] = np.asarray(len(cases()))
    return fx


class VectorObs(Model):
    """Two latents and a D = 8 observable whose loc is a line through them."""

    def __init__(self):
        super().__init__('vector observable')

    def forward(self):
        z = pyprob.sample(Normal(0.0, 1.0))
        u = pyprob.sample(Uniform(0.0, 2.0))
        pyprob.observe(Normal(z * torch.linspace(0, 1, 8) + u, 0.3), name='x')
        return z


EMB = {'x': {'dim': 16, 'depth': 2}}


def ff_fixture(K=4, batch=32, seed=33):
    sys.path.insert(0, make_golden.ROOT)
    from oracle import network as onet
    pyprob.seed(seed)
    model = VectorObs()
    with make_golden._silence():
        model.learn_inference_network(num_traces=128, batch_size=batch, inference_network=InferenceNetwork.FEEDFORWARD,
                                      observe_embeddings=EMB, proposal_mixture_components=K)
    net = model._inference_network
    ds = OnlineDataset(model)
    traces = [ds[i] for i in range(batch)]
    b = Batch(traces)
    with make_golden._silence():
        net._polymorph(b)
    net.zero_grad()
    success, loss = net._loss(b)
    assert success
    loss.backward()
    names = list(EMB)
    fx = {'ff/loss': np.asarray(float(loss), dtype=np.float64), 'ff/observe_names': np.asarray(names),
          'ff/observe_in_dims': np.asarray([8]), 'ff/dims': np.asarray([K, batch])}
    for k, v in net.state_dict().items():
        fx['ff/param/' + k] = v.detach().numpy()
    for k, p in net.named_parameters():
        fx['ff/grad/' + k] = (p.grad if p.grad is not None else torch.zeros_like(p)).detach().numpy()
    fx['ff/address_order'] = np.asarray(list(net._layers_proposal.keys()))
    for s, sub in enumerate(b.sub_batches):
        sb = onet.sub_batch_from_traces(sub, names)
        p = 'ff/sub{}/'.format(s)
        for k in ('addresses', 'families', 'num_categories'):
            fx[p + k] = np.asarray(sb[k])
        for k in ('values', 'prior0', 'prior1', 'obs'):
            fx[p + k] = sb[k].numpy()
    fx['ff/num_sub'] = np.asarray(len(b.sub_batches))
    return fx


def main():
    pyprob.set_verbosity(0)
    fx = case_fixture()
    fx.update(make_golden.network_fixture(VectorObs(), EMB, lstm_dim=32, K=4, batch_size=32, train_traces=128, seed=31,
                                          tag='lstm'))
    fx.update(ff_fixture())
    np.savez_compressed(os.path.join(HERE, 'event_golden.npz'), **fx)
    print('wrote event_golden.npz with', len(fx), 'arrays')


if __name__ == '__main__':
    main()
