"""Generate tests/golden/ff_golden.npz by running the UNMODIFIED reference (pyprob v1.5.0) on the CPU:
InferenceNetworkFeedForward (pyprob/nn/inference_network_feedforward.py).

    python tests/golden/make_ff_golden.py

Needs the reference checkout on sys.path and the import stubs in oracle/ref_stubs, as make_golden.py does.
  ff/*        _loss + backward for a model with all five proposal families (Normal, Uniform, Poisson, Categorical,
              Bernoulli), two trace types through control flow on a Bernoulli value, observables of depth 2 and 1; the
              layout of network_golden.npz (params, grads, sub-batches).  The Bernoulli priors take 1-element tensors,
              so the reference computes the per-row loss.
  infer/*     _infer_init + _infer_step on a few prior traces of the same trained network, called directly at every
              controlled address: the parameters of each returned proposal.
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
from pyprob.distributions import Bernoulli, Categorical, Normal, Poisson, Uniform  # noqa: E402
from pyprob.nn.dataset import Batch, OnlineDataset  # noqa: E402

K, BATCH, N_INFER = 5, 32, 4
EMB = {'y0': {'dim': 8, 'depth': 2}, 'y1': {'dim': 4, 'depth': 1}}


class FiveFamilies(Model):
    def __init__(self):
        super().__init__('five families')

    def forward(self):
        b = pyprob.sample(Bernoulli(torch.tensor([0.4])))
        u = pyprob.sample(Uniform(-1, 2))
        if int(b) == 1:
            k = pyprob.sample(Categorical([0.2, 0.3, 0.5]))
            m = float(k) * 0.5 + float(u)
        else:
            m = float(pyprob.sample(Poisson(3.0))) * 0.25
        mu = pyprob.sample(Normal(m, 1.0))
        pyprob.observe(Normal(mu, 0.5), name='y0')
        pyprob.observe(Normal(float(b) + float(u), 0.3), name='y1')
        return mu


def _priors(d):
    if d.name == 'Normal':
        return float(d.mean), float(d.stddev)
    if d.name == 'Uniform':
        return float(d.low), float(d.high)
    return 0.0, 0.0


def main():
    sys.path.insert(0, make_golden.ROOT)
    from oracle import network as onet
    pyprob.set_verbosity(0)
    pyprob.seed(31)
    model = FiveFamilies()
    with make_golden._silence():
        model.learn_inference_network(num_traces=128, batch_size=BATCH, inference_network=InferenceNetwork.FEEDFORWARD,
                                      observe_embeddings=EMB, proposal_mixture_components=K)
    net = model._inference_network
    ds = OnlineDataset(model)
    traces = [ds[i] for i in range(BATCH)]
    batch = Batch(traces)
    with make_golden._silence():
        net._polymorph(batch)
    net.zero_grad()
    success, loss = net._loss(batch)
    assert success
    loss.backward()
    names = list(EMB)
    fx = {'ff/loss': np.asarray(float(loss), dtype=np.float64), 'ff/observe_names': np.asarray(names),
          'ff/observe_in_dims': np.asarray([1, 1]), 'ff/dims': np.asarray([K, BATCH])}
    for k, v in net.state_dict().items():
        fx['ff/param/' + k] = v.detach().numpy()
    for k, p in net.named_parameters():
        fx['ff/grad/' + k] = (p.grad if p.grad is not None else torch.zeros_like(p)).detach().numpy()
    fx['ff/address_order'] = np.asarray(list(net._layers_proposal.keys()))
    assert len(batch.sub_batches) == 2, 'the model has two trace types'
    for s, sub in enumerate(batch.sub_batches):
        sb = onet.sub_batch_from_traces(sub, names)
        p = 'ff/sub{}/'.format(s)
        for k in ('addresses', 'families', 'num_categories'):
            fx[p + k] = np.asarray(sb[k])
        for k in ('values', 'prior0', 'prior1', 'obs'):
            fx[p + k] = sb[k].numpy()
    fx['ff/num_sub'] = np.asarray(len(batch.sub_batches))
    # _infer_init / _infer_step, called directly (no reference posterior run: its Poisson proposal draws non-integers)
    net.eval()
    with torch.no_grad():
        for i in range(N_INFER):
            trace = ds[BATCH + i]
            obs = {n: trace.named_variables[n].value for n in EMB}
            net._infer_init(obs)
            p = 'infer/trace{}/'.format(i)
            fx[p + 'obs'] = np.asarray([float(obs[n]) for n in EMB], np.float32)
            ctrl = trace.variables_controlled
            fx[p + 'addresses'] = np.asarray([v.address for v in ctrl])
            fx[p + 'families'] = np.asarray([v.distribution.name for v in ctrl])
            fx[p + 'prior0'] = np.asarray([_priors(v.distribution)[0] for v in ctrl], np.float32)
            fx[p + 'prior1'] = np.asarray([_priors(v.distribution)[1] for v in ctrl], np.float32)
            for t, var in enumerate(ctrl):
                q = net._infer_step(var, prev_variable=ctrl[t - 1] if t else None)
                key = '{}step{}/'.format(p, t)
                if q.name in ('Categorical', 'Bernoulli'):
                    fx[key + 'probs'] = (q._probs if q.name == 'Categorical' else q.probs).reshape(-1).numpy()
                else:
                    comps = q._distributions
                    if comps[0].name == 'TruncatedNormal':
                        fx[key + 'means'] = np.asarray([float(c._mean_non_truncated) for c in comps], np.float32)
                        fx[key + 'stddevs'] = np.asarray([float(c._stddev_non_truncated) for c in comps], np.float32)
                    else:
                        fx[key + 'means'] = np.asarray([float(c.mean) for c in comps], np.float32)
                        fx[key + 'stddevs'] = np.asarray([float(c.stddev) for c in comps], np.float32)
                    fx[key + 'probs'] = q._probs.reshape(-1).numpy()
    fx['infer/num_traces'] = np.asarray(N_INFER)
    np.savez_compressed(os.path.join(HERE, 'ff_golden.npz'), **fx)
    print('wrote ff_golden.npz with', len(fx), 'arrays')


if __name__ == '__main__':
    main()
