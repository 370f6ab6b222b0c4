"""Golden input / output of the trace bridge test (tests/test_offline_reference_bridge.py), from the UNMODIFIED reference.

    python tests/golden/make_bridge_golden.py <reference checkout>    # writes tests/golden/bridge_golden.npz

A branching model (all four distribution families, two trace types) trains a small reference LSTM network (seeded); then 40
prior traces are drawn from the reference's OnlineDataset and grouped by the reference's own Batch.  Stored: every controlled
variable of every trace (address, family, category count, value, distribution parameters), the observed values, the
network parameters, the Batch grouping (sub-batch sizes and address lists) and the reference's _loss on that batch.
"""
import contextlib
import io
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if len(sys.argv) != 2:
    sys.exit(__doc__)
sys.path.insert(0, sys.argv[1])
sys.path.insert(0, os.path.join(ROOT, 'oracle', 'ref_stubs'))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import pyprob  # noqa: E402
from pyprob import InferenceNetwork, Model  # noqa: E402
from pyprob.distributions import Categorical, Normal, Poisson, Uniform  # noqa: E402
from pyprob.nn.dataset import Batch, OnlineDataset  # noqa: E402


class Branching(Model):
    def forward(self):
        u = pyprob.sample(Uniform(-1, 2))
        k = pyprob.sample(Categorical([0.2, 0.3, 0.5]))
        if int(k) == 0:
            z = pyprob.sample(Normal(u, 0.5))
        else:
            z = pyprob.sample(Poisson(3.0)) * 0.25
        mu = pyprob.sample(Normal(z * 0.1, 1))
        pyprob.observe(Normal(mu, 0.3), name='y0')
        pyprob.observe(Normal(u, 0.7), name='y1')
        return mu


def _variable(var):
    d = var.distribution
    name = type(d).__name__
    rec = {'address': var.address, 'family': name, 'value': float(var.value)}
    if name == 'Categorical':
        rec['num_categories'] = int(d.num_categories)
    elif name == 'Normal':
        rec['mean'], rec['stddev'] = float(d.mean), float(d.stddev)
    elif name == 'Uniform':
        rec['low'], rec['high'] = float(d.low), float(d.high)
    return rec


def main():
    pyprob.set_verbosity(0)
    pyprob.seed(5)
    model = Branching()
    emb = {'y0': {'dim': 8, 'depth': 2}, 'y1': {'dim': 4, 'depth': 1}}
    with contextlib.redirect_stdout(io.StringIO()):
        model.learn_inference_network(num_traces=48, batch_size=24, inference_network=InferenceNetwork.LSTM,
                                      observe_embeddings=emb, lstm_dim=16, proposal_mixture_components=3)
    net = model._inference_network
    ds = OnlineDataset(model)
    traces = [ds[i] for i in range(40)]
    batch = Batch(traces)
    with contextlib.redirect_stdout(io.StringIO()):
        net._polymorph(batch)
    with torch.no_grad():
        ok, ref_loss = net._loss(batch)
    assert ok
    names = list(emb.keys())
    meta = {
        'observe_names': names,
        'traces': [{'variables': [_variable(v) for v in tr.variables_controlled],
                    'observed': {nm: np.asarray(tr.named_variables[nm].value, np.float32).reshape(-1).tolist()
                                 for nm in names}} for tr in traces],
        'sub_batch_sizes': [len(sb) for sb in batch.sub_batches],
        'sub_batch_addresses': [[v.address for v in sb[0].variables_controlled] for sb in batch.sub_batches],
        'ref_loss': float(ref_loss),
    }
    out = {'meta': np.frombuffer(json.dumps(meta).encode(), np.uint8)}
    for k, v in net.state_dict().items():
        out['param/' + k] = v.detach().cpu().numpy()
    np.savez_compressed(os.path.join(HERE, 'bridge_golden.npz'), **out)


if __name__ == '__main__':
    main()
