"""The CUDA per-site proposal step (ppb_ic_infer_step through InferenceNetwork._infer_step_lanes, the call the IC engine
makes, driven by _infer_step_batched) against the UNMODIFIED reference's _infer_step on real reference traces
(tests/golden/infer_golden.npz)."""
import numpy as np
import pytest
import torch

from pyprob_b200 import synthetic
from tests.test_oracle_infer import load_infer_golden

pytestmark = pytest.mark.gpu


def _network(fx, precision):
    P = fx['params']
    obs_emb = {}
    for name in fx['observe_names']:
        depth = sum(1 for k in P if k.startswith('_layers_observe_embedding.{}.'.format(name)) and k.endswith('weight'))
        dim = P['_layers_observe_embedding.{}._layers.{}.weight'.format(name, depth - 1)].shape[0]
        obs_emb[name] = {'dim': int(dim), 'depth': depth}
    fam = {}
    for tr in fx['traces']:
        for st in tr['steps']:
            fam[st['address']] = (st['family'], st['num_categories'])
    order = [k[len('_layers_address_embedding.'):] for k in P if k.startswith('_layers_address_embedding.')]
    net = synthetic.build_network(obs_emb, fx['observe_in_dims'], [(a, fam[a][0], fam[a][1]) for a in order],
                                  lstm_dim=fx['H'], mixture_components=fx['K'], precision=precision)
    net.load_reference_state_dict(P)
    return net


@pytest.mark.parametrize('precision', [0, 2])
def test_infer_step_matches_reference_proposals(cuda, precision):
    fx = load_infer_golden()
    net = _network(fx, precision)
    n, K = 7, fx['K']          # several particles in lock-step, all fed the golden trace's values
    for tr in fx['traces']:
        obs = {name: tr['obs'][i:i + 1] for i, name in enumerate(fx['observe_names'])}
        net._infer_init(obs)
        prev_a, prev_v = None, None
        for st in tr['steps']:
            p0 = st['prior0'] if st['family'] in ('Normal', 'Uniform') else None
            p1 = st['prior1'] if st['family'] in ('Normal', 'Uniform') else None
            params = net._infer_step_batched(st['address'], prev_a, prev_v, p0, p1, n).cpu()
            want = st['want']
            for row in params:
                if st['family'] == 'Categorical':
                    probs = row[:st['num_categories']]
                    np.testing.assert_allclose((probs / probs.sum()).numpy(), want['probs'], rtol=1e-4, atol=1e-6)
                else:
                    np.testing.assert_allclose(row[:K].numpy(), want['means'], rtol=1e-4, atol=1e-5)
                    np.testing.assert_allclose(row[K:2 * K].numpy(), want['stddevs'], rtol=1e-4, atol=1e-6)
                    np.testing.assert_allclose(row[2 * K:3 * K].numpy(), want['probs'], rtol=1e-4, atol=1e-6)
            prev_a, prev_v = st['address'], torch.full((n,), st['value'], device=cuda)
