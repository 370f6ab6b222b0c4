"""Synthetic networks and trace minibatches of a named shape (bench.py workloads, tests).

Nothing here touches the user-model interpreter: a network is declared by its observables and its address
table, a minibatch by per-sub-batch value arrays — the same inputs the encoder receives from real traces.
"""
import numpy as np
import torch

from .encoding import EncodedBatch, SubBatch
from .network import InferenceNetworkFeedForward, InferenceNetworkLSTM
from .util import InferenceNetwork


class _ExampleTrace:
    """Just enough of a trace for InferenceNetworkLSTM._init_layers_observe_embedding."""

    def __init__(self, shapes):
        self.named_variables = {k: k for k in shapes}
        self._shapes = shapes

    def value_shape(self, variable):
        return self._shapes[variable]


def build_network(observe_embeddings, observe_in_dims, addresses, lstm_dim=512, mixture_components=10, precision=0,
                  seed=0, inference_network=InferenceNetwork.LSTM, sample_embedding_dim=4):
    """addresses: list of (address, distribution name, num_categories) in address-id order."""
    torch.manual_seed(seed)
    if inference_network == InferenceNetwork.FEEDFORWARD:
        net = InferenceNetworkFeedForward(model=None, observe_embeddings=observe_embeddings,
                                          proposal_mixture_components=mixture_components, precision=precision)
    else:
        net = InferenceNetworkLSTM(model=None, observe_embeddings=observe_embeddings, lstm_dim=lstm_dim,
                                   sample_embedding_dim=sample_embedding_dim,
                                   proposal_mixture_components=mixture_components, precision=precision)
    shapes = {name: (d,) if d > 1 else () for name, d in zip(observe_embeddings.keys(), observe_in_dims)}
    net._ensure_initialized(_ExampleTrace(shapes))
    for address, dist_name, C in addresses:
        net._add_address(address, dist_name, C)
    net._rebind()
    return net


class ArrayBatch:
    """A minibatch given as plain arrays (one dict per sub-batch: addresses, values, prior0, prior1, obs)."""

    def __init__(self, subs, families=None):
        self.subs = subs
        self.size = int(sum(np.asarray(sb['values']).shape[1] for sb in subs))
        self.num_sub_batches = len(subs)
        self.mean_length_controlled = sum(np.asarray(sb['values']).shape[0] * np.asarray(sb['values']).shape[1]
                                          for sb in subs) / self.size
        self._encoded = None

    def address_signature(self):
        seen, out = set(), []
        for sb in self.subs:
            for a, f, c in zip(sb['addresses'], sb['families'], sb['num_categories']):
                if a not in seen:
                    seen.add(a)
                    out.append((a, f, int(c)))
        return out

    def encode(self, net):
        if self._encoded is None:
            subs = []
            for sb in self.subs:
                for a in sb['addresses']:
                    if a not in net._addresses:
                        print('Address unknown by inference network: {}'.format(a))
                        return None
                ids = [net._addresses[a]['id'] for a in sb['addresses']]
                subs.append(SubBatch(ids, np.asarray(sb['values']), np.asarray(sb['prior0']), np.asarray(sb['prior1']),
                                     np.asarray(sb['obs'])))
            self._encoded = EncodedBatch(subs, row_align=net.row_align)
        return self._encoded


def random_sub_batch(rng, addresses, B, obs_dim):
    """Random values of the right support for each (address, family, C) step."""
    T = len(addresses)
    values = np.zeros((T, B), np.float32)
    p0 = np.zeros((T, B), np.float32)
    p1 = np.zeros((T, B), np.float32)
    for t, (_, fam, C) in enumerate(addresses):
        if fam == 'Normal':
            p0[t] = rng.normal(0, 1, B)
            p1[t] = rng.uniform(0.5, 2.0, B)
            values[t] = p0[t] + p1[t] * rng.normal(0, 1, B)
        elif fam == 'Uniform':
            p0[t] = rng.uniform(-2, 0, B)
            p1[t] = p0[t] + rng.uniform(0.5, 3.0, B)
            values[t] = p0[t] + (p1[t] - p0[t]) * rng.uniform(0.02, 0.98, B)
        elif fam == 'Poisson':
            values[t] = rng.poisson(3.0, B)
        elif fam == 'Bernoulli':
            values[t] = rng.integers(0, 2, B)
        else:
            values[t] = rng.integers(0, C, B)
    return {'addresses': [a for a, _, _ in addresses], 'families': [f for _, f, _ in addresses],
            'num_categories': [c for _, _, c in addresses], 'values': values, 'prior0': p0, 'prior1': p1,
            'obs': rng.normal(0, 1, (B, obs_dim)).astype(np.float32)}


# ---- BASELINE.json workloads ---------------------------------------------------------------------------------
def gum_network(lstm_dim=512, precision=0, seed=0, inference_network=InferenceNetwork.LSTM):
    """Config 2: GaussianUnknownMean, observe embeddings 32+32 (examples/gaussian_unknown_mean.ipynb)."""
    return build_network({'obs0': {'dim': 32}, 'obs1': {'dim': 32}}, [1, 1],
                         [('98__forward__mu__Normal__1', 'Normal', 0)], lstm_dim=lstm_dim, precision=precision,
                         seed=seed, inference_network=inference_network)


def gum_batch(rng, B):
    mu = (1.0 + np.sqrt(5.0) * rng.normal(0, 1, B)).astype(np.float32)
    obs = (mu[:, None] + np.sqrt(2.0) * rng.normal(0, 1, (B, 2))).astype(np.float32)
    return ArrayBatch([{'addresses': ['98__forward__mu__Normal__1'], 'families': ['Normal'], 'num_categories': [0],
                        'values': mu[None, :], 'prior0': np.full((1, B), 1.0, np.float32),
                        'prior1': np.full((1, B), np.sqrt(5.0), np.float32), 'obs': obs}])


def synthetic50_addresses(T=50, C=4):
    return [('{}__forward__x{}__{}__1'.format(10 + 6 * t, t, 'Normal' if t % 2 == 0 else 'Categorical(len_probs:%d)' % C),
             'Normal' if t % 2 == 0 else 'Categorical', 0 if t % 2 == 0 else C) for t in range(T)]


def synthetic50_network(lstm_dim=512, obs_dim=256, precision=0, seed=0, T=50, inference_network=InferenceNetwork.LSTM):
    """Config 4: 50 addresses alternating Normal(0,1) / Categorical(4), one observable, FF dim 256 depth 2."""
    return build_network({'obs': {'dim': obs_dim}}, [1], synthetic50_addresses(T), lstm_dim=lstm_dim,
                         precision=precision, seed=seed, inference_network=inference_network)


def synthetic50_batch(rng, B, T=50):
    addrs = synthetic50_addresses(T)
    sb = random_sub_batch(rng, addrs, B, 1)
    for t, (_, fam, _) in enumerate(addrs):
        if fam == 'Normal':
            sb['prior0'][t] = 0.0
            sb['prior1'][t] = 1.0
            sb['values'][t] = rng.normal(0, 1, B)
    sb['obs'] = (sb['values'][::2].sum(0) + rng.normal(0, 1, B)).astype(np.float32).reshape(B, 1)
    return ArrayBatch([sb])
