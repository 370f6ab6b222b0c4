"""Oracle for the Bernoulli proposal head (TEST INFRASTRUCTURE ONLY), on top of oracle/network.py.

The reference's ProposalBernoulliBernoulli (pyprob/nn/proposal_bernoulli_bernoulli.py:9-20) is an
EmbeddingFeedForward(H -> 1, two layers, no activation on the last) followed by probs = sigmoid(x) + 1e-8 and a
torch Bernoulli(probs).  Its log_prob is -BCEWithLogits(log pc - log1p(-pc), v) with pc = clamp_probs(probs)
(torch/distributions/bernoulli.py), restated below in plain torch CPU fp32 ops.

oracle.network stays as it is: its loss and infer_sequence look head_log_prob / head_params up by module name, so
`bernoulli_heads()` runs them unchanged with the two head functions below, which handle 'Bernoulli' and hand every
other family to the originals.  The loss is then the per-row -sum_b log q_b(v_b) / B that every family uses; the
reference computes exactly that when the prior's probs is a 1-element tensor.  With a Python-scalar probs its values
are 0-d, the proposal's probs [B, 1], and torch broadcasts the log_prob to [B, B]: `pairwise_loss` restates that case
for the test that pins it.
"""
import contextlib
import os
from unittest import mock

import numpy as np
import torch

from oracle import network as onet
from oracle import scoring

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'bernoulli_golden.npz')
_cache = {}
_head_log_prob, _head_params = onet.head_log_prob, onet.head_params


def load_fixture(tag):
    """One network fixture of bernoulli_golden.npz ('bern' or 'quirk'), in the form tests/netfixture.py gives."""
    if 'npz' not in _cache:
        _cache['npz'] = dict(np.load(GOLDEN))
    z, pre = _cache['npz'], tag + '/'
    fx = {'loss': float(z[pre + 'loss']),
          'observe_names': [str(x) for x in z[pre + 'observe_names']],
          'observe_in_dims': [int(x) for x in z[pre + 'observe_in_dims']],
          'lstm_dim': int(z[pre + 'dims'][0]), 'K': int(z[pre + 'dims'][1]), 'batch_size': int(z[pre + 'dims'][2]),
          'address_order': [str(x) for x in z[pre + 'address_order']],
          'type_order': [str(x) for x in z[pre + 'type_order']],
          'params': {k[len(pre + 'param/'):]: torch.from_numpy(v) for k, v in z.items() if k.startswith(pre + 'param/')},
          'grads': {k[len(pre + 'grad/'):]: torch.from_numpy(v) for k, v in z.items() if k.startswith(pre + 'grad/')},
          'subs': []}
    for s in range(int(z[pre + 'num_sub'])):
        p = '{}sub{}/'.format(pre, s)
        fx['subs'].append({'addresses': [str(x) for x in z[p + 'addresses']],
                           'families': [str(x) for x in z[p + 'families']],
                           'num_categories': [int(x) for x in z[p + 'num_categories']],
                           'values': torch.from_numpy(z[p + 'values']), 'prior0': torch.from_numpy(z[p + 'prior0']),
                           'prior1': torch.from_numpy(z[p + 'prior1']), 'obs': torch.from_numpy(z[p + 'obs'])})
    return fx


def load_scoring():
    if 'npz' not in _cache:
        _cache['npz'] = dict(np.load(GOLDEN))
    z = _cache['npz']
    return {k[len('scoring/'):]: v for k, v in z.items() if k.startswith('scoring/')}


def bernoulli_log_prob(value, probs):
    value, probs = torch.as_tensor(value, dtype=torch.float32), torch.as_tensor(probs, dtype=torch.float32)
    pc = scoring.clamp_probs(probs)
    logits, value = torch.broadcast_tensors(torch.log(pc) - torch.log1p(-pc), value)
    return -torch.nn.functional.binary_cross_entropy_with_logits(logits, value, reduction='none')


def bernoulli_probs(params, address, h):
    x = onet._ff(h, params, '_layers_proposal.{}._ff'.format(address), False)
    return torch.sigmoid(x).view(-1) + 1e-8


def head_log_prob(params, address, family, num_categories, K, h, values, prior0, prior1):
    if family == 'Bernoulli':
        return bernoulli_log_prob(values, bernoulli_probs(params, address, h))
    return _head_log_prob(params, address, family, num_categories, K, h, values, prior0, prior1)


def head_params(params, address, family, K, h, prior0, prior1):
    if family == 'Bernoulli':
        return (bernoulli_probs(params, address, h).view(-1, 1),)
    return _head_params(params, address, family, K, h, prior0, prior1)


@contextlib.contextmanager
def bernoulli_heads(log_prob=head_log_prob):
    with mock.patch.object(onet, 'head_log_prob', log_prob), mock.patch.object(onet, 'head_params', head_params):
        yield


def loss(*args, **kwargs):
    with bernoulli_heads():
        return onet.loss(*args, **kwargs)


def loss_and_grads(*args, **kwargs):
    with bernoulli_heads():
        return onet.loss_and_grads(*args, **kwargs)


def infer_sequence(*args, **kwargs):
    with bernoulli_heads():
        return onet.infer_sequence(*args, **kwargs)


def pairwise_loss(params, sub_batches, observe_names, observe_in_dims, K):
    """The reference's loss when every Bernoulli prior has a Python-scalar probs: each Bernoulli step contributes
    -sum_b sum_b' log q_b(v_b') (0-d values against [B, 1] proposal probs broadcast to [B, B]) instead of
    -sum_b log q_b(v_b); every other step is per row."""
    extra = []

    def log_prob(params_, address, family, num_categories, K_, h, values, prior0, prior1):
        lp = head_log_prob(params_, address, family, num_categories, K_, h, values, prior0, prior1)
        if family == 'Bernoulli':
            pair = bernoulli_log_prob(values.view(1, -1), bernoulli_probs(params_, address, h).view(-1, 1))
            extra.append(float(pair.double().sum()) - float(lp.double().sum()))
        return lp
    with bernoulli_heads(log_prob), torch.no_grad():
        value, _ = onet.loss(params, sub_batches, observe_names, observe_in_dims, K)
    return float(value) - sum(extra) / sum(sb['values'].size(1) for sb in sub_batches)
