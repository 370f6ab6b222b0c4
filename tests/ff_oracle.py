"""Oracle for the feed-forward inference network (TEST INFRASTRUCTURE ONLY), on top of oracle/network.py.

The reference's InferenceNetworkFeedForward (pyprob/nn/inference_network_feedforward.py) feeds the observation embedding
of each trace straight into the proposal layer of every step's address:
  * _loss (:68-98): sum over sub-batches and steps of -sum_b log q(v_b | obs_emb_b), divided by the batch size, with the
    -inf repair of the LSTM network (util.replace_negative_inf);
  * _infer_step (:53-66): proposal_layer.forward(obs_embedding, [variable]) — the previous variable plays no part.
Restated in plain torch CPU fp32 ops with the observation embedding and the proposal heads of oracle/network.py (Bernoulli
through tests/bernoulli_oracle.py).  repaired_rows as in oracle.network.loss; the CUDA path implements 'constant'.
"""
import os

import numpy as np
import torch

from oracle import network as onet
from tests import bernoulli_oracle as bo


def loss(params, sub_batches, observe_names, observe_in_dims, K, repaired_rows='constant'):
    """-> (loss, per-sub-batch list of [T, B] log-prob tensors)."""
    total = 0.0
    batch_size = sum(sb['values'].size(1) for sb in sub_batches)
    all_lp = []
    for sb in sub_batches:
        T = sb['values'].size(0)
        obs_emb = onet.embed_observe(params, sb['obs'], observe_names, observe_in_dims)
        lps = []
        for t in range(T):
            args = (params, sb['addresses'][t], sb['families'][t], sb['num_categories'][t], K)
            lp = bo.head_log_prob(*args, obs_emb, sb['values'][t], sb['prior0'][t], sb['prior1'][t])
            if torch.isinf(lp).any() and not torch.isnan(lp).any():
                dead = lp == -float('inf')
                if repaired_rows == 'constant' and bool(dead.any()) and not bool(dead.all()):
                    keep = torch.nonzero(~dead).view(-1)
                    live = bo.head_log_prob(*args, obs_emb[keep], sb['values'][t][keep], sb['prior0'][t][keep],
                                            sb['prior1'][t][keep])
                    lp = torch.full_like(lp, onet.LOG_EPSILON).index_copy(0, keep, live)
                else:
                    lp = lp.clone()
                    lp[dead] = onet.LOG_EPSILON
                    if repaired_rows == 'constant':
                        lp = lp.detach()
            lps.append(lp)
            total = total + (-lp.sum())
        all_lp.append(torch.stack(lps))
    return total / batch_size, all_lp


def loss_and_grads(params, sub_batches, observe_names, observe_in_dims, K, repaired_rows='constant'):
    p = {k: v.clone().float().requires_grad_(True) for k, v in params.items()}
    value, lps = loss(p, sub_batches, observe_names, observe_in_dims, K, repaired_rows=repaired_rows)
    value.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return value.detach(), grads, [x.detach() for x in lps]


def infer_step(params, obs_row, observe_names, observe_in_dims, K, address, family, prior0, prior1, n=1):
    """Proposal parameters at `address` for n particles that share the observation `obs_row` (see onet.head_params)."""
    obs_emb = onet.embed_observe(params, obs_row.reshape(1, -1).float(), observe_names, observe_in_dims).expand(n, -1)
    return bo.head_params(params, address, family, K, obs_emb, prior0, prior1)


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ff_golden.npz')
_cache = {}


def load_fixture():
    """ff_golden.npz (tests/golden/make_ff_golden.py, the unmodified reference): the network part in the form of
    tests/bernoulli_oracle.load_fixture, plus 'infer': per trace the observation, the steps and the reference's proposals."""
    if 'npz' not in _cache:
        _cache['npz'] = dict(np.load(GOLDEN))
    z = _cache['npz']
    fx = {'loss': float(z['ff/loss']), 'observe_names': [str(x) for x in z['ff/observe_names']],
          'observe_in_dims': [int(x) for x in z['ff/observe_in_dims']], 'K': int(z['ff/dims'][0]),
          'batch_size': int(z['ff/dims'][1]), 'address_order': [str(x) for x in z['ff/address_order']],
          'params': {k[len('ff/param/'):]: torch.from_numpy(v) for k, v in z.items() if k.startswith('ff/param/')},
          'grads': {k[len('ff/grad/'):]: torch.from_numpy(v) for k, v in z.items() if k.startswith('ff/grad/')},
          'subs': [], 'infer': []}
    for s in range(int(z['ff/num_sub'])):
        p = 'ff/sub{}/'.format(s)
        fx['subs'].append({'addresses': [str(x) for x in z[p + 'addresses']],
                           'families': [str(x) for x in z[p + 'families']],
                           'num_categories': [int(x) for x in z[p + 'num_categories']],
                           'values': torch.from_numpy(z[p + 'values']), 'prior0': torch.from_numpy(z[p + 'prior0']),
                           'prior1': torch.from_numpy(z[p + 'prior1']), 'obs': torch.from_numpy(z[p + 'obs'])})
    for i in range(int(z['infer/num_traces'])):
        p = 'infer/trace{}/'.format(i)
        steps = []
        for t, (a, f) in enumerate(zip(z[p + 'addresses'], z[p + 'families'])):
            q = '{}step{}/'.format(p, t)
            steps.append({'address': str(a), 'family': str(f), 'prior0': float(z[p + 'prior0'][t]),
                          'prior1': float(z[p + 'prior1'][t]),
                          'proposal': tuple(z[q + k] for k in ('means', 'stddevs', 'probs') if q + k in z)})
        fx['infer'].append({'obs': torch.from_numpy(z[p + 'obs']), 'steps': steps})
    return fx


def address_table(fx):
    """(address, family, num_categories) in the fixture network's address order."""
    fam = {}
    for sb in fx['subs']:
        for a, f, c in zip(sb['addresses'], sb['families'], sb['num_categories']):
            fam[a] = (f, c)
    return [(a,) + fam[a] for a in fx['address_order']]


def infer_sequence(params, obs_row, observe_names, observe_in_dims, K, steps, n=1):
    """The per-site proposals of one address sequence, in the form of oracle.network.infer_sequence: the feed-forward
    network ignores each step's previous value."""
    def prior(x):
        return 0.0 if x is None else x
    return [infer_step(params, obs_row, observe_names, observe_in_dims, K, st['address'], st['family'], prior(st['prior0']),
                       prior(st['prior1']), n) for st in steps]


def relu_flip_bound(params, sub_batches, observe_names, observe_in_dims, K, rel=2e-5):
    """Elementwise bound on how far every gradient can move when first-layer head units whose pre-activation z lies within
    rounding of zero (|z| <= rel * (|x| |W1|^T + |b1|), x the observation embedding) take the other side of their ReLU.
    Such a flip changes d_hid[b, j] by the full upstream gradient g = dL/dhid[b, j] (taken through the rest of the head,
    independent of the mask): dW1[j] by g x[b], db1[j] by g, and d obs_emb[b] by g W1[j], which the observation layers carry
    back to their parameters.  -> ({name: bound tensor}, number of such units)."""
    p = {k: v.clone().float().requires_grad_(True) for k, v in params.items()}
    batch_size = sum(sb['values'].size(1) for sb in sub_batches)
    bound = {k: torch.zeros_like(v) for k, v in params.items()}
    count = 0
    for sb in sub_batches:
        with torch.no_grad():
            x = onet.embed_observe(params, sb['obs'], observe_names, observe_in_dims)
        for t in range(sb['values'].size(0)):
            a, fam = sb['addresses'][t], sb['families'][t]
            pre = '_layers_proposal.{}._ff._layers.'.format(a)
            W1, b1 = params[pre + '0.weight'], params[pre + '0.bias']
            z = x @ W1.t() + b1
            amb = z.abs() <= rel * (x.abs() @ W1.abs().t() + b1.abs())
            if not bool(amb.any()):
                continue
            hid = z.clamp_min(0).requires_grad_(True)
            top = {'_layers_proposal.top._ff._layers.0.weight': params[pre + '1.weight'],
                   '_layers_proposal.top._ff._layers.0.bias': params[pre + '1.bias']}
            lp = bo.head_log_prob(top, 'top', fam, sb['num_categories'][t], K, hid, sb['values'][t], sb['prior0'][t],
                                  sb['prior1'][t])
            (-lp.sum() / batch_size).backward()
            g = hid.grad
            for bi, j in torch.nonzero(amb).tolist():
                count += 1
                gu = float(g[bi, j].abs())
                bound[pre + '0.weight'][j] += gu * x[bi].abs()
                bound[pre + '0.bias'][j] += gu
                for q in p.values():
                    q.grad = None
                e = onet.embed_observe(p, sb['obs'][bi:bi + 1], observe_names, observe_in_dims)
                e.backward((gu * W1[j]).view(1, -1))
                for k, q in p.items():
                    if q.grad is not None:
                        bound[k] += q.grad.abs()
    return bound, count
