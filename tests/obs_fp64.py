"""The observe embedding restated in plain torch with autograd, at any dtype, layer by layer (TEST INFRASTRUCTURE ONLY).

The same computation as oracle.network.embed_observe (per-observable Linear+ReLU chains, their concatenation, the final
Linear+ReLU chain), driven by the whole network's loss: tests/lstm_fp64.py for the LSTM network, and `ff_loss_and_grads`
below (tests/ff_oracle.py's loss at any dtype) for the feed-forward one.  For every layer of every sub-batch it returns
what a tolerance model needs:
  x    the layer's input        z   its pre-activation        y = relu(z)
  dz   d loss / d z             dy  d loss / d y (retain_grad; dy is what the layer would pass down were its ReLU open)
`term_magnitudes` turns them into M, the size of the terms each weight and bias gradient element sums, and
`relu_flip_bound` into a bound on what units whose pre-activation lies within rounding of zero can move when they land on
the other side of their ReLU.
"""
import torch

from oracle import network as onet
from tests import lstm_fp64


def _chain(x, params, prefix, chain, layers):
    """Linear+ReLU layers `prefix._layers.l` on x, each recorded in `layers` (chain: the observable's index, None for the
    final chain)."""
    l = 0
    while '{}._layers.{}.weight'.format(prefix, l) in params:
        name = '{}._layers.{}'.format(prefix, l)
        z = torch.nn.functional.linear(x, params[name + '.weight'], params[name + '.bias'])
        y = torch.relu(z)
        if z.requires_grad:
            z.retain_grad()
            y.retain_grad()
        layers.append({'name': name, 'chain': chain, 'x': x, 'z': z, 'y': y})
        x = y
        l += 1
    return x


def embed(params, obs, observe_names, observe_in_dims, layers):
    """onet.embed_observe, with every layer appended to `layers` in forward order: the chains of the observables in
    order, then the final chain."""
    pieces, col = [], 0
    for j, (name, d) in enumerate(zip(observe_names, observe_in_dims)):
        pieces.append(_chain(obs[:, col:col + d], params, '_layers_observe_embedding.{}'.format(name), j, layers))
        col += d
    return _chain(torch.cat(pieces, dim=1), params, '_layers_observe_embedding_final', None, layers)


def ff_loss_and_grads(params, sub_batches, observe_names, observe_in_dims, K, dtype=torch.float64, embed=onet.embed_observe):
    """InferenceNetworkFeedForward._loss (tests/ff_oracle.loss, repaired_rows='constant') at `dtype`: every step's head reads
    the observation embedding of its trace.  The heads are lstm_fp64's.  -> {'loss', 'lps', 'grads'}, detached."""
    p = {k: torch.as_tensor(v).detach().to(dtype).clone().requires_grad_(True) for k, v in params.items()}
    batch_size = sum(int(torch.as_tensor(sb['values']).shape[1]) for sb in sub_batches)
    total = torch.zeros((), dtype=dtype)
    lps = []
    for sb in sub_batches:
        values, prior0, prior1 = (torch.as_tensor(sb[k]).to(dtype) for k in ('values', 'prior0', 'prior1'))
        obs_emb = embed(p, torch.as_tensor(sb['obs']).to(dtype), observe_names, observe_in_dims)
        sub = [lstm_fp64._head_log_q(p, a, fam, C, K, obs_emb, values[t], prior0[t], prior1[t])
               for t, (a, fam, C) in enumerate(zip(sb['addresses'], sb['families'], sb['num_categories']))]
        total = total - sum(lp.sum() for lp in sub)
        lps.append(torch.stack(sub))
    loss = total / batch_size
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return {'loss': loss.detach(), 'lps': [x.detach() for x in lps], 'grads': grads}


def loss_and_grads(params, sub_batches, observe_names, observe_in_dims, K, dtype=torch.float64, feedforward=False):
    """The whole network's loss and gradients at `dtype` (lstm_fp64.loss_and_grads, or ff_loss_and_grads), plus 'obs': per
    sub-batch the list of its observe-embedding layers {name, chain, x, z, y, dz, dy}, all detached."""
    recorded = []

    def record(p, obs, names, dims):
        recorded.append([])
        return embed(p, obs, names, dims, recorded[-1])
    run = ff_loss_and_grads if feedforward else lstm_fp64.loss_and_grads
    res = run(params, sub_batches, observe_names, observe_in_dims, K, dtype=dtype, embed=record)

    def grad(t):
        return t.grad.detach() if t.grad is not None else torch.zeros_like(t.detach())
    res['obs'] = [[{'name': L['name'], 'chain': L['chain'], 'x': L['x'].detach(), 'z': L['z'].detach(),
                    'y': L['y'].detach(), 'dz': grad(L['z']), 'dy': grad(L['y'])} for L in sub] for sub in recorded]
    return res


def term_magnitudes(res):
    """{name.weight: M_W, name.bias: M_b} of every observe-embedding layer, over every sub-batch:
    M_W[o, i] = sum_b |dz[b, o]| |x[b, i]|, M_b[o] = sum_b |dz[b, o]|."""
    out = {}
    for sub in res['obs']:
        for L in sub:
            g = L['dz'].abs()
            for k, v in ((L['name'] + '.weight', g.t() @ L['x'].abs()), (L['name'] + '.bias', g.sum(0))):
                out[k] = out[k] + v if k in out else v
    return out


def relu_flip_bound(params, res, rel):
    """Elementwise bound on how far each observe-embedding gradient can move when the units whose pre-activation is within
    rounding of zero, |z| <= rel (|x| |W|^T + |b|), take the other side of their ReLU (ff_oracle.relu_flip_bound does the
    same for the feed-forward network's head units).  A flipped unit (b, o) changes dz[b, o] by at most |dy[b, o]|: its
    layer's dW[o] by that times |x[b]|, db[o] by it, and dx[b] by it times |W[o]|, which every layer below carries on
    through its open (or ambiguous) units, and so on down to the observations.  The forward value of such a unit moves by
    no more than |z|, within rounding.  -> ({name: bound}, number of ambiguous units)."""
    bound, count = {}, 0
    for sub in res['obs']:
        def step(L, D):
            nonlocal count
            W = params[L['name'] + '.weight'].to(L['x'].dtype).abs()
            b = params[L['name'] + '.bias'].to(L['x'].dtype).abs()
            amb = L['z'].abs() <= rel * (L['x'].abs() @ W.t() + b)
            count += int(amb.sum())
            dz = L['dy'].abs() * amb
            if D is not None:
                dz = dz + D * ((L['z'] > 0) | amb)
            for k, v in ((L['name'] + '.weight', dz.t() @ L['x'].abs()), (L['name'] + '.bias', dz.sum(0))):
                bound[k] = bound[k] + v if k in bound else v
            return dz @ W
        D = None
        for L in reversed([L for L in sub if L['chain'] is None]):
            D = step(L, D)
        col = 0
        for j in sorted({L['chain'] for L in sub if L['chain'] is not None}):
            chain = [L for L in sub if L['chain'] == j]
            width = chain[-1]['y'].size(1)
            Dj = D[:, col:col + width]
            for L in reversed(chain):
                Dj = step(L, Dj)
            col += width
    return bound, count
