"""Oracle: the proposal network's training loss, restated from the reference (TEST INFRASTRUCTURE ONLY).

Follows, step by step and with the same tensor shapes,
  * sub-batching                 pyprob/nn/dataset.py:21-37
  * observe embedding            pyprob/nn/inference_network.py:132-139, pyprob/nn/embedding_feedforward.py:35-48
  * LSTM input assembly + LSTM   pyprob/nn/inference_network_lstm.py:146-188 (h0 = c0 = 0, gate order i,f,g,o)
  * proposal heads               pyprob/nn/proposal_normal_normal_mixture.py:18-35,
                                 proposal_uniform_truncated_normal_mixture.py:18-36,
                                 proposal_poisson_truncated_normal_mixture.py:20-36,
                                 proposal_categorical_categorical.py:16-20
  * loss reduction / -inf repair pyprob/nn/inference_network_lstm.py:207-220, pyprob/util.py:278-284
using plain torch CPU fp32 ops with autograd (the reference's own numerics backend).  Parameters are passed
as a dict keyed by the reference's state_dict names.
"""
import math

import torch

from . import scoring

LOG_EPSILON = math.log(1e-8)


def group_traces(traces):
    """Reference Batch: group by concatenated controlled addresses, dict insertion order (dataset.py:25-36)."""
    groups = {}
    for tr in traces:
        key = ''.join(v.address for v in tr.variables_controlled)
        groups.setdefault(key, []).append(tr)
    return list(groups.values())


def sub_batch_from_traces(traces, observe_names):
    """One sub-batch (traces sharing an address sequence) -> plain arrays (duck-typed on reference Traces)."""
    ex = traces[0]
    T, B = len(ex.variables_controlled), len(traces)
    out = {'addresses': [v.address for v in ex.variables_controlled],
           'families': [v.distribution.name for v in ex.variables_controlled],
           'num_categories': [int(getattr(v.distribution, 'num_categories', 0) or 0) for v in ex.variables_controlled]}
    values = torch.zeros(T, B)
    p0 = torch.zeros(T, B)
    p1 = torch.zeros(T, B)
    for b, tr in enumerate(traces):
        for t, v in enumerate(tr.variables_controlled):
            values[t, b] = float(v.value)
            d = v.distribution
            if d.name == 'Normal':
                p0[t, b], p1[t, b] = float(d.mean), float(d.stddev)
            elif d.name == 'Uniform':
                p0[t, b], p1[t, b] = float(d.low), float(d.high)
    obs = torch.stack([torch.cat([torch.as_tensor(tr.named_variables[n].value, dtype=torch.float32).reshape(-1)
                                  for n in observe_names]) for tr in traces])
    out.update(values=values, prior0=p0, prior1=p1, obs=obs)
    return out


def _ff(x, params, prefix, relu_last):
    i = 0
    while '{}._layers.{}.weight'.format(prefix, i) in params:
        i += 1
    for l in range(i):
        x = torch.nn.functional.linear(x, params['{}._layers.{}.weight'.format(prefix, l)],
                                       params['{}._layers.{}.bias'.format(prefix, l)])
        if l < i - 1 or relu_last:
            x = torch.relu(x)
    return x


def embed_observe(params, obs, observe_names, observe_in_dims):
    pieces, col = [], 0
    for name, d in zip(observe_names, observe_in_dims):
        pieces.append(_ff(obs[:, col:col + d], params, '_layers_observe_embedding.{}'.format(name), True))
        col += d
    return _ff(torch.cat(pieces, dim=1), params, '_layers_observe_embedding_final', True)


def lstm(x_seq, params):
    """x_seq [T,B,I] -> outputs [T,B,H]; explicit cell, h0 = c0 = 0."""
    W_ih, W_hh = params['_layers_lstm.weight_ih_l0'], params['_layers_lstm.weight_hh_l0']
    b_ih, b_hh = params['_layers_lstm.bias_ih_l0'], params['_layers_lstm.bias_hh_l0']
    H = W_hh.size(1)
    B = x_seq.size(1)
    h = torch.zeros(B, H)
    c = torch.zeros(B, H)
    outs = []
    for t in range(x_seq.size(0)):
        g = x_seq[t] @ W_ih.t() + b_ih + h @ W_hh.t() + b_hh
        i, f, gg, o = g[:, :H], g[:, H:2 * H], g[:, 2 * H:3 * H], g[:, 3 * H:]
        i, f, gg, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(gg), torch.sigmoid(o)
        c = f * c + i * gg
        h = o * torch.tanh(c)
        outs.append(h)
    return torch.stack(outs)


def head_log_prob(params, address, family, num_categories, K, h, values, prior0, prior1):
    x = _ff(h, params, '_layers_proposal.{}._ff'.format(address), False)
    if family == 'Categorical':
        probs = torch.softmax(x, dim=1) + 1e-8
        return scoring.categorical_log_prob(values, probs)
    means, stddevs, coeffs = x[:, :K], x[:, K:2 * K], torch.softmax(x[:, 2 * K:], dim=1)
    if family == 'Normal':
        means = prior0.view(-1, 1) + means * prior1.view(-1, 1)
        stddevs = torch.exp(stddevs) * prior1.view(-1, 1)
        comp = scoring.normal_log_prob(values.view(-1, 1), means, stddevs)
    elif family == 'Uniform':
        rng = (prior1 - prior0).view(-1, 1)
        means = prior0.view(-1, 1) + torch.sigmoid(means) * rng
        stddevs = rng / 1000 + torch.sigmoid(stddevs) * rng * 10
        comp = scoring.truncated_normal_log_prob(values.view(-1, 1), means, stddevs, prior0.view(-1, 1),
                                                 prior1.view(-1, 1))
    elif family == 'Poisson':
        means = torch.sigmoid(means) * 40.0
        stddevs = torch.exp(stddevs)
        comp = scoring.truncated_normal_log_prob(values.view(-1, 1), means, stddevs, torch.zeros(1), 40 * torch.ones(1))
    else:
        raise RuntimeError('unsupported family ' + family)
    return scoring.mixture_log_prob(comp, coeffs)


def sample_embedding(params, address, family, num_categories, values):
    if family == 'Categorical':
        x = torch.nn.functional.one_hot(values.long(), num_categories).float()
    else:
        x = values.view(-1, 1)
    return _ff(x, params, '_layers_sample_embedding.{}'.format(address), True)


def _sample_dim(params):
    return next(v.size(0) for k, v in params.items() if k.startswith('_layers_sample_embedding.') and k.endswith('.bias'))


def loss(params, sub_batches, observe_names, observe_in_dims, K, addr_dim=64, type_dim=8, repaired_rows='reference'):
    """-> (loss, per-sub-batch list of [T,B] log-prob tensors).  sub_batches: dicts from sub_batch_from_traces.

    repaired_rows: what happens to the GRADIENT of rows whose log q is -inf and gets replaced by log(1e-8)
    (inference_network_lstm.py:207-217, util.py:278-284).  The VALUE is the same either way.
      'reference'  the reference's own autograd graph: the replaced entries receive a zero upstream gradient, but the
                   backward of logsumexp multiplies it by softmax(-inf, ..., -inf) = NaN, so EVERY shared parameter gets
                   a NaN gradient (and the reference's next optimizer.step() destroys the network) — kept to document it;
      'constant'   the replaced value is the constant the reference's code intends: such rows contribute no gradient
                   (the head is evaluated on the remaining rows only).  This is what the CUDA path implements."""
    sample_dim = _sample_dim(params)
    total = 0.0
    batch_size = sum(sb['values'].size(1) for sb in sub_batches)
    all_lp = []
    for sb in sub_batches:
        T, B = sb['values'].shape
        obs_emb = embed_observe(params, sb['obs'], observe_names, observe_in_dims)
        steps = []
        for t in range(T):
            a, fam = sb['addresses'][t], sb['families'][t]
            cur_type = params['_layers_distribution_type_embedding.{}'.format(fam)]
            cur_addr = params['_layers_address_embedding.{}'.format(a)]
            if t == 0:
                smp = torch.zeros(B, sample_dim)
                prev_type, prev_addr = torch.zeros(type_dim), torch.zeros(addr_dim)
            else:
                pa, pf = sb['addresses'][t - 1], sb['families'][t - 1]
                smp = sample_embedding(params, pa, pf, sb['num_categories'][t - 1], sb['values'][t - 1])
                prev_type = params['_layers_distribution_type_embedding.{}'.format(pf)]
                prev_addr = params['_layers_address_embedding.{}'.format(pa)]
            shared = torch.cat([prev_type, prev_addr, cur_type, cur_addr]).expand(B, -1)
            steps.append(torch.cat([obs_emb, smp, shared], dim=1))
        out = lstm(torch.stack(steps), params)
        lps = []
        for t in range(T):
            lp = head_log_prob(params, sb['addresses'][t], sb['families'][t], sb['num_categories'][t], K, out[t],
                               sb['values'][t], sb['prior0'][t], sb['prior1'][t])
            if torch.isinf(lp).any() and not torch.isnan(lp).any():
                dead = lp == -float('inf')
                if repaired_rows == 'constant' and bool(dead.any()) and not bool(dead.all()):
                    keep = torch.nonzero(~dead).view(-1)
                    live = head_log_prob(params, sb['addresses'][t], sb['families'][t], sb['num_categories'][t], K,
                                         out[t][keep], sb['values'][t][keep], sb['prior0'][t][keep], sb['prior1'][t][keep])
                    lp = torch.full_like(lp, LOG_EPSILON).index_copy(0, keep, live)
                else:
                    lp = lp.clone()
                    lp[dead] = LOG_EPSILON   # util.replace_negative_inf
                    if repaired_rows == 'constant':
                        lp = lp.detach()
            lps.append(lp)
            total = total + (-lp.sum())
        all_lp.append(torch.stack(lps))
    return total / batch_size, all_lp


def loss_and_grads(params, sub_batches, observe_names, observe_in_dims, K, repaired_rows='reference'):
    p = {k: v.clone().float().requires_grad_(True) for k, v in params.items()}
    value, lps = loss(p, sub_batches, observe_names, observe_in_dims, K, repaired_rows=repaired_rows)
    value.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    return value.detach(), grads, [x.detach() for x in lps]


def head_params(params, address, family, K, h, prior0, prior1):
    """Proposal parameters a head returns at inference time (proposal_*.py forward, the same transforms as
    head_log_prob): mixtures -> (means, stddevs, probs) each [n, K]; Categorical -> probs [n, C]."""
    x = _ff(h, params, '_layers_proposal.{}._ff'.format(address), False)
    if family == 'Categorical':
        return (torch.softmax(x, dim=1) + 1e-8,)
    means, stddevs, coeffs = x[:, :K], x[:, K:2 * K], torch.softmax(x[:, 2 * K:], dim=1)
    p0 = torch.as_tensor(prior0, dtype=torch.float32).reshape(-1, 1)
    p1 = torch.as_tensor(prior1, dtype=torch.float32).reshape(-1, 1)
    if family == 'Normal':
        return p0 + means * p1, torch.exp(stddevs) * p1, coeffs
    if family == 'Uniform':
        rng = p1 - p0
        return p0 + torch.sigmoid(means) * rng, rng / 1000 + torch.sigmoid(stddevs) * rng * 10, coeffs
    if family == 'Poisson':
        return torch.sigmoid(means) * 40.0, torch.exp(stddevs), coeffs
    raise RuntimeError('unsupported family ' + family)


def infer_sequence(params, obs_row, observe_names, observe_in_dims, K, steps, n=1):
    """InferenceNetworkLSTM._infer_init + _infer_step replayed over one address sequence
    (pyprob/nn/inference_network.py:141-148, pyprob/nn/inference_network_lstm.py:82-134).

    steps: list of dicts {address, family, num_categories, prior0, prior1, prev_value} where prev_value is the value
    ([n] tensor) drawn at the PREVIOUS step (ignored at the first step).  All n particles share the observation.
    Returns one tuple of proposal parameters per step (see head_params)."""
    obs_emb = embed_observe(params, obs_row.reshape(1, -1).float(), observe_names, observe_in_dims).expand(n, -1)
    W_ih, W_hh = params['_layers_lstm.weight_ih_l0'], params['_layers_lstm.weight_hh_l0']
    b_ih, b_hh = params['_layers_lstm.bias_ih_l0'], params['_layers_lstm.bias_hh_l0']
    H = W_hh.size(1)
    h, c = torch.zeros(n, H), torch.zeros(n, H)
    smp_dim = _sample_dim(params)
    out = []
    for t, st in enumerate(steps):
        cur_t = params['_layers_distribution_type_embedding.' + st['family']]
        cur_a = params['_layers_address_embedding.' + st['address']]
        if t == 0:
            smp = torch.zeros(n, smp_dim)
            prev_t, prev_a = torch.zeros_like(cur_t), torch.zeros_like(cur_a)
        else:
            pv = steps[t - 1]
            smp = sample_embedding(params, pv['address'], pv['family'], pv['num_categories'],
                                   torch.as_tensor(st['prev_value'], dtype=torch.float32).reshape(-1))
            prev_t = params['_layers_distribution_type_embedding.' + pv['family']]
            prev_a = params['_layers_address_embedding.' + pv['address']]
        x = torch.cat([obs_emb, smp, torch.cat([prev_t, prev_a, cur_t, cur_a]).expand(n, -1)], dim=1)
        g = x @ W_ih.t() + b_ih + h @ W_hh.t() + b_hh
        i, f, gg, o = (torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H]), torch.tanh(g[:, 2 * H:3 * H]),
                       torch.sigmoid(g[:, 3 * H:]))
        c = f * c + i * gg
        h = o * torch.tanh(c)
        out.append(head_params(params, st['address'], st['family'], K, h, st['prior0'], st['prior1']))
    return out
