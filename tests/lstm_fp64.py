"""InferenceNetworkLSTM._loss restated in plain torch with autograd, at any dtype (TEST INFRASTRUCTURE ONLY).

The same computation as oracle/network.py (observe embedding, step-input assembly [obs_emb | smp_emb | prev type, prev
address, cur type, cur address], an explicit LSTM cell with h0 = c0 = 0 and gate order i, f, g, o, the proposal heads,
-sum log q / B), with two differences that let the CUDA kernels be held to more than the fp32 oracle's own rounding:

* `dtype` is a parameter.  At float64 every operation runs without fp32 rounding; the heads are those of tests/heads_fp64.py,
  which keep the reference's fp32 probability clamps whatever the dtype.  At float32 it is the oracle's arithmetic.
* It returns what a tolerance model needs: log q of every (t, row), and per step the LSTM input x, the gate pre-activations,
  the activations, c, h and d loss / d pre-activation (`dgates`, via retain_grad).  `lstm_term_magnitudes` turns them into
  M = sum over rows |dgates| |x|, the size of the terms each LSTM weight-gradient element sums.

A log q of -inf is replaced by log(1e-8) and its row contributes no gradient, as the CUDA training path does (the oracle's
repaired_rows='constant').  Bernoulli heads are included (tests/bernoulli_oracle.py restates the same head at fp32).
"""
import math

import torch

from oracle import network as onet
from tests import heads_fp64 as hf

LSTM_NAMES = ('_layers_lstm.weight_ih_l0', '_layers_lstm.weight_hh_l0', '_layers_lstm.bias_ih_l0', '_layers_lstm.bias_hh_l0')


def _sample_dim(params):
    return next(v.size(0) for k, v in params.items() if k.startswith('_layers_sample_embedding.') and k.endswith('.bias'))


def sample_embedding(params, address, family, num_categories, values):
    """values [n] (any dtype) -> relu(Linear(one-hot or value)) [n, S] at the dtype of the parameters."""
    dt = params['_layers_sample_embedding.{}._layers.0.bias'.format(address)].dtype
    if family == 'Categorical':
        x = torch.nn.functional.one_hot(torch.as_tensor(values).long(), num_categories).to(dt)
    else:
        x = torch.as_tensor(values).to(dt).view(-1, 1)
    return onet._ff(x, params, '_layers_sample_embedding.{}'.format(address), True)


def head_rows(family, x, values, prior0, prior1, K):
    """Raw head output x [n, out] -> log q [n] of every row, from the formulas of tests/heads_fp64.py."""
    v = values.to(x.dtype)
    p0, p1 = prior0.to(x.dtype).view(-1, 1), prior1.to(x.dtype).view(-1, 1)
    params = hf.proposal(family, x, K, p0, p1)
    if family == 'Categorical':
        probs = params[0] / params[0].sum(-1, keepdim=True)
        return torch.log(hf._clamp_probs(probs)).gather(1, v.long().view(-1, 1)).view(-1)
    if family == 'Bernoulli':
        pc = hf._clamp_probs(params[0].view(-1))
        logits = torch.log(pc) - torch.log1p(-pc)
        return -torch.nn.functional.binary_cross_entropy_with_logits(logits, v, reduction='none')
    means, stddevs, coeffs = params
    w = hf.window(family, p0, p1)
    vv = v.view(-1, 1)
    comp = hf._normal_lp(vv, means, stddevs) if w is None else hf._truncated_normal_lp(vv, means, stddevs, w[0], w[1])
    probs = coeffs / coeffs.sum(-1, keepdim=True)
    return torch.logsumexp(torch.log(hf._clamp_probs(probs)) + comp, dim=-1)


def _head_log_q(params, address, family, num_categories, K, h, values, prior0, prior1):
    def lq(rows):
        x = onet._ff(h[rows], params, '_layers_proposal.{}._ff'.format(address), False)
        return head_rows(family, x, values[rows], prior0[rows], prior1[rows], K)
    every = torch.arange(h.size(0))
    with torch.no_grad():
        dead = lq(every) == -math.inf
    if not bool(dead.any()):
        return lq(every)
    keep = torch.nonzero(~dead).view(-1)
    out = torch.full((h.size(0),), hf.LOG_EPSILON, dtype=h.dtype)
    return out.index_copy(0, keep, lq(keep)) if keep.numel() else out


def loss_and_grads(params, sub_batches, observe_names, observe_in_dims, K, dtype=torch.float64, addr_dim=64, type_dim=8,
                   embed=onet.embed_observe):
    """params: reference state_dict names -> tensors; sub_batches: dicts as synthetic.random_sub_batch makes (numpy or
    torch).  Returns {'loss', 'lps': per sub-batch [T, B] log q, 'grads': keyed like params, 'steps': per sub-batch a list
    over t of {'x', 'pre', 'act', 'c', 'h', 'dgates'}}, all detached, at `dtype`.  `embed` computes each sub-batch's
    observation embedding (signature of onet.embed_observe; tests/obs_fp64.py passes one that keeps every layer)."""
    p = {k: torch.as_tensor(v).detach().to(dtype).clone().requires_grad_(True) for k, v in params.items()}
    W_ih, W_hh = p['_layers_lstm.weight_ih_l0'], p['_layers_lstm.weight_hh_l0']
    b_ih, b_hh = p['_layers_lstm.bias_ih_l0'], p['_layers_lstm.bias_hh_l0']
    H, S = W_hh.size(1), _sample_dim(p)
    batch_size = sum(int(torch.as_tensor(sb['values']).shape[1]) for sb in sub_batches)
    total = torch.zeros((), dtype=dtype)
    lps, steps = [], []
    for sb in sub_batches:
        values, prior0, prior1 = (torch.as_tensor(sb[k]).to(dtype) for k in ('values', 'prior0', 'prior1'))
        T, B = values.shape
        obs_emb = embed(p, torch.as_tensor(sb['obs']).to(dtype), observe_names, observe_in_dims)
        h = torch.zeros(B, H, dtype=dtype)
        c = torch.zeros(B, H, dtype=dtype)
        sub_lp, sub_steps = [], []
        for t in range(T):
            a, fam, C = sb['addresses'][t], sb['families'][t], sb['num_categories'][t]
            cur = [p['_layers_distribution_type_embedding.' + fam], p['_layers_address_embedding.' + a]]
            if t == 0:
                smp = torch.zeros(B, S, dtype=dtype)
                prev = [torch.zeros(type_dim, dtype=dtype), torch.zeros(addr_dim, dtype=dtype)]
            else:
                pa, pf, pc = sb['addresses'][t - 1], sb['families'][t - 1], sb['num_categories'][t - 1]
                smp = sample_embedding(p, pa, pf, pc, values[t - 1])
                prev = [p['_layers_distribution_type_embedding.' + pf], p['_layers_address_embedding.' + pa]]
            x = torch.cat([obs_emb, smp, torch.cat(prev + cur).expand(B, -1)], dim=1)
            pre = x @ W_ih.t() + b_ih + h @ W_hh.t() + b_hh
            pre.retain_grad()
            act = torch.cat([torch.sigmoid(pre[:, :2 * H]), torch.tanh(pre[:, 2 * H:3 * H]), torch.sigmoid(pre[:, 3 * H:])], 1)
            c = act[:, H:2 * H] * c + act[:, :H] * act[:, 2 * H:3 * H]
            h = act[:, 3 * H:] * torch.tanh(c)
            sub_steps.append({'x': x, 'pre': pre, 'act': act, 'c': c, 'h': h})
            lp = _head_log_q(p, a, fam, C, K, h, values[t], prior0[t], prior1[t])
            sub_lp.append(lp)
            total = total - lp.sum()
        lps.append(torch.stack(sub_lp))
        steps.append(sub_steps)
    loss = total / batch_size
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in p.items()}
    steps = [[{'x': s['x'].detach(), 'pre': s['pre'].detach(), 'act': s['act'].detach(), 'c': s['c'].detach(),
               'h': s['h'].detach(),
               'dgates': s['pre'].grad if s['pre'].grad is not None else torch.zeros_like(s['pre'])} for s in sub]
             for sub in steps]
    return {'loss': loss.detach(), 'lps': [x.detach() for x in lps], 'grads': grads, 'steps': steps}


def lstm_term_magnitudes(result):
    """M for each LSTM parameter: the sum over every (t, row) of the absolute values of the terms its gradient adds up,
    |dgates| |x| for W_ih, |dgates_t| |h_{t-1}| for W_hh, |dgates| for both biases."""
    out = None
    for sub in result['steps']:
        for t, s in enumerate(sub):
            g = s['dgates'].abs()
            hp = sub[t - 1]['h'].abs() if t > 0 else torch.zeros(g.size(0), g.size(1) // 4, dtype=g.dtype)
            terms = (g.t() @ s['x'].abs(), g.t() @ hp, g.sum(0), g.sum(0))
            out = terms if out is None else tuple(a + b for a, b in zip(out, terms))
    return dict(zip(LSTM_NAMES, out))


def infer_steps(params, obs_row, observe_names, observe_in_dims, steps, n=1, dtype=torch.float64, addr_dim=64,
                type_dim=8):
    """InferenceNetworkLSTM._infer_init + _infer_step replayed over one address sequence: steps is a list of dicts
    {address, family, num_categories, prev_value} (prev_value: [n] values drawn at the previous step, unused at the
    first).  Returns (h, c) after each step, [n, H] each."""
    p = {k: torch.as_tensor(v).detach().to(dtype) for k, v in params.items()}
    W_ih, W_hh = p['_layers_lstm.weight_ih_l0'], p['_layers_lstm.weight_hh_l0']
    b_ih, b_hh = p['_layers_lstm.bias_ih_l0'], p['_layers_lstm.bias_hh_l0']
    H, S = W_hh.size(1), _sample_dim(p)
    obs_emb = onet.embed_observe(p, torch.as_tensor(obs_row).to(dtype).reshape(1, -1), observe_names,
                                 observe_in_dims).expand(n, -1)
    h, c = torch.zeros(n, H, dtype=dtype), torch.zeros(n, H, dtype=dtype)
    out = []
    for t, st in enumerate(steps):
        cur = [p['_layers_distribution_type_embedding.' + st['family']], p['_layers_address_embedding.' + st['address']]]
        if t == 0:
            smp = torch.zeros(n, S, dtype=dtype)
            prev = [torch.zeros(type_dim, dtype=dtype), torch.zeros(addr_dim, dtype=dtype)]
        else:
            pv = steps[t - 1]
            smp = sample_embedding(p, pv['address'], pv['family'], pv['num_categories'],
                                   torch.as_tensor(st['prev_value']).reshape(-1))
            prev = [p['_layers_distribution_type_embedding.' + pv['family']], p['_layers_address_embedding.' + pv['address']]]
        x = torch.cat([obs_emb, smp, torch.cat(prev + cur).expand(n, -1)], dim=1)
        g = x @ W_ih.t() + b_ih + h @ W_hh.t() + b_hh
        i, f, gg, o = (torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H]), torch.tanh(g[:, 2 * H:3 * H]),
                       torch.sigmoid(g[:, 3 * H:]))
        c = f * c + i * gg
        h = o * torch.tanh(c)
        out.append((h, c))
    return out
