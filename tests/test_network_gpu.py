"""GPU parity of the proposal-network training path (C-ABI ppb_ic_loss_forward/backward, ppb_adam_step_dev):
  (1) against the UNMODIFIED reference's loss and gradients on identical traces/weights (golden fixture),
  (2) against the oracle on seeded random networks/batches with ragged sub-batches and all four families,
  (3) size-independent properties at larger sizes (loss additivity over sub-batches, gradient linearity).
Tolerance: 1e-4 relative on losses / log-probs / gradients (north_star), index tensors exact."""
import numpy as np
import pytest
import torch

from oracle import network as onet
from pyprob_b200 import synthetic
from tests import netfixture

pytestmark = pytest.mark.gpu


def _net_from_fixture(fx, precision=0):
    obs_emb = {}
    for name in fx['observe_names']:
        # recover dim/depth from the parameter shapes
        depth = sum(1 for k in fx['params'] if k.startswith('_layers_observe_embedding.{}.'.format(name)) and k.endswith('weight'))
        dim = fx['params']['_layers_observe_embedding.{}._layers.{}.weight'.format(name, depth - 1)].shape[0]
        obs_emb[name] = {'dim': int(dim), 'depth': depth}
    fam_of = {}
    for sb in fx['subs']:
        for a, f, c in zip(sb['addresses'], sb['families'], sb['num_categories']):
            fam_of[a] = (f, c)
    # create types in the reference's insertion order so that type ids agree
    addresses = [(a, fam_of[a][0], fam_of[a][1]) for a in fx['address_order']]
    net = synthetic.build_network(obs_emb, fx['observe_in_dims'], addresses, lstm_dim=fx['lstm_dim'],
                                  mixture_components=fx['K'], precision=precision)
    net.load_reference_state_dict(fx['params'])
    return net


def _subs_numpy(subs):
    return [{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in sb.items()} for sb in subs]


def _check_grads(net, want, rtol=1e-4):
    for k, g in want.items():
        got = net.grad_view(k).cpu()
        scale = max(float(g.abs().max()), 1e-6)
        err = float((got - g).abs().max())
        assert err <= rtol * scale + 1e-7, (k, err, scale)


@pytest.mark.parametrize('tag', ['gum', 'mixed'])
@pytest.mark.parametrize('precision', [0, 2])
def test_loss_and_grads_vs_reference_fixture(cuda, tag, precision):
    fx = netfixture.load(tag)
    net = _net_from_fixture(fx, precision)
    batch = synthetic.ArrayBatch(_subs_numpy(fx['subs']))
    success, loss = net._loss(batch)
    assert success
    assert abs(float(loss.detach()) - fx['loss']) <= 1e-4 * abs(fx['loss'])
    loss.backward()
    _check_grads(net, fx['grads'])


def test_row_log_probs_vs_oracle(cuda):
    fx = netfixture.load('mixed')
    net = _net_from_fixture(fx)
    batch = synthetic.ArrayBatch(_subs_numpy(fx['subs']))
    enc, lp = net.row_log_probs(batch)
    lp = lp.cpu().numpy()
    _, _, ref = onet.loss_and_grads(fx['params'], fx['subs'], fx['observe_names'], fx['observe_in_dims'], fx['K'])
    a = enc.arrays
    for pos, s in enumerate(enc.sub_order):
        T, B = ref[s].shape
        for t in range(T):
            st = int(np.nonzero(a['step_t'] == t)[0][0]) + pos  # steps of one time index follow sub-batch order
            r0 = a['step_row0'][st]
            np.testing.assert_allclose(lp[r0:r0 + B], ref[s][t].numpy(), rtol=1e-4, atol=1e-5)


def _random_case(seed, lstm_dim, K, spec, precision=0):
    rng = np.random.default_rng(seed)
    table = [('a_u', 'Uniform', 0), ('a_c', 'Categorical', 5), ('a_n', 'Normal', 0), ('a_p', 'Poisson', 0),
             ('a_n2', 'Normal', 0), ('a_c2', 'Categorical', 3)]
    net = synthetic.build_network({'o0': {'dim': 12, 'depth': 2}, 'o1': {'dim': 6, 'depth': 3}}, [3, 1], table,
                                  lstm_dim=lstm_dim, mixture_components=K, seed=seed, precision=precision)
    subs = [synthetic.random_sub_batch(rng, [table[i] for i in seq], B, 4) for seq, B in spec]
    return net, subs


@pytest.mark.parametrize('seed,lstm_dim,K,spec', [
    (1, 32, 3, [([0, 1, 2], 5)]),
    (2, 32, 10, [([0, 1, 2, 3, 4, 5], 7), ([2], 1), ([0, 3], 64), ([1, 5, 4, 0], 3)]),
    (3, 64, 4, [([2, 4], 130), ([5, 1, 5, 1, 5, 1, 0], 33), ([3], 257)]),
])
@pytest.mark.parametrize('precision', [0, 2])
def test_loss_and_grads_vs_oracle_random(cuda, seed, lstm_dim, K, spec, precision):
    net, subs = _random_case(seed, lstm_dim, K, spec, precision)
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
    want_loss, want_grads, _ = onet.loss_and_grads(params, tsubs, ['o0', 'o1'], [3, 1], K)
    success, loss = net._loss(synthetic.ArrayBatch(subs))
    assert success
    assert abs(float(loss.detach()) - float(want_loss)) <= 1e-4 * abs(float(want_loss))
    loss.backward()
    _check_grads(net, want_grads)


def test_adam_step_vs_torch(cuda):
    """Optimizer.ADAM against torch.optim.Adam over the reference's parameter tensors, with .grad = None for the tensors the
    minibatch does not touch (GUM: the sample-embedding layer of its only address is never an input) — torch skips those:
    no weight decay, no moment update (inference_network.py:343-355 on torch >= 2.0)."""
    fx = netfixture.load('gum')
    net = _net_from_fixture(fx)
    batch = synthetic.ArrayBatch(_subs_numpy(fx['subs']))
    from pyprob_b200.util import Optimizer
    net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM, 1e-3, 1e-2
    net._create_optimizer()
    net._auto_skip_absent = True
    names = net._segment_names()
    ref = {k: net.view(k).clone().requires_grad_(True) for k in names}
    opt = torch.optim.Adam([ref[k] for k in names], lr=1e-3, weight_decay=1e-2)
    for _ in range(3):
        net._arena.grad = None
        ok, loss = net._loss(batch)
        loss.backward()
        present = net._segment_presence(net._last_enc, force=True)
        assert not present.all()
        for k, name in enumerate(names):
            ref[name].grad = net.grad_view(name).clone() if present[k] else None
        opt.step()
        net.optimizer_step()
    for name in names:
        torch.testing.assert_close(net.view(name), ref[name].data, rtol=1e-5, atol=1e-6, msg=lambda m, name=name: name + ': ' + m)


def test_flat_adam_step_dev_vs_torch_on_the_whole_arena(cuda):
    """The flat kernel itself (ppb_adam_step_dev): every element updated, as torch.optim.Adam on one tensor."""
    from pyprob_b200._lib import call, ptr, stream
    gen = torch.Generator().manual_seed(0)
    n = 100003
    p = torch.randn(n, generator=gen).to(cuda)
    ref_p = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([ref_p], lr=1e-3, weight_decay=1e-2)
    m, v = torch.zeros(n, device=cuda), torch.zeros(n, device=cuda)
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 1e-2, 1.0], device=cuda)
    state = torch.zeros(2, dtype=torch.int64, device=cuda)
    for step in range(1, 4):
        g = torch.randn(n, generator=gen).to(cuda)
        ref_p.grad = g.clone()
        opt.step()
        call('ppb_adam_step_dev', ptr(p), ptr(g), ptr(m), ptr(v), n, ptr(hyper), ptr(state), stream())
    assert int(state[0]) == 3
    torch.testing.assert_close(p, ref_p.data, rtol=1e-5, atol=1e-6)


def test_loss_is_additive_over_sub_batches_and_grad_scales(cuda):
    """Size-independent properties at a larger size: loss(batch) * B == sum_s loss(sub s) * B_s, and the
    gradient is linear in the upstream gradient."""
    net, subs = _random_case(7, 128, 10, [([0, 1, 2, 3], 300), ([2, 4, 5], 211), ([1], 77)])
    full = synthetic.ArrayBatch(subs)
    _, loss = net._loss(full)
    net._arena.grad = None
    loss.backward()
    g1 = net._arena.grad.clone()
    net._arena.grad = None
    _, loss2 = net._loss(full)
    (loss2 * 3.0).backward()
    parts = 0.0
    for sb in subs:
        b = synthetic.ArrayBatch([sb])
        with torch.no_grad():
            _, l = net._loss(b)
        parts += float(l) * b.size
    assert abs(float(loss.detach()) * full.size - parts) <= 2e-5 * abs(parts)
    with pytest.raises(RuntimeError):
        loss2.backward()  # stale: other batches went through the shared workspace since
    # (a few reductions use atomics: summation order varies run to run)
    torch.testing.assert_close(net._arena.grad, g1 * 3.0, rtol=1e-4, atol=3e-5 * float(g1.abs().max()))


def test_infer_step_tensor_core_vs_simt_and_oracle(cuda):
    """Batched proposal step (ppb_ic_infer_step): the tensor-core path, the fp32 SIMT path and the oracle's
    layer-by-layer restatement of _infer_step (inference_network_lstm.py:82-134) give the same proposal parameters."""
    fx = netfixture.load('mixed')
    n = 300
    gen = torch.Generator().manual_seed(3)
    obs = {name: torch.randn(d, generator=gen) for name, d in zip(fx['observe_names'], fx['observe_in_dims'])}
    sb = fx['subs'][0]
    seq = list(zip(sb['addresses'], sb['families'], sb['num_categories']))
    vals = []
    for a, fam, C in seq:
        if fam == 'Categorical':
            vals.append(torch.randint(0, C, (n,), generator=gen).float())
        elif fam == 'Poisson':
            vals.append(torch.poisson(torch.full((n,), 3.0), generator=gen))
        else:
            vals.append(torch.rand(n, generator=gen) * 1.5 - 0.5)
    outs = {}
    for precision in (0, 2):
        net = _net_from_fixture(fx, precision)
        net._infer_init(obs)
        prev_a, prev_v, res = None, None, []
        for (a, fam, C), v in zip(seq, vals):
            p0 = {'Normal': 0.3, 'Uniform': -1.0}.get(fam)
            p1 = {'Normal': 0.5, 'Uniform': 2.0}.get(fam)
            params = net._infer_step_batched(a, prev_a, prev_v, p0, p1, n)
            res.append(params.cpu())
            prev_a, prev_v = a, v.to(cuda)
        outs[precision] = res
    for a, b in zip(outs[0], outs[2]):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-5)
    # oracle: step the reference-equivalent network for one particle path (all particles share the observation)
    P = fx['params']
    obs_row = torch.cat([obs[nm].reshape(-1) for nm in fx['observe_names']]).view(1, -1)
    obs_emb = onet.embed_observe(P, obs_row, fx['observe_names'], fx['observe_in_dims']).expand(n, -1)
    H, K = fx['lstm_dim'], fx['K']
    h = torch.zeros(n, H)
    c = torch.zeros(n, H)
    for t, ((a, fam, C), v) in enumerate(zip(seq, vals)):
        cur_t, cur_a = P['_layers_distribution_type_embedding.' + fam], P['_layers_address_embedding.' + a]
        if t == 0:
            smp, pt, pa = torch.zeros(n, 4), torch.zeros(8), torch.zeros(64)
        else:
            pa_, pf, pc = seq[t - 1]
            smp = onet.sample_embedding(P, pa_, pf, pc, vals[t - 1])
            pt, pa = P['_layers_distribution_type_embedding.' + pf], P['_layers_address_embedding.' + pa_]
        x = torch.cat([obs_emb, smp, torch.cat([pt, pa, cur_t, cur_a]).expand(n, -1)], dim=1)
        g = x @ P['_layers_lstm.weight_ih_l0'].t() + P['_layers_lstm.bias_ih_l0'] + h @ P['_layers_lstm.weight_hh_l0'].t() \
            + P['_layers_lstm.bias_hh_l0']
        i, f, gg, o = torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H]), torch.tanh(g[:, 2 * H:3 * H]), torch.sigmoid(g[:, 3 * H:])
        c = f * c + i * gg
        h = o * torch.tanh(c)
        raw = onet._ff(h, P, '_layers_proposal.{}._ff'.format(a), False)
        got = outs[0][t]
        if fam == 'Categorical':
            want = torch.softmax(raw, dim=1) + 1e-8
        else:
            coeffs = torch.softmax(raw[:, 2 * K:], dim=1)
            if fam == 'Normal':
                means, sds = 0.3 + raw[:, :K] * 0.5, torch.exp(raw[:, K:2 * K]) * 0.5
            elif fam == 'Uniform':
                means = -1.0 + torch.sigmoid(raw[:, :K]) * 3.0
                sds = 3.0 / 1000 + torch.sigmoid(raw[:, K:2 * K]) * 3.0 * 10
            else:
                means, sds = torch.sigmoid(raw[:, :K]) * 40.0, torch.exp(raw[:, K:2 * K])
            want = torch.cat([means, sds, coeffs], dim=1)
        torch.testing.assert_close(got, want, rtol=2e-4, atol=1e-5)
