"""The feed-forward inference network (InferenceNetworkFeedForward, pyprob/nn/inference_network_feedforward.py) against its
oracle (tests/ff_oracle.py): loss, per-row log q and every parameter gradient on the tensor cores (precisions 0 and 1) and
on the fp32 path (precision 2), for every proposal family, ragged sub-batches in which one address sits at different t,
T = 1 where the NLL runs in the h2 cluster epilogue, a batch large enough for k_head_nll, and T = 50 where the d obs_emb
GEMM reduces over 50 segments; the one-row infer step; training through the public API with the default network type;
save / load; the graph-replayed host step; the optimiser with an address absent from a minibatch."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import pyprob_b200 as pyprob
from pyprob_b200 import InferenceEngine, InferenceNetwork, Model, synthetic
from pyprob_b200._lib import call, ptr
from pyprob_b200.distributions import Normal
from pyprob_b200.network import InferenceNetwork as InferenceNetworkBase
from pyprob_b200.network import InferenceNetworkFeedForward
from pyprob_b200.util import Optimizer
from tests import ff_oracle

from oracle import network as onet
from oracle import optim as ooptim
from oracle import scoring

pytestmark = pytest.mark.gpu

FF = InferenceNetwork.FEEDFORWARD
TABLE = [('t_n', 'Normal', 0), ('t_u', 'Uniform', 0), ('t_p', 'Poisson', 0), ('t_c', 'Categorical', 5),
         ('t_b', 'Bernoulli', 0)]
OBS, IN_DIMS, K = ['o0', 'o1'], [3, 1], 4
EMB = {'o0': {'dim': 12, 'depth': 2}, 'o1': {'dim': 6, 'depth': 1}}
TOL = {0: (1e-4, 1e-4), 1: (2e-3, 5e-2), 2: (1e-4, 1e-4)}
ATOL = {0: 1e-7, 1: 1e-6, 2: 1e-7}


def _net(precision, seed=0):
    return synthetic.build_network(EMB, IN_DIMS, TABLE, mixture_components=K, seed=seed, precision=precision,
                                   inference_network=FF)


def _seq_sub(rng, order, B, obs_dim=4):
    return synthetic.random_sub_batch(rng, [TABLE[i] for i in order], B, obs_dim)


def _oracle(net, subs, names=OBS, dims=IN_DIMS, k=K):
    params = {k_: v.cpu() for k_, v in net.reference_state_dict().items()}
    tsubs = [{k_: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k_, v in sb.items()} for sb in subs]
    return ff_oracle.loss_and_grads(params, tsubs, names, dims, k)


def _check(net, subs, precision, names=OBS, dims=IN_DIMS, k=K, rel=None):
    ltol, gtol = TOL[precision]
    gtol = rel if rel is not None else gtol
    want_loss, want_grads, want_lps = _oracle(net, subs, names, dims, k)
    net._arena.grad = None
    ok, loss = net._loss(synthetic.ArrayBatch(subs))
    assert ok
    assert abs(float(loss.detach()) - float(want_loss)) <= ltol * abs(float(want_loss))
    loss.backward()
    assert set(want_grads) == set(net.parameter_index)
    for key, g in want_grads.items():
        got = net.grad_view(key).cpu()
        scale = max(float(g.abs().max()), 1e-6)
        err = float((got - g).abs().max())
        assert err <= gtol * scale + ATOL[precision], (key, err, scale)
    enc, lp = net.row_log_probs(synthetic.ArrayBatch(subs))
    lp = lp.cpu().numpy()
    step = 0
    for t in range(enc.t_max):   # steps are time-major; the sub-batches active at t come first
        for s, sb in enumerate(subs):
            if sb['values'].shape[0] <= t:
                continue
            r0, B = int(enc.arrays['step_row0'][step]), sb['values'].shape[1]
            np.testing.assert_allclose(lp[r0:r0 + B], want_lps[s][t].numpy(), rtol=10 * ltol, atol=10 * ltol)
            step += 1


def test_parameter_names_and_shapes():
    """The reference's layout: E = 12 + 6 = 18; hidden = int((E + out) / 2)."""
    net = _net(0)
    idx = net.parameter_index
    assert idx['_layers_proposal.t_n._ff._layers.0.weight'][1] == (int((18 + 12) / 2), 18)
    assert idx['_layers_proposal.t_n._ff._layers.1.weight'][1] == (12, 15)
    assert idx['_layers_proposal.t_b._ff._layers.0.weight'][1] == (9, 18)
    assert idx['_layers_proposal.t_b._ff._layers.1.weight'][1] == (1, 9)
    assert not any(k.startswith(('_layers_lstm', '_layers_address_embedding', '_layers_sample_embedding',
                                 '_layers_distribution_type_embedding')) for k in idx)


@pytest.mark.parametrize('precision', [0, 1, 2])
def test_ragged_every_family_vs_oracle(cuda, precision):
    """Three sub-batches (300 / 200 / 101 traces) of different lengths; t_c sits at t = 0, 1 and 2."""
    rng = np.random.default_rng(1)
    subs = [_seq_sub(rng, [3, 0, 4], 300), _seq_sub(rng, [1, 3], 200), _seq_sub(rng, [2, 4, 3], 101)]
    subs.sort(key=lambda sb: -sb['values'].shape[0])
    _check(_net(precision, seed=1), subs, precision)


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('family', range(len(TABLE)))
def test_t1_b256_every_family_vs_oracle(cuda, precision, family):
    """T = 1, B = 256: on the tensor cores the h2 phase runs as a cluster with the NLL in its epilogue."""
    _check(_net(precision, seed=family), [_seq_sub(np.random.default_rng(10 + family), [family], 256)], precision)


@pytest.mark.parametrize('precision', [0, 1])
def test_gum_b256_vs_oracle(cuda, precision):
    net = synthetic.gum_network(precision=precision, seed=2, inference_network=FF)
    sb = synthetic.gum_batch(np.random.default_rng(2), 256).subs
    _check(net, sb, precision, names=['obs0', 'obs1'], dims=[1, 1], k=10)


def test_gum_large_batch_runs_k_head_nll(cuda):
    """9000 traces: 71 row tiles, too many for a cluster h2 phase, so k_head_nll computes the NLL."""
    net = synthetic.gum_network(precision=0, seed=3, inference_network=FF)
    sb = synthetic.gum_batch(np.random.default_rng(3), 9000).subs
    # the bias gradients are sums over 9000 traces that cancel to ~1e-3 of their terms: fp32 summation order shows at 2e-4
    _check(net, sb, 0, names=['obs0', 'obs1'], dims=[1, 1], k=10, rel=1e-3)


@pytest.mark.parametrize('precision', [0, 2])
def test_synthetic50_t50_vs_oracle(cuda, precision):
    """T = 50, E = 256, B = 512: the d obs_emb GEMM reduces over 50 segments; the observation-layer gradients check it.

    Every gradient is held to 1e-4 of its maximum, plus — elementwise — what the first-layer head units whose pre-activation
    lies within rounding of zero can move it by when they take the other side of their ReLU (ff_oracle.relu_flip_bound).
    Without that allowance a few such units of 3.6 M put two heads' W1 off by 1.4 % of their maximum at precision 0; the
    allowance covers those units only, so a lost or misplaced segment of the d obs_emb sum still fails."""
    net = synthetic.synthetic50_network(precision=precision, seed=4, inference_network=FF)
    subs = synthetic.synthetic50_batch(np.random.default_rng(4), 512).subs
    want_loss, want_grads, _ = _oracle(net, subs, ['obs'], [1], 10)
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
    bound, flips = ff_oracle.relu_flip_bound(params, tsubs, ['obs'], [1], 10)
    assert flips < 1e-3 * 512 * 50 * 130, flips    # a few hundred of the 3.6 M hidden units
    net._arena.grad = None
    ok, loss = net._loss(synthetic.ArrayBatch(subs))
    assert ok and abs(float(loss.detach()) - float(want_loss)) <= 1e-4 * abs(float(want_loss))
    loss.backward()
    for key, g in want_grads.items():
        got = net.grad_view(key).cpu()
        scale = max(float(g.abs().max()), 1e-6)
        excess = ((got - g).abs() - 1e-4 * scale - 1e-7 - bound[key]).max()
        assert float(excess) <= 0, (key, float((got - g).abs().max()), scale, float(bound[key].max()))


def test_synthetic50_t50_tf32_vs_oracle(cuda):
    """Precision 1 at T = 50: tf32 rounding of cancelling weight-gradient sums, up to 13 % of a head's W1 maximum (as in
    test_t1_chain_gpu); the observation layers, which the d obs_emb GEMM feeds, stay within 5 %."""
    net = synthetic.synthetic50_network(precision=1, seed=4, inference_network=FF)
    sb = synthetic.synthetic50_batch(np.random.default_rng(4), 512).subs
    _check(net, sb, 1, names=['obs'], dims=[1], k=10, rel=0.25)


def test_forward_only_and_negative_inf_repair(cuda):
    net = _net(0, seed=5)
    sb = _seq_sub(np.random.default_rng(5), [1, 0], 256)
    sb['values'][0, 3] = sb['prior1'][0, 3] + 0.5      # Uniform value outside [low, high]: log q = -inf -> log(1e-8)
    want_loss, _, want_lps = _oracle(net, [sb])
    with torch.no_grad():
        ok, loss = net._loss(synthetic.ArrayBatch([sb]))
    assert ok and abs(float(loss) - float(want_loss)) <= 1e-4 * abs(float(want_loss))
    assert float(want_lps[0][0, 3]) == pytest.approx(math.log(1e-8))
    _check(net, [sb], 0)


@pytest.mark.parametrize('precision', [0, 2])
def test_infer_step_one_head_row_vs_oracle(cuda, precision):
    """Every particle at an address gets the head output of the one shared observation, with its own prior."""
    net = _net(precision, seed=6)
    obs = {'o0': [0.3, -1.2, 0.5], 'o1': 0.7}
    net._infer_init(obs)
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    row = torch.tensor([0.3, -1.2, 0.5, 0.7])
    n = 1000
    rng = np.random.default_rng(6)
    for addr, fam, _ in TABLE:
        p0 = p1 = None
        if fam == 'Normal':
            p0, p1 = torch.from_numpy(rng.normal(0, 1, n).astype(np.float32)), torch.from_numpy(rng.uniform(0.5, 2, n).astype(np.float32))
        elif fam == 'Uniform':
            p0 = torch.from_numpy(rng.uniform(-2, 0, n).astype(np.float32))
            p1 = p0 + 2.0
        got = net._infer_step_batched(addr, 't_n', torch.zeros(n, device=cuda), None if p0 is None else p0.to(cuda),
                                      None if p1 is None else p1.to(cuda), n).cpu()
        want = ff_oracle.infer_step(params, row, OBS, IN_DIMS, K, addr, fam,
                                    0.0 if p0 is None else p0, 0.0 if p1 is None else p1, n=n)
        want = torch.cat([w.reshape(n, -1) for w in want], dim=1)
        np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-4, atol=1e-5)
    assert net._infer_step_batched('unknown', None, None, None, None, n) is None


class GaussianUnknownMean(Model):
    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


def test_learn_inference_network_default_is_feedforward(cuda, tmp_path):
    """The reference's default network type trains, its IC posterior is sane, and save -> load -> continue works."""
    pyprob.seed(7)
    pyprob.set_verbosity(0)
    model = GaussianUnknownMean()
    model.learn_inference_network(num_traces=20000, batch_size=256,
                                  observe_embeddings={'obs0': {'dim': 32}, 'obs1': {'dim': 32}})
    net = model._inference_network
    assert isinstance(net, InferenceNetworkFeedForward)
    assert net._total_train_traces >= 20000 and net._loss_min < net._loss_init
    post = model.posterior_results(4096, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                   observe={'obs0': 8, 'obs1': 9})
    assert abs(float(post.mean) - 7.25) < 0.3
    fn = str(tmp_path / 'ff.network')
    model.save_inference_network(fn)
    model2 = GaussianUnknownMean()
    model2.load_inference_network(fn)
    net2 = model2._inference_network
    assert type(net2) is InferenceNetworkFeedForward
    assert torch.equal(net2._arena.data, net._arena.data)
    for m, nn_ in ((model, net), (model2, net2)):
        nn_._infer_init({'obs0': 8.0, 'obs1': 9.0})
    a = net._infer_step_batched('98__forward__mu__Normal__1', None, None, 1.0, math.sqrt(5), 4)
    b = net2._infer_step_batched('98__forward__mu__Normal__1', None, None, 1.0, math.sqrt(5), 4)
    assert torch.equal(a, b)
    model2.learn_inference_network(num_traces=512, batch_size=256,
                                   observe_embeddings={'obs0': {'dim': 32}, 'obs1': {'dim': 32}})
    assert net2._total_train_traces >= net._total_train_traces + 512


def test_adam_skips_absent_address_like_torch_optim(cuda):
    """Two Adam steps; the second minibatch lacks t_u, whose proposal layer then keeps its parameters and moments."""
    net = _net(0, seed=8)
    net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM, 1e-2, 0.0
    net._create_optimizer()
    rng = np.random.default_rng(8)
    b1 = [_seq_sub(rng, [1, 0], 256)]
    b2 = [_seq_sub(rng, [0, 3], 256)]
    params = {k: v.cpu().clone().requires_grad_(True) for k, v in net.reference_state_dict().items()}
    opt = torch.optim.Adam(params.values(), lr=1e-2)
    for subs in (b1, b2):
        net._arena.grad = None
        ok, loss = net._loss(synthetic.ArrayBatch(subs))
        assert ok
        loss.backward()
        net.optimizer_step()
        opt.zero_grad(set_to_none=True)   # a tensor outside this minibatch's graph keeps .grad None and is skipped
        tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
        want, _ = ff_oracle.loss(params, tsubs, OBS, IN_DIMS, K)
        want.backward()
        opt.step()
    for k, p in params.items():
        got = net.view(k).cpu()
        np.testing.assert_allclose(got.numpy(), p.detach().numpy(), rtol=1e-4, atol=1e-5, err_msg=k)


def test_host_step_eager_and_graph_agree(cuda):
    """ppb_ic_train_step_host on a feed-forward net: the eager first call and the graph replays give the parameters of
    an eager run of the same steps."""
    from pyprob_b200.network import BatchStruct  # noqa: F401
    results = []
    for graph in (False, True):
        net = synthetic.gum_network(precision=0, seed=9, inference_network=FF)
        net._sync_native()
        enc = synthetic.gum_batch(np.random.default_rng(9), 256).encode(net)
        grad = torch.zeros_like(net._arena.data)
        m, v = torch.zeros_like(grad), torch.zeros_like(grad)
        img = enc.pack().copy()
        dimg = torch.empty(img.nbytes, dtype=torch.uint8, device=cuda)
        need = net._ensure_workspace(enc)
        ws = torch.empty(need + 1024, dtype=torch.uint8, device=cuda)
        loss, status = C.c_float(), C.c_int32()
        losses = []
        for step in range(1, 4):
            if not graph:
                call('ppb_net_destroy', net._handle)   # a fresh handle: no cached graph
                net._handle = None
                net._sync_native()
            call('ppb_ic_train_step_host', net._handle, ptr(net._arena.data), ptr(grad), ptr(m), ptr(v), net._arena.numel(),
                 img.ctypes.data, img.nbytes, ptr(dimg), ptr(ws), ws.numel(), 0, 1e-3, 0.9, 0.999, 1e-8, 0.0, step,
                 C.byref(loss), C.byref(status), torch.cuda.current_stream().cuda_stream)
            assert status.value == 0
            losses.append(loss.value)
        results.append((losses, net._arena.data.clone()))
    np.testing.assert_allclose(results[0][0], results[1][0], rtol=1e-6)
    torch.testing.assert_close(results[0][1], results[1][1], rtol=1e-5, atol=1e-7)


def test_load_returns_saved_class(cuda, tmp_path):
    net = _net(0, seed=10)
    fn = str(tmp_path / 'x.network')
    net._save(fn)
    loaded = InferenceNetworkBase._load(fn)
    assert type(loaded) is InferenceNetworkFeedForward
    assert torch.equal(loaded._arena.data, net._arena.data)


@pytest.mark.parametrize('precision', [0, 1, 2])
def test_reference_fixture_parity(cuda, precision):
    """ff_golden.npz, written by the unmodified reference: the network's parameter layout, then — after
    load_reference_state_dict — the loss, per-row log q and every gradient (five families, two trace types, observables of
    depth 2 and 1)."""
    fx = ff_oracle.load_fixture()
    depth = {n: sum(1 for k in fx['params'] if k.startswith('_layers_observe_embedding.{}.'.format(n)) and k.endswith('.weight'))
             for n in fx['observe_names']}
    emb = {n: {'dim': int(fx['params']['_layers_observe_embedding.{}._layers.{}.weight'.format(n, d - 1)].shape[0]),
               'depth': d} for n, d in depth.items()}
    net = synthetic.build_network(emb, fx['observe_in_dims'], ff_oracle.address_table(fx), mixture_components=fx['K'],
                                  precision=precision, inference_network=FF)
    assert {k: tuple(v) for k, (_, v) in net.parameter_index.items()} == {k: tuple(v.shape) for k, v in fx['params'].items()}
    net.load_reference_state_dict(fx['params'])
    ltol, gtol = TOL[precision]
    net._arena.grad = None
    ok, loss = net._loss(synthetic.ArrayBatch(fx['subs']))
    assert ok and abs(float(loss.detach()) - fx['loss']) <= ltol * abs(fx['loss'])
    loss.backward()
    for k, g in fx['grads'].items():
        scale = max(float(g.abs().max()), 1e-6)
        assert float((net.grad_view(k).cpu() - g).abs().max()) <= gtol * scale + ATOL[precision], k
    _, _, want_lps = ff_oracle.loss_and_grads(fx['params'], fx['subs'], fx['observe_names'], fx['observe_in_dims'], fx['K'])
    enc, lp = net.row_log_probs(synthetic.ArrayBatch(fx['subs']))
    lp = lp.cpu().numpy()
    for st in range(enc.n_steps):
        s, t = st % len(fx['subs']), st // len(fx['subs'])     # both trace types have four controlled sites
        r0, B = int(enc.arrays['step_row0'][st]), fx['subs'][s]['values'].shape[1]
        np.testing.assert_allclose(lp[r0:r0 + B], want_lps[s][t].numpy(), rtol=10 * ltol, atol=10 * ltol)
    # _infer_step proposals of the reference at every address
    for tr in fx['infer']:
        net._infer_init({n: tr['obs'][i] for i, n in enumerate(fx['observe_names'])})
        for step in tr['steps']:
            got = net._infer_step_batched(step['address'], None, None, step['prior0'], step['prior1'], 3).cpu()
            want = np.concatenate([np.asarray(w).reshape(-1) for w in step['proposal']])
            for row in got.numpy():
                np.testing.assert_allclose(row, want, rtol=1e-4, atol=1e-6)


def test_infer_step_runs_one_head_row(cuda, tmp_path):
    """Whatever n, the head GEMMs of a feed-forward infer step cover one row: each is a single 64 x 64 tile."""
    from torch.profiler import ProfilerActivity, profile
    import json
    net = _net(0, seed=11)
    net._infer_init({'o0': [0.1, 0.2, 0.3], 'o1': 0.4})
    net._infer_step_batched('t_n', None, None, 0.0, 1.0, 50000)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        net._infer_step_batched('t_n', None, None, torch.zeros(50000, device=cuda), torch.ones(50000, device=cuda), 50000)
        torch.cuda.synchronize()
    path = str(tmp_path / 'trace.json')
    prof.export_chrome_trace(path)
    events = [e for e in json.load(open(path))['traceEvents'] if e.get('cat') == 'kernel']
    gemms = [e for e in events if 'k_grouped' in e['name']]
    assert len(gemms) == 2, [e['name'] for e in events]
    assert all(e['args']['grid'] == [1, 1, 1] for e in gemms), [e['args']['grid'] for e in gemms]
    assert any('k_head_params' in e['name'] and e['args']['grid'][0] > 1 for e in events)


def test_unknown_previous_address_still_gets_the_proposal(cuda):
    """The previous site plays no part (inference_network_feedforward.py:53-66): a lane that comes from an address the
    network does not know gets the proposal of the known current address."""
    net = _net(0, seed=12)
    net._infer_init({'o0': [0.1, 0.2, 0.3], 'o1': 0.4})
    a = net._infer_step_batched('t_u', 'never-seen', torch.zeros(8, device=cuda), -1.0, 2.0, 8)
    b = net._infer_step_batched('t_u', None, None, -1.0, 2.0, 8)
    assert a is not None and torch.equal(a, b)


class GaussianUnknownMeanMarsaglia(Model):
    def marsaglia(self, mean, stddev):
        def body(s):
            x = pyprob.sample(pyprob.distributions.Uniform(-1, 1))
            y = pyprob.sample(pyprob.distributions.Uniform(-1, 1))
            return {'x': x, 'y': y, 's': x * x + y * y}
        st = pyprob.while_loop(lambda s: s['s'] >= 1, body, {'x': 0.0, 'y': 0.0, 's': 2.0})
        x, s = st['x'], st['s']
        return mean + stddev * (x * torch.sqrt(-2 * torch.log(s) / s))

    def forward(self):
        mu = self.marsaglia(1, math.sqrt(5))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


@pytest.mark.parametrize('model_class', [GaussianUnknownMean, GaussianUnknownMeanMarsaglia])
def test_ic_log_weights_vs_oracle(cuda, model_class):
    """IC log-weights particle by particle: sum over each particle's executed sites of log p(v) - log q(v), q from the
    oracle's feed-forward proposals, plus the two observe terms.  Marsaglia's while_loop masks lanes, which proposes for the
    executing lanes only."""
    from unittest import mock
    from pyprob_b200.util import TraceMode
    from tests.ic_replay import site_weight_terms
    pyprob.seed(13)
    pyprob.set_verbosity(0)
    model = model_class()
    model.learn_inference_network(num_traces=4 * 256, batch_size=256,
                                  observe_embeddings={'obs0': {'dim': 16}, 'obs1': {'dim': 16}})
    net = model._inference_network
    assert isinstance(net, InferenceNetworkFeedForward)
    n = 2000
    with torch.no_grad():
        trace = model._run_batched(n, trace_mode=TraceMode.POSTERIOR,
                                   inference_engine=InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                   inference_network=net, observe={'obs0': 8.0, 'obs1': 9.0})
    with mock.patch.object(onet, 'infer_sequence', ff_oracle.infer_sequence):
        want, covered = site_weight_terms(trace, net, torch.tensor([8.0, 9.0]))
    # Marsaglia: a particle whose loop runs longer than any training trace meets addresses the network does not know (the
    # prior proposes there); the replay covers the others
    assert covered.all() if model_class is GaussianUnknownMean else covered.mean() > 0.9
    mu = trace.result.cpu()
    for y in (8.0, 9.0):
        want = want + scoring.normal_log_prob(torch.tensor(y), mu, torch.tensor(math.sqrt(2))).double().numpy()
    np.testing.assert_allclose(trace.log_w.cpu().numpy()[covered], want[covered], rtol=1e-4, atol=2e-4)
    if model_class is GaussianUnknownMeanMarsaglia:
        masks = [s.mask for s in trace.variables_controlled if s.mask is not None]
        assert masks and any(0 < float(m.float().mean()) < 1 for m in masks)


def test_adam_larc_with_an_absent_address_vs_oracle(cuda):
    """ADAM_LARC through the segment-aware step: proposal layers of addresses outside a minibatch are skipped like
    .grad None (the observation layers are always present)."""
    net = _net(0, seed=14)
    net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM_LARC, 1e-2, 1e-5
    net._create_optimizer()
    net._skip_absent_gradients = True   # the reference on torch >= 2.0: zero_grad() leaves absent tensors at .grad None
    names = net._segment_names()
    segs = [(net.parameter_index[k][0], int(np.prod(net.parameter_index[k][1]))) for k in names]
    p = net._arena.data.cpu().clone()
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    steps = torch.zeros(len(names), dtype=torch.int64)
    rng = np.random.default_rng(14)
    for order in ([1, 0], [0, 3], [1, 3, 4]):
        net._arena.grad = None
        ok, loss = net._loss(synthetic.ArrayBatch([_seq_sub(rng, order, 256)]))
        assert ok
        loss.backward()
        present = net._segment_presence(net._last_enc, force=True).astype(bool)
        for k, name in enumerate(names):
            assert present[k] == (not name.startswith('_layers_proposal.') or
                                  any(name.startswith('_layers_proposal.{}.'.format(TABLE[i][0])) for i in order)), name
        g = net._arena.grad.cpu().clone()
        ooptim.larc_adjust(p, g, present, segs, 1e-2, 1e-5)
        ooptim.adam_step(p, g, m, v, steps, present, segs, 1e-2, weight_decay=0.0)
        net.optimizer_step()
        torch.testing.assert_close(net._arena.data.cpu(), p, rtol=2e-5, atol=2e-6)


def test_train_from_offline_dataset_dir(cuda, tmp_path):
    pyprob.seed(15)
    pyprob.set_verbosity(0)
    model = GaussianUnknownMean()
    model.save_dataset(str(tmp_path / 'train'), num_traces=2048, num_traces_per_file=512)
    model.learn_inference_network(num_traces=256 * 30, dataset_dir=str(tmp_path / 'train'), batch_size=256,
                                  observe_embeddings={'obs0': {'dim': 16}, 'obs1': {'dim': 16}}, learning_rate_init=1e-3)
    net = model._inference_network
    assert isinstance(net, InferenceNetworkFeedForward)
    hist = net._history_train_loss
    assert len(hist) == 30 and np.all(np.isfinite(hist)) and np.mean(hist[-5:]) < np.mean(hist[:5])


def _peer_worker(rank, world, port):
    """One feed-forward training step through PeerAdam (fused reduce-scatter + Adam + all-gather over NVLink) against NCCL
    all-reduce followed by Adam on the same per-rank gradients."""
    import os
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    net = synthetic.gum_network(seed=0, inference_network=FF)
    net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM, 1e-3, 0.0
    net._create_optimizer()
    net._learning_rate = 1e-3
    dist.broadcast(net._arena.data, 0)
    p0 = net._arena.data.clone()
    net._arena.grad = None
    ok, loss = net._loss(synthetic.gum_batch(np.random.default_rng(100 + rank), 256))
    assert ok
    loss.backward()
    g = net._arena.grad.clone()
    summed = g.clone()
    dist.all_reduce(summed)
    want = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([want], lr=1e-3)
    want.grad = summed / world
    opt.step()
    net._enable_peer_optimizer()
    net._arena.grad = g
    net._peer_optimizer_step(loss.detach(), world)
    torch.cuda.synchronize()
    if world == 2:      # a two-term sum has one order
        assert torch.equal(net._arena.data, want.data)
    else:
        torch.testing.assert_close(net._arena.data, want.data, rtol=1e-5, atol=1e-7)
    dist.barrier()
    torch.cuda.synchronize()
    os._exit(0)


def test_peer_adam_step_matches_allreduce_adam():
    world = min(torch.cuda.device_count(), 8)
    if world < 2:
        pytest.skip('needs at least two GPUs on one NVLink node')
    import socket
    import torch.multiprocessing as mp
    with socket.socket() as sk:
        sk.bind(('127.0.0.1', 0))
        port = sk.getsockname()[1]
    procs = [mp.get_context('spawn').Process(target=_peer_worker, args=(r, world, port)) for r in range(world)]
    for q in procs:
        q.start()
    for q in procs:
        q.join(180)
    for q in procs:
        if q.is_alive():
            q.kill()
            pytest.fail('worker did not finish')
        assert q.exitcode == 0
