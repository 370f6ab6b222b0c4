"""GPU: Bernoulli random variables end to end — scoring and sampling kernels, the Bernoulli proposal head in the training
loss (every precision, the fused head-output kernel), the infer step, and importance sampling with and without an
inference network.  References: the UNMODIFIED reference (tests/golden/bernoulli_golden.npz), torch.distributions and
the oracle in tests/bernoulli_oracle.py.  Tolerances follow tests/test_scoring_gpu.py and tests/test_network_gpu.py."""
import math

import numpy as np
import pytest
import torch

import pyprob_b200 as pyprob
from pyprob_b200 import InferenceEngine, InferenceNetwork, Model, ops, synthetic
from pyprob_b200.distributions import Bernoulli, Normal
from tests import bernoulli_oracle as bo

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-4, 1e-5


def _check(got, want, rtol=RTOL, atol=ATOL):
    got = got.detach().cpu().double().numpy()
    want = np.asarray(want, dtype=np.float64)
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    np.testing.assert_allclose(got[fin], want[fin], rtol=rtol, atol=atol)


# ---- scoring ------------------------------------------------------------------------------------------------------------
def test_log_prob_vs_reference_fixture_and_torch(cuda):
    g = bo.load_scoring()
    v, p = torch.from_numpy(g['value']), torch.from_numpy(g['probs'])
    _check(ops.bernoulli_log_prob(v.to(cuda), p.to(cuda)), g['lp'])
    _check(Bernoulli(p.to(cuda)).log_prob(v.to(cuda)), g['lp'])
    # odd n and unaligned pointers (scalar path), scalar probs
    _check(ops.bernoulli_log_prob(v.to(cuda)[1:], p.to(cuda)[1:]), g['lp'][1:])
    for q in (0.0, 0.3, 1.0):
        want = torch.distributions.Bernoulli(probs=torch.tensor(q)).log_prob(v)
        _check(ops.bernoulli_log_prob(v.to(cuda), q), want)
        _check(ops.bernoulli_log_prob(v.to(cuda)[3:], q), want[3:])


@pytest.mark.parametrize('n', [1, 7, 4096, 100003])
def test_log_prob_vs_torch_sizes_and_acc(cuda, n):
    gen = torch.Generator().manual_seed(n)
    p = torch.rand(n, generator=gen)
    v = (torch.rand(n, generator=gen) < 0.5).float()
    want = torch.distributions.Bernoulli(probs=p).log_prob(v)
    _check(ops.bernoulli_log_prob(v.to(cuda), p.to(cuda)), want)
    # acc form: fp64 running sum of fp32 terms (pyprob/trace.py:123-125)
    acc = torch.full((n,), 0.25, dtype=torch.float64, device=cuda)
    ops.bernoulli_log_prob(v.to(cuda), p.to(cuda), acc=acc, acc_scale=-1.0)
    lp = ops.bernoulli_log_prob(v.to(cuda), p.to(cuda))
    assert torch.equal(acc, 0.25 - lp.double())


def test_value_outside_support_is_nan(cuda):
    v = torch.tensor([0.0, 1.0, 2.0, -1.0, 0.5], device=cuda)
    lp = ops.bernoulli_log_prob(v, 0.3).cpu().numpy()
    assert np.isfinite(lp[:2]).all() and np.isnan(lp[2:]).all()


# ---- sampling -----------------------------------------------------------------------------------------------------------
def test_sampler_moments_log_prob_and_sharding(cuda):
    n = 25000
    for p in (0.05, 0.3, 0.8):
        x, lp = ops.bernoulli_sample(p, n, 1, 7, with_log_prob=True)
        assert set(torch.unique(x).tolist()) <= {0.0, 1.0}
        m = x.mean().item()
        assert abs(m - p) < 0.1                                   # reference tolerance (tests/test_distributions.py)
        assert abs(m - p) < 5 * math.sqrt(p * (1 - p) / n)        # binomial bound
        _check(lp, torch.distributions.Bernoulli(probs=torch.tensor(p)).log_prob(x.cpu()))
    assert ops.bernoulli_sample(0.0, 1000, 1, 8).sum().item() == 0
    assert ops.bernoulli_sample(1.0, 1000, 1, 8).sum().item() == 1000
    # per-particle probs
    probs = torch.linspace(0, 1, n, device=cuda)
    x = ops.bernoulli_sample(probs, n, 2, 9)
    assert abs(x.mean().item() - 0.5) < 5 * math.sqrt(0.25 / n)
    # sharding: two first_index ranges reproduce the unsharded draw bit for bit
    full = ops.bernoulli_sample(probs, n, 3, 10, first_index=100)
    a = ops.bernoulli_sample(probs[:n // 3], n // 3, 3, 10, first_index=100)
    b = ops.bernoulli_sample(probs[n // 3:], n - n // 3, 3, 10, first_index=100 + n // 3)
    assert torch.equal(torch.cat([a, b]), full)


# ---- training loss: reference fixture -----------------------------------------------------------------------------------
def _net_from_fixture(fx, precision=0):
    obs_emb = {}
    for name in fx['observe_names']:
        depth = sum(1 for k in fx['params'] if k.startswith('_layers_observe_embedding.{}.'.format(name)) and k.endswith('weight'))
        dim = fx['params']['_layers_observe_embedding.{}._layers.{}.weight'.format(name, depth - 1)].shape[0]
        obs_emb[name] = {'dim': int(dim), 'depth': depth}
    fam_of = {}
    for sb in fx['subs']:
        for a, f, c in zip(sb['addresses'], sb['families'], sb['num_categories']):
            fam_of[a] = (f, c)
    addresses = [(a, fam_of[a][0], fam_of[a][1]) for a in fx['address_order']]
    net = synthetic.build_network(obs_emb, fx['observe_in_dims'], addresses, lstm_dim=fx['lstm_dim'],
                                  mixture_components=fx['K'], precision=precision)
    assert list(net._types) == fx['type_order']
    net.load_reference_state_dict(fx['params'])
    return net


def _subs_numpy(subs):
    return [{k: (v.numpy() if torch.is_tensor(v) else v) for k, v in sb.items()} for sb in subs]


def _check_grads(net, want, rtol=1e-4, grad=None):
    for k, g in want.items():
        got = net.grad_view(k, grad).cpu()
        scale = max(float(g.abs().max()), 1e-6)
        err = float((got - g).abs().max())
        assert err <= rtol * scale + 1e-7, (k, err, scale)


# precision 1 rounds every GEMM operand to tf32 (10-bit mantissa)
TOL = {0: (1e-4, 1e-4), 1: (2e-3, 2e-2), 2: (1e-4, 1e-4)}


@pytest.mark.parametrize('precision', [0, 1, 2])
def test_loss_and_grads_vs_reference_fixture(cuda, precision):
    fx = bo.load_fixture('bern')
    net = _net_from_fixture(fx, precision)
    ok, loss = net._loss(synthetic.ArrayBatch(_subs_numpy(fx['subs'])))
    assert ok
    ltol, gtol = TOL[precision]
    assert abs(float(loss.detach()) - fx['loss']) <= ltol * abs(fx['loss'])
    loss.backward()
    _check_grads(net, fx['grads'], gtol)


# ---- training loss: random cases against the oracle ---------------------------------------------------------------------
TABLE = [('b0', 'Bernoulli', 0), ('n0', 'Normal', 0), ('c0', 'Categorical', 3), ('b1', 'Bernoulli', 0),
         ('u0', 'Uniform', 0), ('p0', 'Poisson', 0)]


def _random_case(seed, lstm_dim, spec, precision):
    rng = np.random.default_rng(seed)
    net = synthetic.build_network({'o0': {'dim': 12, 'depth': 2}, 'o1': {'dim': 6, 'depth': 1}}, [3, 1], TABLE,
                                  lstm_dim=lstm_dim, mixture_components=4, seed=seed, precision=precision)
    subs = [synthetic.random_sub_batch(rng, [TABLE[i] for i in seq], B, 4) for seq, B in spec]
    return net, subs


def _oracle(net, subs):
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
    return bo.loss_and_grads(params, tsubs, ['o0', 'o1'], [3, 1], 4)


@pytest.mark.parametrize('seed,lstm_dim,spec', [
    (1, 32, [([0], 1)]),                                            # B = 1, T = 1
    (2, 64, [([3], 129)]),                                          # T = 1, a padding tail
    (3, 32, [([0, 1, 3, 2, 0], 129)]),                              # longer trace, Bernoulli as previous site
    (4, 64, [([0, 2, 3, 1], 40), ([3], 7), ([4, 0, 5, 3, 0, 1], 65)]),   # ragged, three sub-batches, all families
])
@pytest.mark.parametrize('precision', [0, 2])
def test_loss_and_grads_vs_oracle_random(cuda, seed, lstm_dim, spec, precision):
    net, subs = _random_case(seed, lstm_dim, spec, precision)
    want_loss, want_grads, _ = _oracle(net, subs)
    ok, loss = net._loss(synthetic.ArrayBatch(subs))
    assert ok
    assert abs(float(loss.detach()) - float(want_loss)) <= 1e-4 * abs(float(want_loss))
    loss.backward()
    _check_grads(net, want_grads)


@pytest.mark.parametrize('precision', [0, 2])
def test_out_of_support_row_sets_status_and_drops_out(cuda, precision):
    """A Bernoulli value of 2 gives a NaN log q: the row is counted in status and adds neither loss nor gradient (the
    reference returns (False, 0) for such a batch).  The row sits in a one-step sub-batch so that no later step reads it."""
    net, subs = _random_case(5, 32, [([0, 1, 3], 6), ([3], 4)], precision)
    subs[1]['values'][0] = [0.0, 2.0, 1.0, 1.0]
    batch = synthetic.ArrayBatch(subs)
    enc = batch.encode(net)
    grad = torch.zeros_like(net._arena.data)
    loss = net._forward_native(enc, want_grad=True)
    net._backward_native(enc, grad, 1.0)
    assert int(net._last_status.item()) == 1
    assert net._loss(synthetic.ArrayBatch(subs))[0] is False
    kept = [subs[0], dict(subs[1], values=subs[1]['values'][:, [0, 2, 3]], prior0=subs[1]['prior0'][:, [0, 2, 3]],
                          prior1=subs[1]['prior1'][:, [0, 2, 3]], obs=subs[1]['obs'][[0, 2, 3]])]
    want_loss, want_grads, _ = _oracle(net, kept)
    scale = 9.0 / 10.0     # the loss is divided by all 10 traces, the oracle's by the 9 kept ones
    assert abs(float(loss) - scale * float(want_loss)) <= 1e-4 * abs(float(want_loss))
    _check_grads(net, {k: scale * g for k, g in want_grads.items()}, grad=grad)


# ---- infer step ---------------------------------------------------------------------------------------------------------
def test_infer_step_tensor_core_and_simt_vs_oracle(cuda):
    fx = bo.load_fixture('bern')
    n = 300
    gen = torch.Generator().manual_seed(5)
    obs = {name: torch.randn(d, generator=gen) for name, d in zip(fx['observe_names'], fx['observe_in_dims'])}
    obs_row = torch.cat([obs[nm].reshape(-1) for nm in fx['observe_names']])
    for sb in fx['subs']:
        seq = list(zip(sb['addresses'], sb['families'], sb['num_categories']))
        vals, steps = [], []
        for t, (a, fam, C) in enumerate(seq):
            if fam == 'Categorical':
                v = torch.randint(0, C, (n,), generator=gen).float()
            elif fam == 'Bernoulli':
                v = (torch.rand(n, generator=gen) < 0.5).float()
            else:
                v = torch.randn(n, generator=gen)
            p0, p1 = (0.3, 0.5) if fam == 'Normal' else (None, None)
            steps.append({'address': a, 'family': fam, 'num_categories': C, 'prior0': p0 or 0.0, 'prior1': p1 or 0.0,
                          'prev_value': vals[-1] if vals else None})
            vals.append(v)
        want = bo.infer_sequence(fx['params'], obs_row, fx['observe_names'], fx['observe_in_dims'], fx['K'], steps, n)
        for precision in (0, 2):
            net = _net_from_fixture(fx, precision)
            net._infer_init(obs)
            prev_a, prev_v = None, None
            for (a, fam, C), st, w, v in zip(seq, steps, want, vals):
                params = net._infer_step_batched(a, prev_a, prev_v, st['prior0'] if fam == 'Normal' else None,
                                                 st['prior1'] if fam == 'Normal' else None, n).cpu()
                if fam == 'Bernoulli':
                    assert params.shape == (n, 1)
                torch.testing.assert_close(params, torch.cat(w, dim=1), rtol=2e-4, atol=1e-5)
                prev_a, prev_v = a, v.to(cuda)


# ---- models -------------------------------------------------------------------------------------------------------------
P1, MU0, MU1, SIGMA, X_OBS = 0.3, -1.0, 1.5, 1.0, 0.8


class BinarySwitch(Model):
    def __init__(self):
        super().__init__('Bernoulli switch')

    def forward(self):
        z = pyprob.sample(Bernoulli(P1))
        pyprob.observe(Normal(MU0 + (MU1 - MU0) * z, SIGMA), name='x')
        return z


def _closed_form():
    l1 = P1 * math.exp(-0.5 * ((X_OBS - MU1) / SIGMA) ** 2)
    l0 = (1 - P1) * math.exp(-0.5 * ((X_OBS - MU0) / SIGMA) ** 2)
    return l1 / (l0 + l1)


def test_importance_sampling_posterior(cuda):
    pyprob.seed(11)
    post = BinarySwitch().posterior_results(65536, InferenceEngine.IMPORTANCE_SAMPLING, observe={'x': X_OBS})
    assert abs(float(post.mean) - _closed_form()) < 0.01


def test_inference_compilation_posterior(cuda):
    """learn_inference_network on the Bernoulli switch, then IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK.  A trained
    proposal q(z | x) is close to the posterior, so the ESS approaches the number of draws; the prior proposal gets 0.66
    of them at this observation.  scripts/bernoulli_ic_ess.py on an H100 at this budget (40k traces), three draws of 8192
    per seed, ESS fraction (same to 0.002 across a seed's draws) and P(z = 1 | x) against the closed form 0.629:
    seed 1: 0.986, 0.623-0.639; seed 2: 0.970, 0.625-0.640; seed 3: 0.934, 0.622-0.633; seed 4: 0.835, 0.624-0.632;
    seed 5: 0.941, 0.627-0.634; seed 12 (this test): 1.000, 0.621-0.625.  At 20k traces seed 5 fell to 0.77, close to the
    prior proposal's 0.66, hence the doubled budget.  The floor of 0.75 sits below the smallest run and well above the
    prior proposal, so it fails when training does not improve on the prior."""
    pyprob.seed(12)
    pyprob.set_verbosity(0)
    model = BinarySwitch()
    model.learn_inference_network(num_traces=40000, batch_size=256, inference_network=InferenceNetwork.LSTM,
                                  lstm_dim=64, observe_embeddings={'x': {'dim': 16}})
    net = model._inference_network
    assert net._loss_min < net._loss_init
    n = 8192
    post = model.posterior_results(n, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK, observe={'x': X_OBS})
    assert abs(float(post.mean) - _closed_form()) < 0.03
    assert float(post.effective_sample_size) > 0.75 * n, float(post.effective_sample_size)
