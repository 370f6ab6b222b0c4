"""CPU: pins tests/obs_fp64.py, the layer-by-layer restatement of the observe embedding that the GPU observe-embedding tests
(tests/test_obs_embed_fp64_gpu.py) compare against.  At float32 it must be the oracle (oracle/network.embed_observe and
the losses of oracle/network.py and tests/ff_oracle.py) to fp32 rounding; at float64 it must agree with the reference's own
loss and gradients (tests/golden/network_golden.npz, ff_golden.npz) to the reference's fp32 rounding; its per-layer
gradients must add up to the bias gradients, and its term magnitudes and ReLU-flip bound must hold the float32 restatement
to float64."""
import pytest
import torch

from oracle import network as onet
from tests import bernoulli_oracle as bo
from tests import ff_oracle, lstm_fp64, netfixture, obs_fp64
from tests.test_lstm_fp64 import IN_DIMS, OBS, _subs, random_params


def _close(got, want, rel, atol=1e-9):
    assert set(got) >= set(want)
    for k, w in want.items():
        scale = max(float(w.abs().max()), 1e-12)
        assert float((got[k].double() - w.double()).abs().max()) <= rel * scale + atol, k


def test_embedding_is_the_oracle():
    params = random_params(4, 32, 3)
    obs = torch.randn(37, sum(IN_DIMS), generator=torch.Generator().manual_seed(4))
    layers = []
    got = obs_fp64.embed(params, obs, list(OBS), IN_DIMS, layers)
    assert torch.equal(got, onet.embed_observe(params, obs, list(OBS), IN_DIMS))
    # chains in observable order, then the final chain; each layer's output is the next one's input
    names = [L['name'] for L in layers]
    assert names == ['_layers_observe_embedding.o0._layers.{}'.format(i) for i in range(2)] + \
        ['_layers_observe_embedding.o1._layers.{}'.format(i) for i in range(3)] + \
        ['_layers_observe_embedding_final._layers.{}'.format(i) for i in range(2)]
    assert [L['chain'] for L in layers] == [0, 0, 1, 1, 1, None, None]
    assert torch.equal(layers[1]['x'], layers[0]['y']) and torch.equal(layers[-1]['y'], got)


@pytest.mark.parametrize('seed,spec', [(2, [([0, 1, 2, 3, 4, 5, 6], 7), ([2], 1), ([0, 3], 64)]),
                                       (3, [([2, 4], 130), ([5, 1, 6, 1, 5, 1, 0], 33)])])
def test_float32_is_the_oracle(seed, spec):
    params = random_params(seed, 32, 4)
    subs = _subs(seed, spec)
    want_loss, want_grads, _ = bo.loss_and_grads(params, subs, list(OBS), IN_DIMS, 4, repaired_rows='constant')
    got = obs_fp64.loss_and_grads(params, subs, list(OBS), IN_DIMS, 4, dtype=torch.float32)
    torch.testing.assert_close(got['loss'], want_loss, rtol=2e-6, atol=0)
    _close(got['grads'], want_grads, 1e-5)
    for sb, layers in zip(subs, got['obs']):
        assert torch.equal(layers[-1]['y'], onet.embed_observe(params, sb['obs'], list(OBS), IN_DIMS).detach())


def test_feedforward_float32_is_the_oracle():
    fx = ff_oracle.load_fixture()
    args = (fx['params'], fx['subs'], fx['observe_names'], fx['observe_in_dims'], fx['K'])
    want_loss, want_grads, _ = ff_oracle.loss_and_grads(*args)
    got = obs_fp64.loss_and_grads(*args, dtype=torch.float32, feedforward=True)
    torch.testing.assert_close(got['loss'], want_loss, rtol=2e-6, atol=0)
    _close(got['grads'], want_grads, 1e-5)


@pytest.mark.parametrize('tag', ['gum', 'mixed', 'ff'])
def test_float64_matches_the_reference_fixture(tag):
    fx = ff_oracle.load_fixture() if tag == 'ff' else netfixture.load(tag)
    got = obs_fp64.loss_and_grads(fx['params'], fx['subs'], fx['observe_names'], fx['observe_in_dims'], fx['K'],
                                  feedforward=tag == 'ff')
    assert got['loss'].dtype == torch.float64
    assert abs(float(got['loss']) - fx['loss']) <= 1e-6 * abs(fx['loss'])
    assert any(k.startswith('_layers_observe_embedding') for k in fx['grads'])
    _close(got['grads'], fx['grads'], 1e-4, atol=1e-7)   # test_lstm_fp64's tolerance: the reference ran in fp32


def test_layer_gradients_term_magnitudes_and_flip_bound():
    """dz sums to the bias gradient and dz^T x is the weight gradient; M bounds every gradient; the float32 restatement is
    within tau M + bound of float64, where the bound covers the units whose ReLU float32 puts on the other side."""
    seed, K = 5, 4
    params = random_params(seed, 32, K)
    subs = _subs(seed, [([0, 1, 2, 3], 700), ([2, 0], 300), ([1], 101)])
    res = obs_fp64.loss_and_grads(params, subs, list(OBS), IN_DIMS, K)
    res32 = obs_fp64.loss_and_grads(params, subs, list(OBS), IN_DIMS, K, dtype=torch.float32)
    M = obs_fp64.term_magnitudes(res)
    assert len(M) == 14 and all(k.startswith('_layers_observe_embedding') for k in M)
    for k in M:
        name, what = k.rsplit('.', 1)
        want = sum((L['dz'].sum(0) if what == 'bias' else L['dz'].t() @ L['x'])
                   for sub in res['obs'] for L in sub if L['name'] == name)
        torch.testing.assert_close(want, res['grads'][k], rtol=1e-10, atol=1e-15)
        assert bool((res['grads'][k].abs() <= M[k] * (1 + 1e-12)).all()) and float(M[k].max()) > 0, k
    # dy is dz where the unit is open
    L = res['obs'][0][0]
    assert torch.equal(torch.where(L['z'] > 0, L['dy'], torch.zeros_like(L['dy'])), L['dz'])
    bound, n = obs_fp64.relu_flip_bound(params, res, 2e-5)
    assert set(bound) == set(M) and n >= 0
    for k in M:
        err = (res32['grads'][k].double() - res['grads'][k]).abs()
        assert bool((err <= 1e-2 * (M[k] + 1e-6 * float(M[k].max())) + bound[k]).all()), k
    # at rel = 1 every unit is ambiguous (|z| <= |x| |W|^T + |b| always), and the bound only grows with rel
    big, every = obs_fp64.relu_flip_bound(params, res, 1.0)
    assert every == sum(L['z'].numel() for sub in res['obs'] for L in sub) > n
    assert all(bool((big[k] >= bound[k]).all()) for k in M)
