"""CPU: pins tests/lstm_fp64.py, the restatement of InferenceNetworkLSTM._loss at any dtype that the GPU recurrence tests
(tests/test_lstm_fp64_gpu.py) compare against.  At float32 it must be the oracle (oracle/network.py, with the Bernoulli
head of tests/bernoulli_oracle.py) to fp32 rounding; at float64 it must agree with the reference's own loss and gradients
(tests/golden/network_golden.npz) to the reference's fp32 rounding; its per-step state must be the infer step's."""
import numpy as np
import pytest
import torch

from pyprob_b200 import synthetic
from tests import bernoulli_oracle as bo
from tests import lstm_fp64, netfixture

TABLE = [('a_u', 'Uniform', 0), ('a_c', 'Categorical', 5), ('a_n', 'Normal', 0), ('a_p', 'Poisson', 0),
         ('a_n2', 'Normal', 0), ('a_c2', 'Categorical', 3), ('a_b', 'Bernoulli', 0)]
OBS = {'o0': {'dim': 12, 'depth': 2}, 'o1': {'dim': 6, 'depth': 3}}
IN_DIMS = [3, 1]


def _linear(gen, prefix, n_in, n_out, out):
    bound = 1 / np.sqrt(n_in)
    out[prefix + '.weight'] = (torch.rand(n_out, n_in, generator=gen) * 2 - 1) * bound
    out[prefix + '.bias'] = (torch.rand(n_out, generator=gen) * 2 - 1) * bound


def _ff(gen, prefix, n_in, n_out, depth, out):
    dims = [(n_in, n_out)] if depth == 1 else \
        [(n_in, (n_in + n_out) // 2)] + [((n_in + n_out) // 2,) * 2] * (depth - 2) + [((n_in + n_out) // 2, n_out)]
    for i, (a, b) in enumerate(dims):
        _linear(gen, '{}._layers.{}'.format(prefix, i), a, b, out)


def random_params(seed, H, K, S=4, table=TABLE):
    """A network's parameters under the reference's state_dict names, with the shapes InferenceNetworkLSTM gives them
    (pyprob_b200/network.py), drawn on the CPU."""
    gen = torch.Generator().manual_seed(seed)
    p = {}
    for (name, spec), d in zip(OBS.items(), IN_DIMS):
        _ff(gen, '_layers_observe_embedding.' + name, d, spec['dim'], spec['depth'], p)
    E = sum(spec['dim'] for spec in OBS.values())
    _ff(gen, '_layers_observe_embedding_final', E, E, 2, p)
    I = E + S + 2 * (64 + 8)
    bound = 1 / np.sqrt(H)
    for k, shape in (('weight_ih_l0', (4 * H, I)), ('weight_hh_l0', (4 * H, H)), ('bias_ih_l0', (4 * H,)),
                     ('bias_hh_l0', (4 * H,))):
        p['_layers_lstm.' + k] = (torch.rand(*shape, generator=gen) * 2 - 1) * bound
    for a, fam, C in table:
        p['_layers_address_embedding.' + a] = torch.randn(64, generator=gen)
        p.setdefault('_layers_distribution_type_embedding.' + fam, torch.randn(8, generator=gen))
        out = C if fam == 'Categorical' else 1 if fam == 'Bernoulli' else 3 * K
        _ff(gen, '_layers_proposal.{}._ff'.format(a), H, out, 2, p)
        _linear(gen, '_layers_sample_embedding.{}._layers.0'.format(a), C if fam == 'Categorical' else 1, S, p)
    return p


def _subs(seed, spec, table=TABLE):
    rng = np.random.default_rng(seed)
    subs = [synthetic.random_sub_batch(rng, [table[i] for i in seq], B, 4) for seq, B in spec]
    return [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]


CASES = [   # the random cases of tests/test_network_gpu.py, with a Bernoulli site (index 6) added to the last two
    (1, 32, 3, [([0, 1, 2], 5)]),
    (2, 32, 10, [([0, 1, 2, 3, 4, 5, 6], 7), ([2], 1), ([0, 3], 64), ([1, 5, 4, 0], 3)]),
    (3, 64, 4, [([2, 4], 130), ([5, 1, 6, 1, 5, 1, 0], 33), ([3], 257)]),
]


@pytest.mark.parametrize('seed,H,K,spec', CASES)
def test_float32_is_the_oracle(seed, H, K, spec):
    params = random_params(seed, H, K)
    subs = _subs(seed, spec)
    want_loss, want_grads, want_lps = bo.loss_and_grads(params, subs, list(OBS), IN_DIMS, K, repaired_rows='constant')
    got = lstm_fp64.loss_and_grads(params, subs, list(OBS), IN_DIMS, K, dtype=torch.float32)
    assert got['loss'].dtype == torch.float32
    torch.testing.assert_close(got['loss'], want_loss, rtol=2e-6, atol=0)
    for g, w in zip(got['lps'], want_lps):
        torch.testing.assert_close(g, w, rtol=1e-5, atol=1e-5)
    assert set(got['grads']) == set(want_grads)
    for k, w in want_grads.items():
        scale = max(float(w.abs().max()), 1e-12)
        assert float((got['grads'][k] - w).abs().max()) <= 1e-5 * scale + 1e-9, k


@pytest.mark.parametrize('tag', ['gum', 'mixed'])
def test_float64_matches_the_reference_fixture(tag):
    fx = netfixture.load(tag)
    got = lstm_fp64.loss_and_grads(fx['params'], fx['subs'], fx['observe_names'], fx['observe_in_dims'], fx['K'])
    assert got['loss'].dtype == torch.float64
    assert abs(float(got['loss']) - fx['loss']) <= 1e-6 * abs(fx['loss'])
    for k, w in fx['grads'].items():
        scale = max(float(w.abs().max()), 1e-12)
        assert float((got['grads'][k] - w.double()).abs().max()) <= 1e-4 * scale + 1e-7, k


def test_step_state_and_term_magnitudes():
    """infer_steps replays the per-step h and c of one trace, d loss / d pre-activation sums to the bias gradient, and
    M bounds every LSTM gradient element."""
    seed, H, K = 3, 16, 4
    params = random_params(seed, H, K)
    subs = _subs(seed, [([5, 1, 6, 0, 2], 9), ([3, 4], 4)])
    res = lstm_fp64.loss_and_grads(params, subs, list(OBS), IN_DIMS, K)
    sb, b = subs[0], 7
    steps = [{'address': a, 'family': f, 'num_categories': c, 'prev_value': sb['values'][t - 1, b:b + 1] if t else None}
             for t, (a, f, c) in enumerate(zip(sb['addresses'], sb['families'], sb['num_categories']))]
    replay = lstm_fp64.infer_steps(params, sb['obs'][b], list(OBS), IN_DIMS, steps)
    for t, (h, c) in enumerate(replay):
        torch.testing.assert_close(h[0], res['steps'][0][t]['h'][b], rtol=1e-12, atol=1e-14)
        torch.testing.assert_close(c[0], res['steps'][0][t]['c'][b], rtol=1e-12, atol=1e-14)
    # d loss / d bias_ih[j] is the sum of dgates[:, j] over every (t, row)
    db = sum(s['dgates'].sum(0) for sub in res['steps'] for s in sub)
    torch.testing.assert_close(db, res['grads']['_layers_lstm.bias_ih_l0'], rtol=1e-12, atol=1e-15)
    M = lstm_fp64.lstm_term_magnitudes(res)
    for k in lstm_fp64.LSTM_NAMES:
        assert bool((res['grads'][k].abs() <= M[k] * (1 + 1e-12)).all()), k
        assert float(M[k].max()) > 0, k
