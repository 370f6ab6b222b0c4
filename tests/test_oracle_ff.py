"""CPU: the feed-forward oracle (tests/ff_oracle.py) against the UNMODIFIED reference's InferenceNetworkFeedForward
(tests/golden/ff_golden.npz, written by tests/golden/make_ff_golden.py): the loss and every gradient of a minibatch with
all five proposal families and two trace types, and the _infer_step proposal at every address of a few prior traces."""
import numpy as np
import torch

from tests import ff_oracle


def test_oracle_loss_and_every_gradient_match_reference():
    fx = ff_oracle.load_fixture()
    assert {f for sb in fx['subs'] for f in sb['families']} == {'Normal', 'Uniform', 'Poisson', 'Categorical', 'Bernoulli'}
    assert len(fx['subs']) == 2
    loss, grads, _ = ff_oracle.loss_and_grads(fx['params'], fx['subs'], fx['observe_names'], fx['observe_in_dims'], fx['K'])
    assert abs(float(loss) - fx['loss']) <= 1e-5 * abs(fx['loss'])
    assert set(grads) == set(fx['grads'])
    for k, g in fx['grads'].items():
        scale = max(float(g.abs().max()), 1e-8)
        assert float((grads[k] - g).abs().max()) <= 1e-5 * scale + 1e-8, k


def test_oracle_infer_step_matches_reference():
    fx = ff_oracle.load_fixture()
    seen = set()
    for tr in fx['infer']:
        for st in tr['steps']:
            got = ff_oracle.infer_step(fx['params'], tr['obs'], fx['observe_names'], fx['observe_in_dims'], fx['K'],
                                       st['address'], st['family'], st['prior0'], st['prior1'])
            assert len(got) == len(st['proposal'])
            for g, w in zip(got, st['proposal']):
                np.testing.assert_allclose(torch.as_tensor(g).reshape(-1).numpy(), w.reshape(-1), rtol=1e-5, atol=1e-7)
            seen.add(st['family'])
    assert seen == {'Normal', 'Uniform', 'Poisson', 'Categorical', 'Bernoulli'}
