"""GPU end-to-end acceptance through the public API, mirroring the reference's own integration tests:
tests/test_inference.py:94-246 (GaussianUnknownMean: posterior mean/stddev within 0.75 of Normal(7.25,
sqrt(1/1.2)), ESS floors), :249-410 (Marsaglia variant with stochastic control flow), tests/test_train.py
(learn_inference_network runs, save -> load -> continue)."""
import math

import numpy as np
import pytest
import torch

import pyprob_b200 as pyprob
from oracle import scoring, weights
from pyprob_b200 import InferenceEngine, InferenceNetwork, Model
from pyprob_b200.distributions import Normal, Uniform

pytestmark = pytest.mark.gpu

TRUE_MEAN, TRUE_STD = 7.25, math.sqrt(1 / 1.2)


class GaussianUnknownMean(Model):
    def __init__(self):
        super().__init__('Gaussian with unknown mean')

    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


class GaussianUnknownMeanMarsaglia(Model):
    """Stochastic control flow (reference tests/test_inference.py:249-275) in lock-step form."""

    def __init__(self):
        super().__init__('Gaussian with unknown mean (Marsaglia)')

    def marsaglia(self, mean, stddev):
        def body(s):
            x = pyprob.sample(Uniform(-1, 1))
            y = pyprob.sample(Uniform(-1, 1))
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


class ScalarControlFlow(Model):
    """Python-scalar control flow on a sampled value: must still work (one particle per execution)."""

    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)))
        if float(mu) > 100:
            mu = mu * 0
        pyprob.observe(Normal(mu, math.sqrt(2)), name='obs0')
        return mu


def test_gum_importance_sampling_posterior(cuda):
    pyprob.seed(1)
    model = GaussianUnknownMean()
    post = model.posterior_results(65536, InferenceEngine.IMPORTANCE_SAMPLING, observe={'obs0': 8, 'obs1': 9})
    assert post.length == 65536
    assert abs(float(post.mean) - TRUE_MEAN) < 0.1 and abs(float(post.stddev) - TRUE_STD) < 0.1
    assert post.effective_sample_size > 0.005 * 65536  # reference floor: tests/test_inference.py:121
    # weights are exactly the double sum of the two observe log-likelihoods of each particle's mu
    mu = post.values.cpu()
    terms = np.stack([scoring.normal_log_prob(np.float32(o), mu, np.float32(math.sqrt(2))).numpy() for o in (8., 9.)])
    want = weights.accumulate(terms).astype(np.float32)
    np.testing.assert_allclose(post.log_weights.cpu().numpy(), want, rtol=1e-4, atol=1e-5)
    lse, ess, logits = weights.finalize(want)
    np.testing.assert_allclose(post.effective_sample_size, ess, rtol=1e-3)


def test_prior_and_scalar_control_flow_fallback(cuda):
    pyprob.seed(2)
    prior = GaussianUnknownMean().prior_results(20000)
    assert abs(float(prior.mean) - 1.0) < 0.1 and abs(float(prior.stddev) - math.sqrt(5)) < 0.1
    with pytest.warns(UserWarning):
        post = ScalarControlFlow().posterior_results(40, observe={'obs0': 8})
    assert post.length == 40


def test_marsaglia_is_posterior_lock_step(cuda):
    pyprob.seed(3)
    post = GaussianUnknownMeanMarsaglia().posterior_results(50000, observe={'obs0': 8, 'obs1': 9})
    assert abs(float(post.mean) - TRUE_MEAN) < 0.2 and abs(float(post.stddev) - TRUE_STD) < 0.2


def test_gum_inference_compilation_end_to_end(cuda, tmp_path):
    pyprob.seed(4)
    pyprob.set_verbosity(0)
    model = GaussianUnknownMean()
    model.learn_inference_network(num_traces=30000, batch_size=256, inference_network=InferenceNetwork.LSTM,
                                  lstm_dim=64, observe_embeddings={'obs0': {'dim': 32}, 'obs1': {'dim': 32}})
    net = model._inference_network
    assert net._total_train_traces >= 30000 and net._loss_min < net._loss_init
    post = model.posterior_results(4096, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                   observe={'obs0': 8, 'obs1': 9})
    assert abs(float(post.mean) - TRUE_MEAN) < 0.3 and abs(float(post.stddev) - TRUE_STD) < 0.3
    assert post.effective_sample_size > 0.15 * 4096  # reference floor for IC-LSTM: tests/test_inference.py:178
    # save -> load -> continue (tests/test_train.py:107-150)
    fn = str(tmp_path / 'net.network')
    model.save_inference_network(fn)
    model2 = GaussianUnknownMean()
    model2.load_inference_network(fn)
    assert model2._inference_network._optimizer_step == net._optimizer_step
    model2.learn_inference_network(num_traces=512, batch_size=256, inference_network=InferenceNetwork.LSTM,
                                   observe_embeddings={'obs0': {'dim': 32}, 'obs1': {'dim': 32}})
    assert model2._inference_network._total_train_traces >= net._total_train_traces + 512
    post2 = model2.posterior_results(2048, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                     observe={'obs0': 8, 'obs1': 9})
    assert abs(float(post2.mean) - TRUE_MEAN) < 0.3


def test_marsaglia_inference_compilation(cuda):
    """Reference acceptance (tests/test_inference.py:335-360): posterior mean within 0.75, ESS above 1.6 % of the draws.
    The ESS of an importance sampler is a heavy-tailed statistic (one large weight halves it) and training is not
    run-to-run reproducible (fp32 reductions with atomics), so the floor is checked on the median of five independent
    posterior draws of a 600k-trace training run.  scripts/marsaglia_ess.py on an H100 (seeds 5-10, three draws each):
    per-run medians 416-1711 against the floor of 131, single draws down to 228 (one draw of 36 over three kernel paths
    fell to 126) — the median over five draws keeps one or two such draws from deciding the test."""
    pyprob.seed(5)
    pyprob.set_verbosity(0)
    model = GaussianUnknownMeanMarsaglia()
    model.learn_inference_network(num_traces=600000, batch_size=256, inference_network=InferenceNetwork.LSTM,
                                  lstm_dim=128, observe_embeddings={'obs0': {'dim': 16}, 'obs1': {'dim': 16}})
    ess, means = [], []
    for _ in range(5):
        post = model.posterior_results(8192, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                       observe={'obs0': 8, 'obs1': 9})
        ess.append(float(post.effective_sample_size))
        means.append(float(post.mean))
    assert abs(sorted(means)[2] - TRUE_MEAN) < 0.5
    assert sorted(ess)[2] > 0.016 * 8192, ess  # reference floor: tests/test_inference.py:344


def test_online_minibatches_are_disjoint_between_ranks(cuda, monkeypatch):
    """Data-parallel online training: rank r draws particles [r*B, (r+1)*B) of one Philox draw, so two ranks' minibatches
    are the two halves of a single 2B-trace batch — never the same traces twice."""
    from pyprob_b200 import parallel
    from pyprob_b200.dataset import OnlineDataset
    model = GaussianUnknownMean()
    halves = []
    for rank in (0, 1):
        pyprob.seed(9)
        monkeypatch.setattr(parallel, 'world_info', lambda r=rank: (2, r))
        batch = OnlineDataset(model).next_batch(64)
        halves.append(batch.trace.variables_controlled[0].value.cpu())
    assert not torch.equal(halves[0], halves[1])
    pyprob.seed(9)
    monkeypatch.setattr(parallel, 'world_info', lambda: (1, 0))
    full = OnlineDataset(model).next_batch(128).trace.variables_controlled[0].value.cpu()
    assert torch.equal(torch.cat(halves), full)


class DivergingPaths(Model):
    """Lanes reach the last site from DIFFERENT previous sites: half of them run an extra masked statement."""

    def forward(self):
        a = pyprob.sample(Uniform(0, 1))
        st = pyprob.while_loop(lambda s: s['todo'] > 0,
                               lambda s: {'b': pyprob.sample(Normal(2.0, 1.0)), 'todo': s['todo'] * 0},
                               {'b': 0.0, 'todo': (a > 0.5).float()})
        c = pyprob.sample(Normal(st['b'] + a, 1.0))
        pyprob.observe(Normal(c, 0.5), name='obs')
        return c


def test_ic_weights_follow_each_lanes_own_previous_site(cuda):
    """Per-lane previous site / LSTM state in lock-step IC (ADVICE round 1): particles that skipped the masked statement
    must be conditioned on the site THEY executed last, exactly like one reference trace each (state.py:203-219)."""
    from pyprob_b200.util import TraceMode
    from tests.ic_replay import site_weight_terms
    pyprob.seed(31)
    pyprob.set_verbosity(0)
    model = DivergingPaths()
    model.learn_inference_network(num_traces=30 * 256, batch_size=256, inference_network=InferenceNetwork.LSTM, lstm_dim=64,
                                  observe_embeddings={'obs': {'dim': 16}})
    net = model._inference_network
    n = 2000
    with torch.no_grad():
        trace = model._run_batched(n, trace_mode=TraceMode.POSTERIOR,
                                   inference_engine=InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                   inference_network=net, observe={'obs': 3.0})
    want, covered = site_weight_terms(trace, net, torch.tensor([3.0]))
    assert covered.all()
    c = trace.result.cpu()
    want = want + scoring.normal_log_prob(torch.tensor(3.0), c, torch.tensor(0.5)).double().numpy()
    got = trace.log_w.cpu().numpy()
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=2e-4)
    took_b = trace.variables_controlled[1].mask.cpu().numpy()
    assert 0.3 < took_b.mean() < 0.7      # both kinds of lanes are present
