"""GPU: the Metropolis-Hastings engines (LMH, RMH) as lock-step chains.

  * replay: every chain's chosen site, log alpha and accept decision, recomputed on the host from the engine's own
    current and candidate traces (oracle/mcmc.py, oracle/philox.py and the rules of include/pyprob_b200.h section 7);
  * the exact law after S steps: Branching's LMH transition matrix, built in numpy, against 65,536 chains;
  * posteriors of independent chains at the last step against closed forms and forward-backward;
  * the public surface: lengths, step-major order, indexing, seeding, the scalar fallback, errors, no syncs.
Tolerances come from Monte Carlo standard errors (KS / chi-square p-values, z-scores)."""
import math

import numpy as np
import pytest
import scipy.stats
import torch

import pyprob_b200 as pyprob
from oracle import mcmc as omcmc
from oracle import philox
from pyprob_b200 import InferenceEngine, Model, mcmc, state, util
from pyprob_b200.distributions import Categorical, Normal, Poisson, Uniform
from pyprob_b200.empirical import Empirical
from pyprob_b200.model import trace_result
from pyprob_b200.util import TraceMode

pytestmark = pytest.mark.gpu

LMH = InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS
RMH = InferenceEngine.RANDOM_WALK_METROPOLIS_HASTINGS
GUM_OBS = {'obs0': 8, 'obs1': 9}
TRUE_MEAN, TRUE_STD = 7.25, math.sqrt(1 / 1.2)
P_MIN = 1e-3


class GUM(Model):
    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


class Marsaglia(Model):
    def forward(self):
        def body(s):
            x = pyprob.sample(Uniform(-1, 1))
            y = pyprob.sample(Uniform(-1, 1))
            return {'x': x, 'y': y, 's': x * x + y * y}
        st = pyprob.while_loop(lambda s: s['s'] >= 1, body, {'x': 0.0, 'y': 0.0, 's': 2.0})
        mu = 1 + math.sqrt(5) * (st['x'] * torch.sqrt(-2 * torch.log(st['s']) / st['s']))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


class VaryingCategorical(Model):
    """The live categories of the second sample depend on the first: categories >= k have probability 0, so a reused
    index that the new k excludes is rescored at log(eps32) (torch's clamped Categorical) and enters log alpha."""

    def forward(self):
        k = pyprob.sample(Categorical([1, 1, 1, 1])) + 1
        probs = (torch.arange(4, device='cuda').view(1, -1) < k.view(-1, 1)).float()
        j = pyprob.sample(Categorical(probs))
        pyprob.observe(Normal(j, 1.0), name='obs')
        return j


def _fib(n):      # the reference Branching model's fibonacci
    if n < 2:
        return 1
    a = fib = 1
    for _ in range(n - 2):
        a, fib = fib, a + fib
    return fib


FIB = [_fib(3 * r) for r in range(5)]


class BranchingLockstep(Model):
    """The reference's Branching (tests/test_inference.py:579-603) in lock-step form: the inner sample runs in a
    one-iteration while_loop for the chains with r <= 4.  Returns (r, s) with s = -1 where the inner sample did not run."""

    def forward(self):
        r = pyprob.sample(Poisson(4))
        st = pyprob.while_loop(lambda s: (r <= 4) & (s['i'] < 1),
                               lambda s: {'i': s['i'] + 1, 's': pyprob.sample(Poisson(4))}, {'i': 0.0, 's': -1.0})
        fib = torch.tensor(FIB, dtype=torch.float32, device='cuda')[r.clamp(max=4).long()]
        lam = torch.where(r > 4, torch.full_like(r, 6.0), 1 + fib + st['s'])
        pyprob.observe(Poisson(lam), name='obs')
        return torch.stack([r, st['s']], dim=1)


class Branching(Model):
    """The reference's Branching, unmodified: python-scalar control flow on a sample."""

    def forward(self):
        count_prior = Poisson(4)
        r = pyprob.sample(count_prior)
        if 4 < float(r):
            lam = 6
        else:
            lam = 1 + _fib(3 * int(r)) + pyprob.sample(count_prior)
        pyprob.observe(Poisson(lam), name='obs')
        return r


class MovingUniform(Model):
    """The second Uniform's upper bound is the first sample: a reused value above a smaller new bound is outside the
    support, scores -inf and is drawn fresh."""

    def forward(self):
        b = pyprob.sample(Uniform(1, 3))
        y = pyprob.sample(Uniform(0, b))
        pyprob.observe(Normal(y, 1.0), name='obs')
        return y


class UniformPrior(Model):
    def forward(self):
        x = pyprob.sample(Uniform(0, 10))
        pyprob.observe(Normal(x, 1.0), name='obs')
        return x


HMM_OBS = [0.9, 0.8, 0.7, 0.0, -0.025, -5.0, -2.0, -0.1, 0.0, 0.13, 0.45, 6, 0.2, 0.3, -1, -1]
HMM_T = np.array([[0.1, 0.5, 0.4], [0.2, 0.2, 0.6], [0.15, 0.15, 0.7]])
HMM_MEANS = np.array([-1.0, 1.0, 0.0])


class HMMLockstep(Model):
    """The reference's hidden Markov model (tests/test_inference.py:416-440) with per-chain transition rows."""

    def forward(self):
        T = torch.tensor(HMM_T, dtype=torch.float32, device='cuda')
        means = torch.tensor(HMM_MEANS, dtype=torch.float32, device='cuda')
        states = [pyprob.sample(Categorical([1, 1, 1]))]
        for i in range(len(HMM_OBS)):
            s = pyprob.sample(Categorical(T[states[-1].long()]))
            pyprob.observe(Normal(means[s.long()], 1.0), name='obs{}'.format(i))
            states.append(s)
        return torch.stack(states, dim=1)


def _hmm_marginals():
    """Exact posterior marginals of the 17 states by forward-backward."""
    def lik(y):
        return np.exp(-0.5 * (y - HMM_MEANS) ** 2)
    n = len(HMM_OBS)
    alpha = np.zeros((n + 1, 3))
    alpha[0] = 1 / 3
    for t in range(n):
        alpha[t + 1] = (alpha[t] @ HMM_T) * lik(HMM_OBS[t])
        alpha[t + 1] /= alpha[t + 1].sum()
    beta = np.ones((n + 1, 3))
    for t in range(n - 1, -1, -1):
        beta[t] = HMM_T @ (lik(HMM_OBS[t]) * beta[t + 1])
        beta[t] /= beta[t].sum()
    m = alpha * beta
    return m / m.sum(1, keepdims=True)


# ---- helpers -------------------------------------------------------------------------------------------------------
def _last_states(post, num_chains):
    v = post.values
    return v[len(post) - num_chains:].double().cpu().numpy()


def _run(model, engine, steps, num_chains, observe, thinning=None):
    """Records step 0 and step steps - 1 only (thinning steps - 1), so that the last num_chains states are the chains'
    states after `steps` steps."""
    return model.posterior(steps, inference_engine=engine, observe=observe, num_chains=num_chains,
                           thinning_steps=thinning if thinning is not None else steps - 1)


def _chi2_p(counts, probs):
    """Chi-square goodness-of-fit p-value, cells with expected count below 5 pooled."""
    counts = np.asarray(counts, dtype=np.float64)
    expected = np.asarray(probs, dtype=np.float64) * counts.sum()
    big = expected >= 5
    obs = np.append(counts[big], counts[~big].sum())
    exp = np.append(expected[big], expected[~big].sum())
    if exp[-1] < 5:
        obs[-2] += obs[-1]
        exp[-2] += exp[-1]
        obs, exp = obs[:-1], exp[:-1]
    return scipy.stats.chisquare(obs, exp).pvalue


# ---- 1. replay ----------------------------------------------------------------------------------------------------
def _replay(model, engine, observe, num_chains, steps, rmh_prior=None):
    util.seed(11)
    state._init_traces(model.forward, trace_mode=TraceMode.POSTERIOR, inference_engine=engine, observe=observe)
    ch = mcmc.Chains(num_chains, engine, steps)
    ch.run_step(model, trace_result, -1, False)
    checked_choice = checked_accept = refreshed = 0
    C = num_chains
    for i in range(steps):
        b0, cs0 = ch.buf.clone(), ch.cur_stamp.clone()
        cur_n0, cur_lpo0 = ch.cur_n.clone(), ch.cur_lpo.clone()
        ch.run_step(model, trace_result, i, False)
        off_select, off_accept = ch.offsets
        val, lp = ch.val.cpu().numpy(), ch.lp.cpu().numpy()
        stamp, reused = ch.stamp.cpu().numpy(), ch.reused.cpu().numpy()
        b0, cs0, b1 = b0.cpu().numpy(), cs0.cpu().numpy(), ch.buf.cpu().numpy()
        cur_n0, cur_lpo0 = cur_n0.cpu().numpy(), cur_lpo0.cpu().numpy()
        choice, la_gpu = ch.choice.cpu().numpy(), ch.log_alpha.cpu().numpy()
        cand_n, cand_lpo, trans = ch.cand_n.cpu().numpy(), ch.cand_lpo.cpu().numpy(), ch.trans.cpu().numpy()
        w_sel = philox.philox4x32_10(util._seed, np.arange(C, dtype=np.uint64), off_select)[:, 0]
        w_acc = philox.philox4x32_10(util._seed, np.arange(C, dtype=np.uint64), off_accept)[:, 0]
        for c in range(C):
            cur_cols = np.nonzero(stamp[b0[c], c, :ch.ncols] == cs0[c])[0]
            cand_cols = np.nonzero(stamp[1 - b0[c], c, :ch.ncols] == ch.step)[0]
            assert len(cur_cols) == cur_n0[c] and len(cand_cols) == cand_n[c]
            # chosen column: k = min(floor(u m), m - 1), the k-th present column
            m = len(cur_cols)
            um = np.float32(philox.u01(w_sel[c:c + 1])[0]) * np.float32(m)
            if abs(um - round(float(um))) > 1e-4:
                assert choice[c] == cur_cols[min(int(um), m - 1)]
                checked_choice += 1
            cur, cand = (b0[c], c), (1 - b0[c], c)
            rc = [a for a in cand_cols if reused[cand][a]]
            assert all(stamp[cur][a] == cs0[c] for a in rc)      # a reused site is in the current trace
            assert choice[c] not in rc
            # present in both, neither chosen nor reused: the current value fell outside the new support
            refreshed += sum(1 for a in cand_cols if a != choice[c] and not reused[cand][a] and stamp[cur][a] == cs0[c])
            t = 0.0
            if rmh_prior is not None:
                a = choice[c]
                t = omcmc.rmh_transition(rmh_prior[0], float(val[cur][a]), float(lp[cur][a]), float(val[cand][a]),
                                         float(lp[cand][a]), *rmh_prior[1:])
                assert abs(t - trans[c]) <= 1e-4 * (1 + abs(t)), (t, trans[c])
            la = omcmc.log_acceptance(cur_n0[c], cand_n[c], cur_lpo0[c], cand_lpo[c], lp[cand][rc], lp[cur][rc],
                                      float(trans[c]))
            scale = 1 + abs(cur_lpo0[c]) + abs(cand_lpo[c]) + np.abs(lp[cand][rc]).sum() + np.abs(lp[cur][rc]).sum()
            assert abs(la - la_gpu[c]) <= 1e-6 * scale, (c, la, la_gpu[c])
            lu = math.log(float(philox.u01_open0(w_acc[c:c + 1])[0]))
            if abs(lu - la) > 1e-4:
                assert (b1[c] != b0[c]) == (lu < la), (c, lu, la)
                checked_accept += 1
    assert checked_choice > 0.9 * C * steps and checked_accept > 0.9 * C * steps
    return ch, refreshed


def test_replay_gum_lmh():
    _, refreshed = _replay(GUM(), LMH, GUM_OBS, 256, 6)
    assert refreshed == 0


def test_replay_gum_rmh():
    _replay(GUM(), RMH, GUM_OBS, 256, 6, rmh_prior=('Normal', 1.0, math.sqrt(5)))


def test_replay_marsaglia_lmh():
    ch, refreshed = _replay(Marsaglia(), LMH, GUM_OBS, 256, 6)
    assert ch.ncols > 2 and refreshed == 0          # chains hold different numbers of loop iterations


def test_replay_varying_categorical():
    _replay(VaryingCategorical(), LMH, {'obs': 2.0}, 256, 8)


def test_replay_out_of_support_draws_fresh():
    _, refreshed = _replay(MovingUniform(), LMH, {'obs': 1.5}, 256, 8)
    assert refreshed > 0


def test_replay_uniform_rmh():
    _replay(UniformPrior(), RMH, {'obs': 7.0}, 256, 6, rmh_prior=('Uniform', 0.0, 10.0))


# ---- 2. exact law after S steps -------------------------------------------------------------------------------------
def _branching_matrix(obs=6, top=40):
    """Exact one-step transition matrix of the reference's LMH (model.py:141-167, state.py:225-276) on Branching.
    States: (r, s) for r <= 4, (r, -1) for r > 4, r and s in 0 .. top."""
    pr = scipy.stats.poisson.pmf(np.arange(top + 1), 4)
    pr = pr / pr.sum()
    states = [(r, s) for r in range(5) for s in range(top + 1)] + [(r, -1) for r in range(5, top + 1)]
    index = {x: i for i, x in enumerate(states)}

    def lpo(x):
        r, s = x
        return scipy.stats.poisson.logpmf(obs, 6 if r > 4 else 1 + FIB[r] + s)

    def nsites(x):
        return 1 if x[0] > 4 else 2

    P = np.zeros((len(states), len(states)))
    for i, x in enumerate(states):
        r, s = x
        moves = []     # (probability, candidate)
        for r2 in range(top + 1):       # site r chosen: fresh r'; s reused when both have it, else fresh
            if r2 > 4:
                moves.append((pr[r2] / nsites(x), (r2, -1)))
            elif s >= 0:
                moves.append((pr[r2] / nsites(x), (r2, s)))
            else:
                for s2 in range(top + 1):
                    moves.append((pr[r2] * pr[s2] / nsites(x), (r2, s2)))
        if s >= 0:                      # site s chosen: r reused, fresh s'
            for s2 in range(top + 1):
                moves.append((pr[s2] / 2, (r, s2)))
        for p, y in moves:
            # reused sites rescore under unchanged priors: the reuse sum is 0, the transition term is 0 (LMH)
            a = min(1.0, math.exp(math.log(nsites(x)) - math.log(nsites(y)) + lpo(y) - lpo(x)))
            P[i, index[y]] += p * a
            P[i, i] += p * (1 - a)
    pi0 = np.array([pr[r] * (pr[s] if s >= 0 else 1.0) for r, s in states])
    return states, index, P, pi0


@pytest.mark.parametrize('engine', [LMH, RMH])
def test_branching_exact_s_step_law(engine):
    S, C = 4, 65536
    states, index, P, pi0 = _branching_matrix()
    want = pi0 @ np.linalg.matrix_power(P, S)
    util.seed(3)
    post = _run(BranchingLockstep(), engine, S, C, {'obs': 6})
    got = _last_states(post, C).reshape(C, 2).astype(np.int64)
    counts = np.zeros(len(states))
    for r, s in got:
        counts[index[(int(r), int(s))]] += 1
    assert _chi2_p(counts, want) > P_MIN


# ---- 3. posteriors --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('engine', [LMH, RMH])
def test_gum_posterior(engine):
    C = 16384
    util.seed(5)
    post = _run(GUM(), engine, 2000, C, GUM_OBS)
    x = _last_states(post, C)
    assert scipy.stats.kstest(x, scipy.stats.norm(TRUE_MEAN, TRUE_STD).cdf).pvalue > P_MIN


def test_marsaglia_posterior():
    C = 16384
    util.seed(6)
    post = _run(Marsaglia(), LMH, 2000, C, GUM_OBS)
    x = _last_states(post, C)
    assert scipy.stats.kstest(x, scipy.stats.norm(TRUE_MEAN, TRUE_STD).cdf).pvalue > P_MIN


def test_uniform_prior_rmh_posterior():
    C = 16384
    util.seed(7)
    post = _run(UniformPrior(), RMH, 1000, C, {'obs': 7.0})
    x = _last_states(post, C)
    a, b = (0 - 7.0) / 1.0, (10 - 7.0) / 1.0
    assert scipy.stats.kstest(x, scipy.stats.truncnorm(a, b, 7.0, 1.0).cdf).pvalue > P_MIN


def test_hmm_posterior_marginals():
    C = 16384
    util.seed(8)
    post = _run(HMMLockstep(), LMH, 1500, C, {'obs{}'.format(i): v for i, v in enumerate(HMM_OBS)})
    got = _last_states(post, C).reshape(C, len(HMM_OBS) + 1).astype(np.int64)
    want = _hmm_marginals()
    for t in range(len(HMM_OBS) + 1):
        counts = np.bincount(got[:, t], minlength=3)
        assert _chi2_p(counts, want[t]) > P_MIN / (len(HMM_OBS) + 1), (t, counts / C, want[t])


# ---- 4. surface ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('num_chains', [1, 64])
@pytest.mark.parametrize('thinning', [None, 3])
def test_length_and_step_major_order(num_chains, thinning):
    util.seed(1)
    steps = 10
    post = GUM().posterior_results(steps, inference_engine=LMH, observe=GUM_OBS, num_chains=num_chains,
                                   thinning_steps=thinning)
    records = math.ceil(steps / (thinning or 1))
    assert len(post) == records * num_chains
    assert 'LMH' in post.name and post._metadata[-1]['num_chains'] == num_chains
    # step-major: the same run thinned by 1 holds every step; recorded step k of chain c is its entry k * thinning
    util.seed(1)
    full = GUM().posterior_results(steps, inference_engine=LMH, observe=GUM_OBS, num_chains=num_chains)
    fv = full.values.view(steps, num_chains)
    pv = post.values.view(records, num_chains)
    assert torch.equal(pv, fv[::thinning or 1])


def test_empirical_indexing():
    util.seed(2)
    C = 32
    post = GUM().posterior(20, inference_engine=RMH, observe=GUM_OBS, num_chains=C)
    assert float(post[3]) == float(post.values[3])
    tail = post[5 * C:]
    assert isinstance(tail, Empirical) and len(tail) == 15 * C
    assert torch.equal(tail.values, post.values[5 * C:])
    assert tail.name == post.name and tail._metadata[-1]['op'] == 'slice'
    assert tail._metadata[0]['num_chains'] == C


def test_same_seed_same_bits():
    out = []
    for _ in range(2):
        util.seed(9)
        out.append(Marsaglia().posterior(8, inference_engine=LMH, observe=GUM_OBS, num_chains=128).values)
    assert torch.equal(out[0], out[1])


def test_reference_branching_scalar_fallback():
    util.seed(4)
    model = Branching()
    with pytest.warns(UserWarning, match='python-scalar'):
        post = model.posterior(400, inference_engine=LMH, observe={'obs': 6}, num_chains=4)
    assert model._scalar_mode and len(post) == 1600
    r = post[400:].values.cpu().numpy()      # after 100 steps of burn-in
    states, index, P, pi0 = _branching_matrix()
    pr_r = {}
    post_exact = np.linalg.matrix_power(P, 4000)[0]
    for (rr, _), p in zip(states, post_exact):
        pr_r[rr] = pr_r.get(rr, 0.0) + p
    mean_exact = sum(k * p for k, p in pr_r.items())
    assert abs(r.mean() - mean_exact) < 1.0      # loose: 4 correlated chains


class NoSample(Model):
    def forward(self):
        pyprob.observe(Normal(0, 1), name='obs')
        return torch.zeros(1, device='cuda')


def test_errors():
    with pytest.raises(RuntimeError, match='empty initial trace'):
        NoSample().posterior(3, inference_engine=LMH, observe={'obs': 0.0})
    with pytest.raises(NotImplementedError, match='initial_trace'):
        GUM().posterior(3, inference_engine=RMH, observe=GUM_OBS, initial_trace=object())


def test_straight_line_steps_do_not_sync():
    util.seed(12)
    model = GUM()
    state._init_traces(model.forward, trace_mode=TraceMode.POSTERIOR, inference_engine=LMH, observe=GUM_OBS)
    ch = mcmc.Chains(1024, LMH, 20)
    for i in range(3):      # warm-up: the initial trace and the first steps allocate the tables and constants
        ch.run_step(model, trace_result, i - 1 if i else -1, False)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        for i in range(2, 20):
            ch.run_step(model, trace_result, i, False)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert int(ch.accepted.sum()) > 0
