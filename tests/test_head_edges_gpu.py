"""Proposal-head NLL (net.cu: nll_row) row by row against fp64 (tests/heads_fp64.py), at the edges of every head.

The last head layer of each address has zero weights and the head output under test as its bias, so that every row of the
address has exactly that output in every precision mode (the tf32 split of 0 is 0 and the bias is added in fp32).  Every
sub-batch is one site long (T = 1) and holds one address, and its rows share (x, v, prior0, prior1): the address's
head-bias gradient is then (rows / B) d(-log q)/dx of that one row.  A second, forward-only pass gives the rows of each
sub-batch different values and checks each row's log q.

Each case runs through every form of nll_row, chosen by the number of addresses per call (one 128-row tile each):
NllRowEpi, the reduce phase of the h2 cluster GEMM, at CS = 8, 4 and 2 (pick_cluster with spread_epilogue over 132 SMs:
<= 16, 17-33 and 34-66 tiles), k_head_nll after the h2 GEMM at precision 0 (> 66 tiles) and on the SIMT path
(precision 2), and the feed-forward network.  The kernel names in a torch.profiler trace show which one ran.

Bound, per entry: |kernel - fp64| <= 4 m + floor, where m is what fp32 evaluation can move the entry by (Ref): the
larger of the reference's formula in torch fp32 with autograd, fp64 at the fp32-rounded proposal parameters (a Uniform
mean sigmoid(30) (hi - lo) + lo is hi in fp32), and the first-order sum of single roundings (the means, stddevs or
mixture probs one ulp off, the truncation mass's CDF values and densities three ulps off — erff's and expf's error
bounds plus one rounding —, each component's log density two ulps off, z, alpha, beta one ulp off).  Where the expression
is ill-conditioned — the window mass Z cancelling at a large Poisson stddev, v - mean at a prior mean of 1e4, the
truncation terms of a window much narrower than the stddev — the bound follows it, while a wrong term, index or lane is
off by far more than that on the well-conditioned entries.  A non-finite alternative (0 * inf in fp32 autograd) says
nothing and is left out.  The floors are a few fp32 roundings of the largest quantity the entry is computed from: for
log q, 16 eps (1 + |log q|); for a gradient entry, 16 eps times the row's largest gradient entry.  Non-finite results are
checked by class: a batch with status 0 must have finite log q and gradients everywhere, and a case that must fail —
the reference's fp32 log q is NaN or +inf, or the exact gradient does not fit fp32 — runs on its own and must set the
status for each of its rows.
"""
import math
import re

import numpy as np
import pytest
import torch

from pyprob_b200 import synthetic
from pyprob_b200.util import InferenceNetwork
from tests import heads_fp64 as hf

pytestmark = pytest.mark.gpu

EPS32 = hf.EPS32
ROWS = 3                  # rows of a sub-batch in the gradient pass
FILLERS = 80              # benign Normal addresses that pad a call to the size that selects a path
# path -> (precision, addresses per call, the kernel that must run the NLL)
PATHS = {'cs8': (0, 12, 8), 'cs4': (0, 24, 4), 'cs2': (0, 48, 2), 'nll_p0': (0, FILLERS, None), 'nll_p2': (2, 40, None)}
KS = (1, 2, 3, 10, 31, 32)
_SHOW = 8                 # failing entries a message lists


def _f32(a):
    return np.float32(a)


def _next(a, b):
    return float(np.nextafter(_f32(a), _f32(b)))


def _weights(K):
    w = {'equal': np.zeros(K)}
    if K > 1:
        w['lead16'] = np.r_[16.0, np.zeros(K - 1)]     # other weights e^-16 = 1.1e-7: just below eps32 at K = 2 ...
        w['lead20'] = np.r_[20.0, np.zeros(K - 1)]     # ... and clamped at every K
        w['tie'] = np.r_[5.0, 5.0, np.zeros(K - 2)]
    return w


def _mix_x(K, xm0, xsd0, xp, base_scale):
    """Component 0 carries the edge; the others are spread out with unit stddev so that they explain other values."""
    xm = np.linspace(-base_scale, base_scale, K) if K > 1 else np.zeros(1)
    xm[0] = xm0
    xsd = np.zeros(K)
    xsd[0] = xsd0
    return np.concatenate([xm, xsd, xp]).astype(np.float32)


def _mean_sd0(family, x, K, p0, p1):
    q = hf.proposal(family, torch.tensor(x, dtype=torch.float64), K, torch.tensor(float(_f32(p0)), dtype=torch.float64),
                    torch.tensor(float(_f32(p1)), dtype=torch.float64))
    return float(q[0][0]), float(q[1][0])


def mixture_cases(K):
    """(family, num_categories, x, v, p0, p1, values for the forward-only pass)"""
    out = []
    W = _weights(K)
    eq = W['equal']
    # Normal: prior stddev 1e-3 / 1 / 1e3, prior mean 1e4, component stddev e^xsd * p1, values k sd from the mean
    normal = [(0.0, 1.0, xsd, k, 'equal') for xsd in (-50, -45, -10, 0, 10, 40) for k in (0, 5, 30, 1e3)]
    normal += [(0.0, p1, xsd, k, 'equal') for p1 in (1e-3, 1e3) for xsd in (-10, 0, 10) for k in (0, 5, 30)]
    normal += [(1e4, 1.0, xsd, k, 'equal') for xsd in (-10, 0) for k in (0, 5, 30)]
    normal += [(0.0, 1.0, 0, k, w) for w in W if w != 'equal' for k in (0, 5)]
    for p0, p1, xsd, k, w in normal:
        x = _mix_x(K, 0.5, xsd, W[w], 2.0)
        m, s = _mean_sd0('Normal', x, K, p0, p1)
        vs = [float(_f32(m + j * s)) for j in (0, 5, 30, 1e3)]
        out.append(('Normal', 0, x, float(_f32(m + k * s)), p0, p1, vs))
    # a component whose t is -inf (its tiny stddev puts v at z^2 = inf) next to components that explain v
    for xsd in (-50, -45):
        x = _mix_x(K, 0.5, xsd, eq, 2.0)
        m, _ = _mean_sd0('Normal', x, K, 0.0, 1.0)
        out.append(('Normal', 0, x, float(_f32(m + 0.3)), 0.0, 1.0, [float(_f32(m + d)) for d in (0.0, 0.3, -1.0)]))
    # Uniform: ranges, v at / one float inside each bound and in the middle, mean and stddev logits at +-30 and 0
    for lo, hi in ((0.0, 1.0), (-1e3, 1e3), (1000.0, 1001.0), (-5.0, -4.99)):
        lo, hi = float(_f32(lo)), float(_f32(hi))
        vs = [lo, _next(lo, hi), float(_f32((lo + hi) / 2)), _next(hi, lo), hi]
        grid = [(a, b) for a in (-30, 0, 30) for b in (-30, 0, 30)] if (lo, hi) == (0.0, 1.0) else \
            [(0, 0), (-30, -30), (30, 30), (-30, 30)]
        for xm0, xsd0 in grid:
            x = _mix_x(K, xm0, xsd0, eq, 2.0)
            for v in vs:
                out.append(('Uniform', 0, x, v, lo, hi, vs))
    # Poisson: the [0, 40] window, 41 outside it (-inf, repaired); stddev from 1e-22 to e^25.  Near e^20 the fp32 window
    # mass Z is one rounding step of Phi(beta) - Phi(alpha), at e^25 it is 0 and log q is +inf (the batch fails)
    vs = [0.0, 1.0, 39.0, 40.0, 41.0]
    for xm0 in (-30, 0, 30):
        for xsd0 in (-50, -45, -30, -5, 0, 5, 10, 15, 20, 25):
            x = _mix_x(K, xm0, xsd0, eq, 3.0)
            for v in vs:
                out.append(('Poisson', 0, x, v, 0.0, 0.0, vs))
    w = W.get('lead20', eq)
    for v in (0.0, 39.0):
        out.append(('Poisson', 0, _mix_x(K, 0, 0, w, 3.0), v, 0.0, 0.0, vs))
    return out


def other_cases():
    out = []
    for C in (1, 2, 31, 32, 33, 64, 65, 127, 128):
        ramp = np.linspace(-1, 1, C) if C > 1 else np.zeros(1)
        for s in (0, 20, -20, 100, -100):
            x = (s * ramp).astype(np.float32)
            vs = sorted({0, C - 1, int(np.argmax(x)), int(np.argmin(x)), C // 2})
            for v in vs:
                out.append(('Categorical', C, x, float(v), 0.0, 0.0, [float(u) for u in vs]))
        x = np.zeros(C, np.float32)
        x[C // 2] = 30.0                                   # one category far ahead, at an interior lane
        out.append(('Categorical', C, x, float(C // 2), 0.0, 0.0, [0.0, float(C // 2), float(C - 1)]))
        out.append(('Categorical', C, x, float(C), 0.0, 0.0, [float(C)]))     # outside: NaN and status
    for x in (100, -100, 20, -20, 17, -17, 16, -16, 1, -1, 0):
        for v in (0.0, 1.0):
            out.append(('Bernoulli', 0, np.array([x], np.float32), v, 0.0, 0.0, [0.0, 1.0]))
    return out


def _filler(K):
    return ('Normal', 0, np.zeros(3 * K, np.float32), 0.5, 0.0, 1.0, [0.5, -1.0])


class Ref:
    """Results of one (case, value), cached: fp64, then what fp32 evaluation can move it by.  First the reference's
    formula in fp32 and fp64 at the fp32-rounded proposal parameters; then, one source at a time, fp64 with the means,
    the stddevs or the mixture probs one fp32 ulp up, the truncation mass's two CDF values and densities three ulps apart,
    the component log densities two ulps up and down, and z, alpha, beta one ulp each (heads_fp64.head,
    nudge)."""
    _cache = {}
    NUDGES = ((1, 0, 0, 0, 0, 0), (0, 1, 0, 0, 0, 0), (0, 0, 1, 0, 0, 0), (0, 0, 0, 1, 0, 0), (0, 0, 0, 0, 1, 0),
              (0, 0, 0, 0, 0, 1))

    @classmethod
    def get(cls, case, v):
        fam, C, x, _, p0, p1, _ = case
        key = (fam, C, x.tobytes(), v, p0, p1)
        if key not in cls._cache:
            kw = dict(num_categories=C) if fam in ('Categorical', 'Bernoulli') else {}
            alts = [hf.head(fam, x, v, p0, p1, dtype=torch.float32, **kw), hf.head(fam, x, v, p0, p1, round_params=True, **kw)]
            alts += [hf.head(fam, x, v, p0, p1, nudge=n, **kw) for n in cls.NUDGES]
            cls._cache[key] = (hf.head(fam, x, v, p0, p1, **kw), alts)
        return cls._cache[key]


FLT_MAX = float(np.finfo(np.float32).max)


def _fails(case):
    """The batch must fail with this row: the reference's fp32 log q is NaN or +inf (the reference aborts such a batch),
    or its fp32 log q is finite but the exact gradient does not fit fp32 (an inf would otherwise reach the optimiser).
    An fp32 log q of -inf is repaired and does not fail the batch."""
    r64, alts = Ref.get(case, case[3])
    r32 = alts[0]
    if not math.isfinite(r32['lp']):
        return True
    return not r32['repaired'] and not (np.abs(r64['grad']) <= FLT_MAX).all()


def _bound(k64, alts, floor):
    """4 x the largest of: the fp32 formula's error, the error of fp64 at fp32-rounded parameters, and the first-order sum
    of the single-source roundings (the moves of the nudged evaluations added up, since the kernel's roundings add), plus
    the floor (Ref).  A non-finite alternative says nothing (0 * inf in fp32 autograd, an overflow at a nudged parameter)
    and is left out."""
    moves = []
    for k in alts:
        e = np.abs(np.asarray(k, np.float64) - k64)
        moves.append(np.where(np.isfinite(e), e, 0.0))
    d = np.maximum(np.maximum(moves[0], moves[1]), sum(moves[2:], np.zeros_like(moves[0])))
    return 4 * d + floor


def _net(cases, K, precision, kind=InferenceNetwork.LSTM):
    table = [('e{}'.format(i), fam, C) for i, (fam, C, *_) in enumerate(cases)]
    net = synthetic.build_network({'o0': {'dim': 8, 'depth': 1}}, [2], table, lstm_dim=32, mixture_components=K,
                                  seed=1, precision=precision, inference_network=kind)
    sd = net.reference_state_dict()
    for (a, _, _), case in zip(table, cases):
        sd['_layers_proposal.{}._ff._layers.1.weight'.format(a)].zero_()
        sd['_layers_proposal.{}._ff._layers.1.bias'.format(a)].copy_(torch.from_numpy(case[2]))
    net.load_reference_state_dict(sd)
    return net, [a for a, _, _ in table]


def _sub(addr, fam, C, vs, p0, p1):
    B = len(vs)
    return {'addresses': [addr], 'families': [fam], 'num_categories': [C],
            'values': np.asarray(vs, np.float32).reshape(1, B), 'prior0': np.full((1, B), p0, np.float32),
            'prior1': np.full((1, B), p1, np.float32), 'obs': np.zeros((B, 2), np.float32)}


def _kernels(prof):
    return [e.key for e in prof.key_averages() if e.device_time_total > 0]


def _assert_path(names, cs):
    nll = [n for n in names if 'k_head_nll' in n]
    epi = [int(m.group(1)) for n in names for m in [re.search(r'k_cluster<\w+, (\d+), 3, [^<>]*NllRowEpi>', n)] if m]
    if cs is None:
        assert nll and not epi, names
    else:
        assert not nll and epi == [cs], names


def _run_call(net, addrs, cases, idx, K, profile=False):
    """One training step over the cases idx (one address each): checks status, per-row log q and head-bias gradients."""
    subs = [_sub(addrs[i], cases[i][0], cases[i][1], [cases[i][3]] * ROWS, cases[i][4], cases[i][5]) for i in idx]
    B = ROWS * len(idx)
    net._arena.grad = None
    names = None
    if profile:
        from torch.profiler import ProfilerActivity, profile as prof_
        with prof_(activities=[ProfilerActivity.CUDA]) as prof:
            ok, loss = net._loss(synthetic.ArrayBatch(subs))
            torch.cuda.synchronize()
        names = _kernels(prof)
    else:
        ok, loss = net._loss(synthetic.ArrayBatch(subs))
    status = int(net._last_status.item())
    assert ok and status == 0, ('status', status, [cases[i][:2] + cases[i][3:6] for i in idx])
    loss.backward()
    grad = net._arena.grad
    bad = []
    assert bool(torch.isfinite(grad).all()), ('non-finite gradient with status 0',
                                              [(cases[i][0], cases[i][2].tolist(), cases[i][3], cases[i][4], cases[i][5])
                                               for i in idx if not bool(torch.isfinite(net.grad_view(
                                                   '_layers_proposal.{}._ff._layers.1.bias'.format(addrs[i]))).all())])
    present = set(idx)
    for i, a in enumerate(addrs):
        g = net.grad_view('_layers_proposal.{}._ff._layers.1.bias'.format(a)).cpu().double().numpy()
        if i not in present:
            assert not g.any(), ('absent address with a gradient', a)
            continue
        r64, alts = Ref.get(cases[i], cases[i][3])
        want = r64['grad'] * ROWS / B
        w32 = alts[0]['grad'] * ROWS / B
        floor = 16 * EPS32 * np.abs(want).max()
        err = np.abs(g - want)
        lim = _bound(want, [a['grad'] * ROWS / B for a in alts], floor)
        if not (err <= lim).all():
            j = int(np.argmax(err - lim))
            bad.append((cases[i][0], cases[i][2].tolist(), cases[i][3], cases[i][4], cases[i][5], j, float(g[j]),
                        float(want[j]), float(w32[j])))
    # forward-only pass: the rows of each sub-batch take different values
    subs = []
    for i in idx:
        vs = [v for v in cases[i][6] if not _fails(cases[i][:3] + (v,) + cases[i][4:])]
        subs.append(_sub(addrs[i], cases[i][0], cases[i][1], vs or [cases[i][3]], cases[i][4], cases[i][5]))
    enc, lp = net.row_log_probs(synthetic.ArrayBatch(subs))
    assert int(net._last_status.item()) == 0
    lp = lp.cpu().double().numpy()
    for s, i in enumerate(idx):
        r0 = int(enc.arrays['step_row0'][s])
        for r, v in enumerate(subs[s]['values'][0]):
            r64, alts = Ref.get(cases[i], float(v))
            got = lp[r0 + r]
            lim = _bound(r64['lp'], [a['lp'] for a in alts], 16 * EPS32 * (1 + abs(r64['lp'])))
            if not (abs(got - r64['lp']) <= lim):
                bad.append(('lp', cases[i][0], cases[i][2].tolist(), float(v), cases[i][4], cases[i][5], float(got),
                            r64['lp'], alts[0]['lp']))
    if bad:
        pytest.fail('{} entries outside the bound: {!r}'.format(len(bad), bad[:_SHOW]))
    return names


def _run_path(path, cases, K, kind=InferenceNetwork.LSTM):
    precision, per_call, cs = PATHS[path]
    fill = [_filler(K)] * FILLERS
    good = [c for c in cases if not _fails(c)]
    net, addrs = _net(good + fill, K, precision, kind)
    n_real = per_call - 2                          # at least two fillers per call, so that every call has the same size
    chunks = [list(range(j, min(j + n_real, len(good)))) for j in range(0, len(good), n_real)]
    for c, idx in enumerate(chunks):
        idx = idx + list(range(len(good), len(good) + per_call - len(idx)))
        names = _run_call(net, addrs, good + fill, idx, K, profile=(c == 0))
        if c == 0:
            _assert_path(names, cs)


@pytest.mark.parametrize('path', list(PATHS))
@pytest.mark.parametrize('K', KS)
def test_mixture_heads_vs_fp64(cuda, K, path):
    """Normal, Uniform and Poisson heads.  Includes components whose t is -inf, or whose responsibility is 0 while z / sd
    overflows, next to components that explain v (Normal at xsd = -50 / -45 with v 0.3 away, the Poisson head at
    xsd = -50 / -45): their gradient is exactly 0, not 0 * inf = NaN."""
    _run_path(path, mixture_cases(K), K)


@pytest.mark.parametrize('path', list(PATHS))
def test_categorical_bernoulli_heads_vs_fp64(cuda, path):
    _run_path(path, other_cases(), 3)


def test_feedforward_network_heads_vs_fp64(cuda):
    _run_path('cs4', mixture_cases(3)[::2] + other_cases()[::2], 3, InferenceNetwork.FEEDFORWARD)


@pytest.mark.parametrize('K', (1, 3, 32))
def test_failing_rows_set_status(cuda, K):
    """Cases that must fail the batch (Z = 0 at a huge Poisson stddev, a Categorical value C, a gradient beyond fp32 at
    K = 1), each in a batch with one benign address: the status counts each of their rows."""
    cases = [c for c in mixture_cases(K) + (other_cases() if K == 3 else []) if _fails(c)]
    assert cases
    assert any(c[0] == 'Poisson' for c in cases)
    if K == 3:
        assert sum(c[0] == 'Categorical' for c in cases) == 9
    net, addrs = _net(cases + [_filler(K)], K, 0)
    for i, c in enumerate(cases):
        subs = [_sub(addrs[i], c[0], c[1], [c[3]] * ROWS, c[4], c[5]), _sub(addrs[-1], 'Normal', 0, [0.5] * ROWS, 0.0, 1.0)]
        enc = synthetic.ArrayBatch(subs).encode(net)
        net._forward_native(enc, want_grad=True)
        status = int(net._last_status.item())
        assert status == ROWS, (c[0], c[2].tolist(), c[3], status)
    if K == 1:
        assert any(c[0] == 'Normal' for c in cases)     # xsd = -45, v 0.3 from the mean: d(-log q)/d xm = -3.5e38


@pytest.mark.parametrize('kind', [InferenceNetwork.LSTM, InferenceNetwork.FEEDFORWARD])
@pytest.mark.parametrize('K', (1, 31, 32))
def test_ic_proposal_step_vs_fp64(cuda, K, kind):
    """The other copy of the transforms: the IC proposal step (ppb_ic_infer_step -> heads::mixture_params /
    categorical_probs / bernoulli_prob) at every distinct head output of the grid, against the fp64 proposal parameters.
    Bound: 4 |fp32 - fp64| (torch fp32 of the same transforms) plus floors of 16 eps of the value, plus 16 eps
    (|p0| + |p1|) for a mean (p0 + x p1 and p0 + sigmoid(x) (p1 - p0) round on the scale of the priors) and
    16 eps 10 |p1 - p0| for a Uniform stddev."""
    seen, cases = set(), []
    for c in mixture_cases(K) + [c for c in other_cases() if c[0] == 'Bernoulli' or c[1] in (1, 33, 128)]:
        key = (c[0], c[1], c[2].tobytes(), c[4], c[5])
        if key not in seen:
            seen.add(key)
            cases.append(c)
    net, addrs = _net(cases, K, 0, kind)
    net._infer_init({'o0': np.zeros(2, np.float32)})
    n, bad = 4, []
    for a, c in zip(addrs, cases):
        fam, C, x, v, p0, p1, _ = c
        got = net._infer_step_batched(a, None, None, p0, p1, n).cpu().double().numpy()
        r64, alts = Ref.get(c, v)
        want, w32 = np.concatenate(r64['params']), np.concatenate(alts[0]['params'])
        floor = 16 * EPS32 * np.abs(want)
        if fam in hf.MIXTURES:
            floor[:K] += 16 * EPS32 * (abs(p0) + abs(p1))
            if fam == 'Uniform':
                floor[K:2 * K] += 16 * EPS32 * 10 * abs(p1 - p0)
        lim = _bound(want, [w32, w32], floor)     # no nudged alternatives: m = |fp32 - fp64|
        for r in range(n):
            if not (np.abs(got[r] - want) <= lim).all():
                j = int(np.argmax(np.abs(got[r] - want) - lim))
                bad.append((fam, C, x.tolist(), p0, p1, r, j, float(got[r, j]), float(want[j]), float(w32[j])))
    if bad:
        pytest.fail('{} entries outside the bound: {!r}'.format(len(bad), bad[:_SHOW]))
