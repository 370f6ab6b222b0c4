"""GPU: the LSTM recurrence of the training step and its backward pass against the float64 restatement (tests/lstm_fp64.py),
at every kernel form the dispatcher picks for a T > 1 step.

Each case asserts, from the kernel names torch.profiler records, the form it is meant to reach (pick_cluster in net_tc.inc,
132 SMs, tiles = 128-row tiles x H / 32 unit blocks per step):
  k_lstm_step                   H < 128 (too few 32-element chunks to split), or more than 66 tiles in a step
  k_lstm_cluster<., 2, 4>       H = 128 and H = 160 (5 chunks over 2 CTAs: an uneven split)
  k_lstm_cluster<., 4, 4>       H = 256 at <= 4 row tiles, and H = 512 at one row tile (a pick of 8 runs the CS = 4 kernel)
  k_lstm_cluster<., ., 8>       sample_embedding_dim 5 and 8
  k_grouped + k_cell_fwd        PPB_FUSED_CELL=0
  k_cell_bwd<true>              at t = 0 when B % 128 == 0 (it writes the d_pobs tile images), else k_cell_bwd<false>
  no tensor-core kernel         every case at precision 2 (fp32 SIMT), and H % 32 != 0 (precisions 0 and 1 refuse it)

Observables and tolerances (TOL; tau per precision and observable, about 4x the worst error seen on one NVIDIA H100 80GB
HBM3 at 700 W, except where said):
  lq          log q of every (t, row) and the loss: |got - want| <= tau (1 + |want|)
  lstm        LSTM weight and bias grads per element: |got - want| <= tau M, M = sum over rows of |dgates| |x|
  lstm_row    the saturated case's LSTM grads per row (below)
  trunc       Uniform / Poisson (truncated-normal) head grads, per output row: |got - want| <= tau max(row max |want|,
              1e-3 tensor max) (per 32-element block of a vector)
  other       every other gradient, per row as trunc
  norm        ||got - want|| / ||want|| per tensor (norm_trunc: the truncated-normal head tensors): below 1, so a tensor
              that is zero, halved or of the wrong sign fails at every precision
  infer       h and c of the infer step against lstm_fp64.infer_steps, |got - want| <= tau (1 + |want|)
Worst seen (precision 0 / 2 / 1):
  lq          1.7e-6 (unfused ragged) / 2.0e-6 (workspace) / 3.3e-4 (saturated)
  lstm        2.8e-4 (S = 8, H = 128) / 1.7e-4 (workspace) / 0.33 (H = 512)
  lstm_row    6.5e-5 / 6.5e-5 / 0.17 (saturated)
  trunc       6.4e-2 (H = 96) / 5.7e-2 (H = 96) / 1.1 (H = 256, B = 1100)
  other       4.9e-4 (S = 8, H = 128) / 4.9e-4 / 2.3 (ragged)
  norm        4.1e-4 / 4.3e-4 / 0.55 (S = 5, H = 256; its tolerance 0.8 keeps it below 1)
  norm_trunc  4.1e-4 / 4.4e-4 / 0.10
  infer       3.2e-7 (H = 128; H = 100 on the SIMT GEMMs is lower)
The truncated-normal heads' gradients cancel over a minibatch: the float32 restatement itself is 1.7e-2 of a row from
float64 on the Uniform head at H = 96, so their per-row tau is set by conditioning, not by a kernel, and kept apart from the
other tensors.  The LSTM gradients of the S = 8, H = 128 case sit above the other cases at precision 0 and also at precision
2, whose fp32 SIMT path shares no GEMM or cell kernel with the tensor-core path: the fp32 rounding of dgates where its terms
cancel.  In the saturated case fp32 rounds sigmoid(x) to 1 above x = 17, so sigmoid' is 0 there and a unit saturated at every
step gets an exactly zero gradient where fp64 has one of 1e-13 of its terms (error = M at precisions 0 and 2 alike): its
LSTM gradients are held per row instead, at lstm_row.  Precision 1 rounds every GEMM operand to tf32 (10-bit mantissa);
rows that cancel to a small maximum show that rounding at more than their own size, so its per-row and per-element
tolerances only catch gross faults and its norm tolerance is the check that a tensor is right as a whole.
"""
import math
import re

import numpy as np
import pytest
import torch

from pyprob_b200 import _lib, synthetic
from tests import lstm_fp64

pytestmark = pytest.mark.gpu

TABLE = [('a_u', 'Uniform', 0), ('a_c', 'Categorical', 5), ('a_n', 'Normal', 0), ('a_p', 'Poisson', 0),
         ('a_n2', 'Normal', 0), ('a_c2', 'Categorical', 3), ('a_b', 'Bernoulli', 0)]
OBS, IN_DIMS, K = {'o0': {'dim': 12, 'depth': 2}, 'o1': {'dim': 6, 'depth': 3}}, [3, 1], 4

# per precision, the observables of `errors` (lstm_row holds the saturated case only; infer the infer-step test)
TOL = {0: dict(lq=7e-6, lstm=1.2e-3, lstm_row=2.6e-4, trunc=0.25, other=2e-3, norm=1.6e-3, norm_trunc=1.6e-3, infer=1.3e-6),
       1: dict(lq=1.3e-3, lstm=1.5, lstm_row=0.67, trunc=4.5, other=9.0, norm=0.8, norm_trunc=0.4),
       2: dict(lq=8e-6, lstm=7e-4, lstm_row=2.6e-4, trunc=0.25, other=2e-3, norm=1.8e-3, norm_trunc=1.8e-3)}

STEP, CS2, CS4, CS2S8, CS4S8 = 'step', ('cluster', 2, 4), ('cluster', 4, 4), ('cluster', 2, 8), ('cluster', 4, 8)


def _cycle(T, start=0):
    return [(start + t) % len(TABLE) for t in range(T)]


# name: (H, sample_dim, [(address sequence, traces)], LSTM forms at precisions 0 and 1)
CASES = {
    'h32': (32, 4, [(_cycle(7), 5), ([2], 1), ([0, 3], 64), ([1, 5, 4, 0], 3)], {STEP}),
    'h64': (64, 4, [([2, 4], 130), ([5, 1, 6, 1, 5, 1, 0], 33), ([3], 257)], {STEP}),
    'h96': (96, 4, [([4, 0, 1, 2], 40), ([6, 3], 90)], {STEP}),
    'h128': (128, 4, [(_cycle(10), 300)], {CS2}),
    'h160': (160, 4, [([3, 4, 0, 1, 6], 256)], {CS2}),
    'h256': (256, 4, [([2, 0, 4, 1], 140), ([3, 5, 6], 20)], {CS4}),
    'h256_b1100': (256, 4, [([2, 0, 4], 1100)], {STEP}),
    'h512': (512, 4, [(_cycle(6, 3), 100)], {CS4}),
    's5_h128': (128, 5, [(_cycle(5), 200)], {CS2S8}),
    's8_h128': (128, 8, [(_cycle(6, 2), 128)], {CS2S8}),
    's5_h256': (256, 5, [(_cycle(4, 1), 384)], {CS4S8}),
    's8_h256': (256, 8, [(_cycle(4, 4), 128)], {CS4S8}),
    # steps t = 1, 2 hold 10 row tiles (80 tiles: k_lstm_step), t = 3..7 four, t >= 8 one (CS = 4); BPTT phases of 3 problems
    'ragged': (256, 4, [(_cycle(3), 700), (_cycle(8, 1), 300), (_cycle(20, 2), 100)], {STEP, CS4}),
    # a sub-batch ends at every t, three of them one trace long
    'short': (128, 4, [(_cycle(T, T), B) for T, B in zip(range(1, 9), [1, 3, 1, 17, 5, 1, 2, 9])], {CS2}),
    'h100': (100, 4, [(_cycle(5), 150), ([1, 6], 30)], set()),
}
CELL_BWD = {name: 'true' if sum(B for _, B in spec) % 128 == 0 else 'false' for name, (_, _, spec, _) in CASES.items()}

_cache = {}


def _network(H, S, precision, seed):
    return synthetic.build_network(OBS, IN_DIMS, TABLE, lstm_dim=H, mixture_components=K, seed=seed, precision=precision,
                                   sample_embedding_dim=S)


def _subs(spec, seed):
    rng = np.random.default_rng(seed)
    return [synthetic.random_sub_batch(rng, [TABLE[i] for i in seq], B, 4) for seq, B in spec]


def _reference(key, net, subs):
    """The float64 restatement on the network's parameters (cached per key: every precision builds the same weights)."""
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    if key not in _cache or not all(torch.equal(params[k], v) for k, v in _cache[key][0].items()):
        res = lstm_fp64.loss_and_grads(params, subs, list(OBS), IN_DIMS, K)
        _cache[key] = (params, res, lstm_fp64.lstm_term_magnitudes(res))
    return _cache[key][1], _cache[key][2]


def _run(net, subs, profile=False):
    """One training forward (with per-row log q) and backward on the network's own workspace -> (loss, row log q, the
    gradient arena, the encoding, kernel names)."""
    from torch.profiler import ProfilerActivity, profile as prof_ctx
    enc = synthetic.ArrayBatch(subs).encode(net)
    lp = torch.full((enc.n_rows,), float('nan'), device='cuda')
    grad = torch.zeros_like(net._arena.data)
    names = []

    def go():
        loss = net._forward_native(enc, want_grad=True, row_lp=lp)
        net._backward_native(enc, grad, 1.0)
        torch.cuda.synchronize()
        return loss
    if profile:
        with prof_ctx(activities=[ProfilerActivity.CUDA]) as prof:
            loss = go()
        names = [e.key for e in prof.key_averages() if e.device_time_total > 0]
    else:
        loss = go()
    assert int(net._last_status.item()) == 0
    return float(loss), lp.cpu().double(), grad, enc, names


def _forms(names):
    """Kernel names -> the LSTM and cell-backward forms they show."""
    out = set()
    for n in names:
        m = re.search(r'k_lstm_cluster<\w+, (\d+), (\d+)>', n)
        if m:
            out.add(('cluster', int(m.group(1)), int(m.group(2))))
        m = re.search(r'k_cell_bwd<(\w+)>', n)
        if m:
            out.add('cell_bwd_' + m.group(1))
        for k in ('k_lstm_step', 'k_cell_fwd', 'k_pack_rows', 'k_grouped'):
            if re.search(r'\b' + k + r'\b', n):
                out.add(k)
        if re.search(r'\btc[glcp]::', n):
            out.add('tensor_core')
    return out


def _check_forms(names, lstm_forms, cell_bwd, fused=True):
    got = _forms(names)
    if not lstm_forms:   # fp32 SIMT path
        assert 'tensor_core' not in got, names
        return
    lstm = {f for f in got if f == 'k_lstm_step' or (isinstance(f, tuple) and f[0] == 'cluster')}
    if fused:   # (t = 0 has no recurrent GEMM: its cell is k_cell_fwd either way)
        assert lstm == {('k_lstm_step' if f == STEP else f) for f in lstm_forms}, (lstm, names)
    else:
        assert not lstm and {'k_grouped', 'k_cell_fwd'} <= got, names
    # B % 128 == 0: the t = 0 launch is k_cell_bwd<true>, the later ones k_cell_bwd<false>
    assert ('cell_bwd_true' in got) == (cell_bwd == 'true') and 'cell_bwd_false' in got, names


def _per_row(err, want):
    """Worst error of a gradient tensor against the largest entry of its own output row (32-element block of a vector),
    floored at 1e-3 of the tensor's largest entry."""
    rows = (lambda x: x.reshape(x.size(0), -1)) if want.dim() > 1 else \
        (lambda x: torch.nn.functional.pad(x, (0, -x.numel() % 32)).view(-1, 32))
    scale = torch.clamp(rows(want.abs()).max(1, keepdim=True).values, min=1e-3 * float(want.abs().max()) + 1e-30)
    return float((rows(err) / scale).max())


def _truncated_head(name):
    """Parameters of a proposal head whose mixture is truncated normal (Uniform, Poisson): their gradients cancel over the
    rows of a minibatch, so the fp32 rounding of their terms shows at a larger share of a row."""
    return any(name.startswith('_layers_proposal.{}.'.format(a)) for a, fam, _ in TABLE if fam in ('Uniform', 'Poisson'))


def _abs_err(got, want):
    """|got - want| with NaN as +inf: a NaN that reaches a result (an unwritten or poisoned row) fails every tolerance,
    where torch's max and norm would turn it into a NaN that Python's max() then drops."""
    return torch.nan_to_num((torch.as_tensor(got, dtype=torch.float64) - want).abs(), nan=math.inf)


def errors(net, subs, enc, loss, lp, grad, ref, M):
    """Worst error of each observable in units of its tolerance scale:
      lq        log q of every (t, row) and the loss, against 1 + |want|
      lstm      LSTM weight / bias gradients per element, against their term magnitudes M
      lstm_row  the same gradients per row (_per_row)
      trunc     truncated-normal head gradients per row
      other     every other gradient per row
      norm      every other gradient tensor: ||got - want|| / ||want|| (an all-zero or halved tensor fails it)
      norm_trunc  the same for the truncated-normal head tensors"""
    a = enc.arrays
    out = dict.fromkeys(('lq', 'lstm', 'lstm_row', 'trunc', 'other', 'norm', 'norm_trunc'), 0.0)
    out['lq'] = float(_abs_err(loss, ref['loss'])) / (1 + abs(float(ref['loss'])))
    for pos, s in enumerate(enc.sub_order):
        want = ref['lps'][s]
        T, B = want.shape
        for t in range(T):
            st = int(np.nonzero(a['step_t'] == t)[0][0]) + pos   # the steps of one t follow the sorted sub-batch order
            assert a['step_nrows'][st] == B
            r0 = int(a['step_row0'][st])
            got = lp[r0:r0 + B]
            out['lq'] = max(out['lq'], float((_abs_err(got, want[t]) / (1 + want[t].abs())).max()))
    for k, want in ref['grads'].items():
        got = net.grad_view(k, grad).cpu().double()
        err = _abs_err(got, want)
        nk = 'norm_trunc' if _truncated_head(k) else 'norm'
        out[nk] = max(out[nk], float(err.norm()) / max(float(want.norm()), 1e-12))
        if k in M:
            floor = 1e-9 * float(M[k].max())
            out['lstm'] = max(out['lstm'], float((err / (M[k] + floor)).max()))
            out['lstm_row'] = max(out['lstm_row'], _per_row(err, want))
        else:
            key = 'trunc' if _truncated_head(k) else 'other'
            out[key] = max(out[key], _per_row(err, want))
    assert all(math.isfinite(v) for v in out.values()), out
    return out


def check(got, precision, keys=('lq', 'lstm', 'trunc', 'other', 'norm', 'norm_trunc')):
    assert all(got[k] <= TOL[precision][k] for k in keys), ({k: got[k] for k in keys}, TOL[precision])


def _case(name, precision, fused=True, seed=11):
    H, S, spec, forms = CASES[name]
    net = _network(H, S, precision, seed)
    subs = _subs(spec, seed)
    ref, M = _reference(name, net, subs)
    loss, lp, grad, enc, names = _run(net, subs, profile=True)
    _check_forms(names, forms if precision != 2 else set(), CELL_BWD[name], fused)
    check(errors(net, subs, enc, loss, lp, grad, ref, M), precision)


@pytest.mark.parametrize('precision', [0, 1, 2])
@pytest.mark.parametrize('name', [n for n in CASES if n != 'h100'])
def test_recurrence_vs_fp64(cuda, name, precision):
    _case(name, precision)


def test_h_not_a_multiple_of_32_vs_fp64(cuda):
    """H = 100: the fp32 SIMT path trains it (no tensor-core kernel at all) and is right; the tensor-core path refuses it
    rather than fall back."""
    _case('h100', 2)
    H, S, spec, _ = CASES['h100']
    with pytest.raises(RuntimeError, match='multiple of 32'):
        _run(_network(H, S, 0, 11), _subs(spec, 11))


@pytest.mark.parametrize('precision', [0, 1])
@pytest.mark.parametrize('name', ['h128', 'ragged'])
def test_unfused_step_vs_fp64(cuda, monkeypatch, name, precision):
    monkeypatch.setenv('PPB_FUSED_CELL', '0')    # read when the native network handle is created
    _case(name, precision, fused=False)


@pytest.mark.parametrize('precision', [0, 1, 2])
def test_saturated_gates_vs_fp64(cuda, precision):
    """W_ih and the biases scaled so that gate pre-activations reach |x| ~ 30: f ~ 1, c grows over T = 100 steps (CS = 4).
    W_hh keeps its size: scaled with them the recurrence is chaotic and fp32 rounding alone moves log q by O(1)."""
    H, spec, seed = 256, [(_cycle(100), 128)], 5
    net = _network(H, 4, precision, seed)
    for k in ('_layers_lstm.weight_ih_l0', '_layers_lstm.bias_ih_l0', '_layers_lstm.bias_hh_l0'):
        net.view(k).mul_(60.0)
    subs = _subs(spec, seed)
    ref, M = _reference('saturated', net, subs)
    pre = torch.cat([s['pre'].abs().flatten() for s in ref['steps'][0]])
    assert float(pre.max()) > 30 and float((pre > 10).double().mean()) > 0.1
    assert float(ref['steps'][0][-1]['c'].abs().max()) > 20
    loss, lp, grad, enc, names = _run(net, subs, profile=True)
    _check_forms(names, {CS4} if precision != 2 else set(), 'true')
    # fp32 rounds sigmoid(x) to 1 above x = 17, so sigmoid' is 0 there in any fp32 evaluation and a unit saturated at every
    # step has an exactly zero gradient where fp64 has one of 1e-13 of its terms: the term-magnitude model would fail on
    # representation, not on a kernel (seen as error = M at precisions 0 and 2 alike); per-row scaling still holds every
    # row that carries gradient
    check(errors(net, subs, enc, loss, lp, grad, ref, M), precision, keys=('lq', 'lstm_row', 'trunc', 'other', 'norm', 'norm_trunc'))


@pytest.mark.parametrize('precision', [0, 2])
def test_workspace_reuse_and_poison_vs_fp64(cuda, precision):
    """One network on one workspace: a large ragged batch, a small one, a no-grad forward of a larger batch whose buffers
    lie over the small batch's backward lists, the small batch again, a differently ragged one, then a batch after the
    whole workspace was filled with NaN and with large finite values: every training result against float64.  No call
    reads workspace memory it did not write, apart from the problem lists uploaded there, which are sent again when the
    layout changes (forget_on_new_layout, net.cu) or the caller says the memory changed (ppb_net_forget_uploads)."""
    H, seed = 256, 13
    net = _network(H, 4, precision, seed)
    specs = [CASES['ragged'][2], [([0, 1], 5)], [(_cycle(5, 3), 130), (_cycle(2, 1), 260), (_cycle(9, 5), 1)],
             [(_cycle(4, 6), 129), (_cycle(6), 33)]]
    subs = [_subs(spec, seed + i) for i, spec in enumerate(specs)]
    plan = [(0, None), (1, None), (2, 'no_grad'), (1, None), (2, None), (3, float('nan')), (3, 3.0e38), (3, -1.0e30)]
    for i, fill in plan:
        if fill == 'no_grad':
            net.row_log_probs(synthetic.ArrayBatch(subs[i]))
            continue
        ref, M = _reference(('reuse', i), net, subs[i])
        if fill is not None:
            net._ensure_workspace(synthetic.ArrayBatch(subs[i]).encode(net))
            ws = net._workspace
            ws[:ws.numel() // 4 * 4].view(torch.float32).fill_(fill)
            _lib.call('ppb_net_forget_uploads', net._handle)   # the problem lists the workspace held are gone
        loss, lp, grad, enc, _ = _run(net, subs[i])
        check(errors(net, subs[i], enc, loss, lp, grad, ref, M), precision)


@pytest.mark.parametrize('H', [100, 128])
def test_infer_step_vs_fp64(cuda, H):
    """ppb_ic_infer_step at precision 0 over seven sites of every family: at H % 32 != 0 it takes the fp32 SIMT GEMMs (no
    tensor-core kernel), at H = 128 the tensor cores.  h and c of 300 particles after every step against
    lstm_fp64.infer_steps, |got - want| <= tau (1 + |want|)."""
    from torch.profiler import ProfilerActivity, profile
    n, seed = 300, 17
    net = _network(H, 4, 0, seed)
    gen = torch.Generator().manual_seed(seed)
    obs = {'o0': torch.randn(3, generator=gen), 'o1': torch.randn(1, generator=gen)}
    seq = [TABLE[i] for i in _cycle(8, 2)]
    sb = synthetic.random_sub_batch(np.random.default_rng(seed), seq, n, 4)
    h, c = torch.zeros(n, H, device='cuda'), torch.zeros(n, H, device='cuda')
    got = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        net._infer_init(obs)
        for t, (a, fam, C) in enumerate(seq):
            prev_a = seq[t - 1][0] if t else None
            prev_v = torch.from_numpy(sb['values'][t - 1]).cuda() if t else None
            p0, p1 = (torch.from_numpy(sb[k][t]).cuda() for k in ('prior0', 'prior1'))
            net._infer_step_lanes(a, p0, p1, n, prev_a, prev_v, h, c)
            got.append((h.cpu().double(), c.cpu().double()))
    names = [e.key for e in prof.key_averages() if e.device_time_total > 0]
    assert ('tensor_core' in _forms(names)) == (H % 32 == 0), names
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    steps = [{'address': a, 'family': f, 'num_categories': C, 'prev_value': sb['values'][t - 1] if t else None}
             for t, (a, f, C) in enumerate(seq)]
    want = lstm_fp64.infer_steps(params, torch.cat([obs['o0'], obs['o1']]), list(OBS), IN_DIMS, steps, n=n)
    worst = max(float((_abs_err(g, w) / (1 + w.abs())).max()) for gw, ww in zip(got, want) for g, w in zip(gw, ww))
    check({'infer': worst}, 0, keys=('infer',))


# ---- the cell activations, element by element through the infer step's k_cell_infer ------------------------------------
def _sweep_points():
    pts = [np.linspace(-100, 100, 4001), [0.0, 1e-30, -1e-30, 1e-7, -1e-7]]
    for c, w in ((0.25, 2e-3), (17.0, 0.05), (88.0, 0.5), (89.0, 0.5), (1.0, 0.05), (5.0, 0.05)):
        for s in (1, -1):
            pts.append(s * c + np.linspace(-w, w, 401))
    return np.unique(np.concatenate(pts).astype(np.float32))


def _cell_through_infer_step(pre, precision):
    """pre [N, 4] fp32 gate pre-activations (i, f, g, o) -> (c, h) of one infer step from h = c = 0, one unit per point:
    W_ih = W_hh = 0 and b_ih = the pre-activations, b_hh = 0."""
    H = 512
    net = synthetic.build_network({'o0': {'dim': 4, 'depth': 1}}, [1], [('a', 'Normal', 0)], lstm_dim=H,
                                  mixture_components=2, precision=precision)
    for k in ('_layers_lstm.weight_ih_l0', '_layers_lstm.weight_hh_l0', '_layers_lstm.bias_hh_l0'):
        net.view(k).zero_()
    net._infer_init({'o0': torch.zeros(1)})
    cs, hs = [], []
    for i in range(0, len(pre), H):
        chunk = np.zeros((H, 4), np.float32)
        n = min(H, len(pre) - i)
        chunk[:n] = pre[i:i + n]
        net.view('_layers_lstm.bias_ih_l0').copy_(torch.from_numpy(chunk.T.copy().reshape(-1)))
        h, c = torch.zeros(1, H, device='cuda'), torch.zeros(1, H, device='cuda')
        net._infer_step_lanes('a', 0.0, 1.0, 1, None, None, h, c)
        cs.append(c[0, :n].cpu().double())
        hs.append(h[0, :n].cpu().double())
    return torch.cat(cs), torch.cat(hs)


# Relative error of ppb_cell_sigmoid and ppb_cell_tanh over the sweep, about 2x what one NVIDIA H100 80GB HBM3 showed
# (DESIGN §8): sigmoid 1.5e-7 for x >= -1, growing as 4.5e-8 to 6.7e-8 |x| below (3.8e-6 at x = -84), the fp32 rounding
# of x log2(e) before ex2; tanh 3.7e-7, at |x| just above 0.25 where 1 - 2 / (1 + exp(2|x|)) takes over.
SIGMOID_REL = (3e-7, 1.2e-7)   # a + b |x| for x < 0; a for x >= 0
TANH_REL = 1e-6


def activation_errors(precision):
    x = torch.from_numpy(_sweep_points()).double()
    big = torch.full_like(x, 100.0)
    tiny = 2.0 ** -126   # below the smallest normal fp32 (the approximations flush to zero there): absolute error
    out = {}
    # tanh: i = o = sigmoid(100) = 1, so c = tanh(x) and h = tanh(c)
    c, h = _cell_through_infer_step(torch.stack([big, big, x, big], 1).float().numpy(), precision)
    want = torch.tanh(x)
    out['tanh'] = (x, (c - want).abs() / torch.clamp(want.abs(), min=tiny), want)
    out['tanh_h'] = (c, (h - torch.tanh(c)).abs() / torch.clamp(torch.tanh(c).abs(), min=tiny), torch.tanh(c))
    # sigmoid: g = tanh(100) = 1, so c = sigmoid(x); o = sigmoid(x) too
    c, h = _cell_through_infer_step(torch.stack([x, big, big, x], 1).float().numpy(), precision)
    want = torch.sigmoid(x)
    out['sigmoid'] = (x, (c - want).abs() / torch.clamp(want, min=tiny), want)
    return out


@pytest.mark.parametrize('precision', [0, 2])
def test_cell_activations_vs_fp64(cuda, precision):
    err = activation_errors(precision)
    x, e, want = err['sigmoid']
    bound = torch.where(x < 0, SIGMOID_REL[0] + SIGMOID_REL[1] * x.abs(), torch.full_like(x, SIGMOID_REL[0]))
    bound = torch.where(want < 2.0 ** -126, torch.ones_like(x), bound)   # no more than the smallest normal fp32 off
    assert bool((e <= bound).all()), (float(x[(e / bound).argmax()]), float((e / bound).max()))
    for k in ('tanh', 'tanh_h'):
        x, e, _ = err[k]
        assert bool((e <= TANH_REL).all()), (k, float(x[e.argmax()]), float(e.max()))
