"""GPU: the observe embedding of the training step, in each of its three forms, against the float64 restatement
(tests/obs_fp64.py driven by tests/lstm_fp64.py, or by the feed-forward loss for that network).

Each case asserts, from the kernel names torch.profiler records, the form it is meant to reach (obs_weight_images in
obs_embed.inc; the fp32 pipeline, precision 2, always runs the SIMT chain):
  fused        obsmlp::k_fwd and obsmlp::k_bwd (obs_fused_ok: every layer at most 96 wide, the plan within kMaxSmem)
  tensor_core  k_pack_rows_masked, the start of its backward (obs_tc_ok)
  simt         neither
The shapes aim at the branches of each form: widths that are not multiples of four floats (Layer::pitch), 96 and 97 (the
widest fused and the narrowest that leaves it), the largest plan obsmlp::smem_fwd / smem_bwd accept and the smallest they
refuse, batches around kMT = 4 traces per chunk, one trace per SM (132) and past it, backward grids rounded up to whole
8-CTA clusters; for the tensor-core form B % 128 == 0 and != 0 at one row tile and at many, hidden widths that are not
multiples of 32, widths above 128 and E = 256, and a last observable whose width is not a multiple of 32 (its dx and dW read
the concatenated gradient at its own column offset).

Observables and tolerances (TOL, per precision; tau is about 4x the worst error seen on one NVIDIA H100 80GB HBM3 at
700 W):
  lq     log q of every (t, row) and the loss: |got - want| <= tau (1 + |want|)
  obs    every observe-embedding weight and bias gradient, per element: |got - want| <= tau (M + 1e-6 max M) + bound, M the
         term magnitudes (obs_fp64.term_magnitudes) and bound what units within rounding of zero can move when they take
         the other side of their ReLU (obs_fp64.relu_flip_bound, REL below)
  wih    W_ih[:, :E] (the LSTM reads the embedding through it; its gradient reduces over the embedding's tile images), per
         element against its own M (lstm_fp64.lstm_term_magnitudes)
  norm   ||got - want|| / ||want|| of each of those tensors: below 1, so a tensor that is zero, halved or of the wrong sign
         fails at every precision
  infer  ppb_ic_embed_observe, per element against the largest entry of its row
Worst seen (precision 0 / 1 / 2; precision 1 runs two cases):
  lq     8.8e-7 (workspace, SIMT form) / 1.3e-4 (tc2 700/300/101) / 1.2e-6 (narrow, B = 1100)
  obs    1.0e-3 (workspace, tensor-core form, B = 8) / 0.17 (tc2 700/300/101) / 2.0e-4 (tc_wide)
  wih    1.5e-4 (workspace, tensor-core form) / 3.6e-2 / 8.6e-5 (narrow, B = 5)
  norm   1.8e-4 (tc2 512/300/101) / 1.2e-2 / 4.0e-3 (tc2 700/300: the fp32 chain flips the unit below, and the norm
         check carries no flip bound)
  infer  3.6e-7 (tc2, n = 300)
The 700/300/101 batch holds 45 ambiguous units at REL = 2e-5 (8574 at precision 1's REL).  Per element, M counts |dz|, not
the terms dz itself sums: below the top layer dz cancels, and its rounding shows at 1e-4..1e-3 of M in every form.
What the flip bound lets through, on that batch: at precisions 0 and 2 up to 15 % of max |g| on some elements of the first
layers (b._layers.0.weight; below 0.4 % on the final chain), so the per-element check is tight everywhere but where
ambiguous units sit.  At precision 1 the bound is 0.8 to 70 times max |g| on every layer below the final chain and exceeds
|g| on 70 to 100 % of their elements: there the per-element obs check (with tau 0.7) constrains nothing, and the norm check
(0.05) is the only check of the observe-embedding gradients.  The two precision-1 cases only show that single-pass TF32
reaches the right tensors.

The former strict xfail of test_obs_mlp_gpu.py (the tensor-core form on a 700/300/101 batch, observe-embedding gradients
8e-3 of their maximum from the fp32 oracle) was a ReLU flip, not a kernel fault: trace 508 of the 700-trace sub-batch holds a
unit of the final chain's first layer at z = 3.4e-9 in float64 that fp32 rounding puts at -1.5e-8, so the fp32 oracle drops
the unit's whole gradient.  The fp32 oracle is 8.2e-3 of the maximum away from float64 there by itself; the kernels agree
with float64 to rounding plus the bound of that unit (test_former_xfail_is_a_relu_flip).
"""
import math

import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from pyprob_b200 import _lib, synthetic
from pyprob_b200.util import InferenceNetwork
from tests import lstm_fp64, obs_fp64

pytestmark = pytest.mark.gpu

TABLE = [('a_u', 'Uniform', 0), ('a_c', 'Categorical', 5), ('a_n', 'Normal', 0), ('a_p', 'Poisson', 0)]
SEQS = ([0, 1, 2, 3], [2, 0], [1])
H, K = 64, 3
W_IH = '_layers_lstm.weight_ih_l0'

TOL = {0: dict(lq=3.5e-6, obs=4e-3, wih=6e-4, norm=7e-4, infer=1.5e-6),
       1: dict(lq=5e-4, obs=0.7, wih=0.15, norm=0.05),
       2: dict(lq=5e-6, obs=8e-4, wih=3.5e-4, norm=1.6e-2)}
# relative rounding of a pre-activation against |x| |W|^T + |b|: fp32 and 3xTF32 GEMMs, and single-pass TF32 (10-bit operands)
REL = {0: 2e-5, 1: 4e-3, 2: 2e-5}

# name: (observe embeddings, input dims, seed, form at precisions 0 and 1)
NETS = {
    # widths 1, 3 and 30 (rows of 1, 3 and 30 floats), depths 1 to 3
    'narrow': ({'o_a': {'dim': 1, 'depth': 1}, 'o_b': {'dim': 3, 'depth': 2}, 'o_c': {'dim': 30, 'depth': 3}}, [2, 5, 3], 3,
               'fused'),
    'w96': ({'o': {'dim': 96}}, [4], 7, 'fused'),                   # E = 96: the widest the fused kernels take
    'w97': ({'o': {'dim': 97}}, [4], 7, 'tensor_core'),             # E = 97 leaves the fused form
    # two depth-4 chains of width 48: 232280 bytes of shared memory, the largest such plan within kMaxSmem (232448) ...
    'smem_max': ({'a': {'dim': 48, 'depth': 4}, 'b': {'dim': 48, 'depth': 4}}, [9, 20], 9, 'fused'),
    # ... and with an 8-wide input (its rows padded by four floats) 232488 bytes; a 28-wide hidden layer rules out the
    # tensor-core form
    'smem_min': ({'a': {'dim': 48, 'depth': 4}, 'b': {'dim': 48, 'depth': 4}}, [8, 20], 9, 'simt'),
    # the shapes of test_obs_mlp_gpu.py (same seed, same draws): E = 160, 'b' starts at column 64
    'tc2': ({'a': {'dim': 64, 'depth': 2}, 'b': {'dim': 96, 'depth': 3}}, [40, 3], 31, 'tensor_core'),
    # hidden widths 40 and 100, and a last observable 100 wide at column 64
    'tc_odd': ({'a': {'dim': 64, 'depth': 3}, 'b': {'dim': 100, 'depth': 2}}, [16, 100], 13, 'tensor_core'),
    # widths 146 and 256 (several N tiles), E = 256
    'tc_wide': ({'a': {'dim': 192, 'depth': 3}, 'b': {'dim': 64, 'depth': 2}}, [100, 8], 17, 'tensor_core'),
    'tc_e256': ({'obs': {'dim': 256}}, [1], 19, 'tensor_core'),     # the configs[3] embedding
    # a depth-1 chain in an embedding too wide to fuse; a 21-wide hidden layer (obs_tc_ok wants in_dim >= 32)
    'simt_d1': ({'a': {'dim': 100, 'depth': 1}, 'b': {'dim': 20, 'depth': 2}}, [3, 5], 41, 'simt'),
    'simt_in': ({'a': {'dim': 40, 'depth': 2}, 'b': {'dim': 64, 'depth': 2}}, [3, 1], 43, 'simt'),
}
FUSED_B = [(1,), (3,), (4,), (5,), (131,), (132,), (133,), (1100,)]
CASES = [('narrow', s) for s in FUSED_B] + [
    ('w96', (133,)), ('w96', (700, 300, 101)), ('w97', (133,)), ('smem_max', (133,)), ('smem_min', (133,)),
    ('tc2', (128,)), ('tc2', (129,)), ('tc2', (1024,)), ('tc2', (512, 300, 101)), ('tc2', (700, 300, 101)),
    ('tc2', (700, 300)), ('tc_odd', (256,)), ('tc_odd', (300, 40)), ('tc_wide', (129,)), ('tc_e256', (256,)),
    ('tc_e256', (300,)), ('simt_d1', (129,)), ('simt_d1', (700, 300, 101)), ('simt_in', (133,))]

_cache = {}


def _network(name, precision, feedforward=False):
    emb, in_dims, seed, _ = NETS[name]
    kw = {'inference_network': InferenceNetwork.FEEDFORWARD} if feedforward else {}
    return synthetic.build_network(emb, in_dims, TABLE, lstm_dim=H, mixture_components=K, seed=seed, precision=precision,
                                   **kw)


def _subs(name, sizes, seed=None):
    """The sub-batches test_obs_mlp_gpu._run draws for these sizes."""
    emb, in_dims, s, _ = NETS[name]
    rng = np.random.default_rng(s if seed is None else seed)
    return [synthetic.random_sub_batch(rng, [TABLE[i] for i in SEQS[i % 3]], b, sum(in_dims)) for i, b in enumerate(sizes)]


def _reference(key, net, subs, feedforward=False):
    """float64 loss, log q and gradients, the observe-embedding term magnitudes and, per precision, the ReLU-flip bound
    (cached per key: every precision builds the same weights)."""
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    if key not in _cache or not all(torch.equal(params[k], v) for k, v in _cache[key][0].items()):
        emb = NETS[key[0]][0]
        res = obs_fp64.loss_and_grads(params, subs, list(emb), NETS[key[0]][1], K, feedforward=feedforward)
        M = obs_fp64.term_magnitudes(res)
        if not feedforward:
            M[W_IH] = lstm_fp64.lstm_term_magnitudes(res)[W_IH]
        bounds = {p: obs_fp64.relu_flip_bound(params, res, REL[p]) for p in REL}
        _cache[key] = (params, res, M, bounds)
    return _cache[key][1:]


def _run(net, subs, poison=None):
    """One training forward (with per-row log q) and backward -> (loss, row log q, gradient arena, encoding, kernel
    names).  poison: fill the whole workspace with this value first (the uploaded problem lists are then sent again)."""
    enc = synthetic.ArrayBatch(subs).encode(net)
    if poison is not None:
        net._sync_native()
        net._ensure_workspace(enc)
        ws = net._workspace
        ws[:ws.numel() // 4 * 4].view(torch.float32).fill_(poison)
        _lib.call('ppb_net_forget_uploads', net._handle)
    lp = torch.full((enc.n_rows,), float('nan'), device='cuda')
    grad = torch.zeros_like(net._arena.data)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        loss = net._forward_native(enc, want_grad=True, row_lp=lp)
        net._backward_native(enc, grad, 1.0)
        torch.cuda.synchronize()
    assert int(net._last_status.item()) == 0
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return float(loss), lp.cpu().double(), grad, enc, names


def form_of(names):
    fused = [any('obsmlp::k_fwd' in n for n in names), any('obsmlp::k_bwd' in n for n in names)]
    tc = any('k_pack_rows_masked' in n for n in names)
    if fused == [True, True] and not tc:
        return 'fused'
    if not any(fused):
        return 'tensor_core' if tc else 'simt'
    return ('mixed', fused, tc)


def _abs_err(got, want):
    """|got - want| with NaN as +inf: a NaN that reaches a result (an unwritten or poisoned row) fails every tolerance,
    where torch's max and norm would turn it into a NaN that Python's max() then drops."""
    return torch.nan_to_num((torch.as_tensor(got, dtype=torch.float64) - want).abs(), nan=math.inf)


def errors(net, enc, loss, lp, grad, ref, M, bound):
    """Worst error of each observable in units of its tolerance scale (see the module docstring).  A NaN anywhere in a
    compared result counts as an infinite error."""
    out = dict.fromkeys(('lq', 'obs', 'wih', 'norm'), 0.0)
    out['lq'] = float(_abs_err(loss, ref['loss'])) / (1 + abs(float(ref['loss'])))
    a = enc.arrays
    for pos, s in enumerate(enc.sub_order):
        want = ref['lps'][s]
        T, B = want.shape
        for t in range(T):
            st = int(np.nonzero(a['step_t'] == t)[0][0]) + pos   # the steps of one t follow the sorted sub-batch order
            assert a['step_nrows'][st] == B
            r0 = int(a['step_row0'][st])
            out['lq'] = max(out['lq'], float((_abs_err(lp[r0:r0 + B], want[t]) / (1 + want[t].abs())).max()))
    E = net._observe_embedding_dim
    for k, m in M.items():
        want = ref['grads'][k]
        got = net.grad_view(k, grad).cpu().double()
        if k == W_IH:
            want, got, m = want[:, :E], got[:, :E], m[:, :E]
        err = _abs_err(got, want)
        out['norm'] = max(out['norm'], float(err.norm()) / max(float(want.norm()), 1e-30))
        scale = m + 1e-6 * float(m.max()) + 1e-30
        if k == W_IH:
            out['wih'] = max(out['wih'], float((err / scale).max()))
        else:
            out['obs'] = max(out['obs'], float(((err - bound[k]).clamp_min(0) / scale).max()))
    assert all(math.isfinite(v) for v in out.values()), out
    return out


def check(got, precision, keys=('lq', 'obs', 'wih', 'norm')):
    assert all(got[k] <= TOL[precision][k] for k in keys), ({k: got[k] for k in keys}, TOL[precision])


def _case(name, sizes, precision, feedforward=False, poison=None, net=None):
    net = net or _network(name, precision, feedforward)
    subs = _subs(name, sizes)
    ref, M, bounds = _reference((name, sizes, feedforward), net, subs, feedforward)
    loss, lp, grad, enc, names = _run(net, subs, poison)
    want_form = 'simt' if precision == 2 else NETS[name][3]
    assert form_of(names) == want_form, (want_form, sorted(set(names)))
    got = errors(net, enc, loss, lp, grad, ref, M, bounds[precision][0])
    check(got, precision, ('lq', 'obs', 'norm') if feedforward else ('lq', 'obs', 'wih', 'norm'))
    return got, bounds[precision][1]


@pytest.mark.parametrize('precision', [0, 2])
@pytest.mark.parametrize('name,sizes', CASES)
def test_form_vs_fp64(cuda, name, sizes, precision):
    _case(name, sizes, precision)


@pytest.mark.parametrize('name,sizes', [('tc2', (700, 300, 101)), ('narrow', (133,))])
def test_tf32_vs_fp64(cuda, name, sizes):
    _case(name, sizes, 1)


def test_fused_plan_boundary():
    """smem_max and smem_min sit on either side of kMaxSmem by the sizing of obs_plan_of (restated here)."""
    def smem(emb, in_dims):
        def dims(i, o, depth):
            h = (i + o) // 2
            return [(i, o)] if depth == 1 else [(i, h)] + [(h, h)] * (depth - 2) + [(h, o)]
        E = sum(s['dim'] for s in emb.values())
        chains = [dims(d, s['dim'], s.get('depth', 2)) for s, d in zip(emb.values(), in_dims)]
        fin = dims(E, E, 2)
        w = part = 0
        for i, o in [x for c in chains + [fin] for x in c]:
            w += (o * (i if (i & 3) or (i & 7) else i + 4) + o + 3) & ~3
            part += o * i + o
        A = sum(i for c in chains for i, _ in c) + E + sum(o for _, o in fin)
        Dz = sum(o for c in chains for _, o in c[:-1]) + E + sum(o for _, o in fin)
        return 4 * (w + 4 * A), 4 * (w + part + 4 * (A + Dz))
    k_max = 227 * 1024
    assert max(smem(*NETS['smem_max'][:2])) == 232280 <= k_max < max(smem(*NETS['smem_min'][:2])) == 232488


def test_former_xfail_is_a_relu_flip(cuda):
    """The 700/300/101 batch on the tensor-core form: the fp32 oracle's distance from float64 is the flip of a unit within
    rounding of zero, and the kernels stay inside the bound of such units."""
    name, sizes = 'tc2', (700, 300, 101)
    net = _network(name, 0)
    ref, M, bounds = _reference((name, sizes, False), net, _subs(name, sizes))
    bound, n_amb = bounds[0]
    assert 0 < n_amb < 200, n_amb
    z = [L for L in ref['obs'][0] if L['name'] == '_layers_observe_embedding_final._layers.0'][0]['z']
    assert abs(float(z[508, 121])) < 1e-8
    _case(name, sizes, 0, net=net)


FORM_NETS = {'fused': 'narrow', 'tensor_core': 'tc2', 'simt': 'simt_d1'}


@pytest.mark.parametrize('form', list(FORM_NETS))
def test_workspace_reuse_and_poison_vs_fp64(cuda, form):
    """One network per form on one workspace, batches with B % 128 != 0: a ragged batch, a small one, the ragged one again,
    then the small one after the whole workspace was filled with NaN and with large finite values (ppb_net_forget_uploads:
    the problem lists the workspace held are gone).  Every result against float64."""
    name = FORM_NETS[form]
    net = _network(name, 0)
    for sizes, poison in [((700, 300, 101), None), ((5, 3), None), ((700, 300, 101), None), ((5, 3), float('nan')),
                          ((133,), 3.0e38), ((133,), float('nan')), ((133,), -1.0e30)]:
        _case(name, sizes, 0, poison=poison, net=net)


@pytest.mark.parametrize('poison', [None, float('nan')])
def test_feedforward_vs_fp64(cuda, poison):
    """The feed-forward network shares obs_embed.inc: its tensor-core form on a ragged batch, on a fresh and on a
    NaN-filled workspace."""
    _case('tc2', (700, 300, 101), 0, feedforward=True, poison=poison)


@pytest.mark.parametrize('n', [1, 300])
@pytest.mark.parametrize('name', ['narrow', 'tc2'])
def test_infer_embed_vs_fp64(cuda, name, n):
    """ppb_ic_embed_observe (the fp32 chain whatever the training form) on n observation rows against the float64
    forward."""
    emb, in_dims, seed, _ = NETS[name]
    net = _network(name, 0)
    net._sync_native()
    obs = torch.randn(n, sum(in_dims), generator=torch.Generator().manual_seed(seed))
    need = net._infer_workspace(n)
    out = torch.full((n, net._observe_embedding_dim), float('nan'), device='cuda')
    obs_d = obs.cuda()
    _lib.call('ppb_ic_embed_observe', net._handle, _lib.ptr(net._arena.data), _lib.ptr(obs_d), _lib.ptr(out), n,
              _lib.ptr(net._infer_ws), need, _lib.stream())
    params = {k: v.cpu().double() for k, v in net.reference_state_dict().items()}
    want = obs_fp64.embed(params, obs.double(), list(emb), in_dims, [])
    err = _abs_err(out.cpu().double(), want) / (want.abs().max(1, keepdim=True).values + 1e-30)
    check({'infer': float(err.max())}, 0, keys=('infer',))
