"""The observe embedding in each of its three forms under the tensor-core pipeline (precision 0), at shapes the workload
tests do not reach.  Loss and every gradient are checked against the oracle.

- fused (obs_mlp.cuh): three observables with input dims above one, chain depths 1 to 3, widths up to 96 (rows that are
  and are not multiples of four floats), and batches from one trace to more traces than there are SMs; and a shape the
  tensor-core form would also take, which must still run the fused kernels;
- tensor-core: two observables of depths 2 and 3, with one sub-batch and with three ragged ones; each gradient element may
  also differ by what ReLU flips can move it (obs_fp64.relu_flip_bound): the 700/300/101 batch holds a unit of the final
  chain at z = 3.4e-9 that the fp32 oracle rounds to the other side of its ReLU (tests/test_obs_embed_fp64_gpu.py);
- SIMT: an observable of depth 1 (the tensor-core form needs two layers per chain) in an embedding too wide to fuse.
Each of these cases also checks from the kernels of the step that it ran the form it is meant to test, and the fused form
is checked to carve no tile images for the observe-embedding layers."""
import numpy as np
import pytest
import torch
from torch.profiler import ProfilerActivity, profile

from oracle import network as onet
from pyprob_b200 import _lib, synthetic
from tests import obs_fp64

pytestmark = pytest.mark.gpu

TABLE = [('a_u', 'Uniform', 0), ('a_c', 'Categorical', 5), ('a_n', 'Normal', 0), ('a_p', 'Poisson', 0)]


def _check(net, batch, observe_names, observe_in_dims, K, rtol=1e-4, flips=False):
    """flips: each gradient element may also differ by obs_fp64.relu_flip_bound (units within fp32 rounding of zero may
    land on either side of their ReLU, in the oracle as in the kernels)"""
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in batch.subs]
    want_loss, want_grads, _ = onet.loss_and_grads(params, tsubs, observe_names, observe_in_dims, K)
    bound = {}
    if flips:
        bound, _ = obs_fp64.relu_flip_bound(params, obs_fp64.loss_and_grads(params, tsubs, observe_names, observe_in_dims, K),
                                            2e-5)
    ok, loss = net._loss(batch)
    assert ok
    assert abs(float(loss.detach()) - float(want_loss)) <= rtol * abs(float(want_loss))
    loss.backward()
    bad = {}
    for k, g in want_grads.items():
        got = net.grad_view(k).cpu()
        scale = max(float(g.abs().max()), 1e-6)
        err = float(((got - g).abs() - bound.get(k, 0.0)).max())
        if err > rtol * scale + 1e-7:
            bad[k] = (err, scale)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0] / kv[1][1])[:5]


def _run(embeddings, in_dims, sizes, seed, flips=False):
    rng = np.random.default_rng(seed)
    net = synthetic.build_network(embeddings, in_dims, TABLE, lstm_dim=64, mixture_components=3, seed=seed, precision=0)
    seqs = ([0, 1, 2, 3], [2, 0], [1])
    subs = [synthetic.random_sub_batch(rng, [TABLE[i] for i in seqs[i % 3]], b, sum(in_dims)) for i, b in enumerate(sizes)]
    _check(net, synthetic.ArrayBatch(subs), list(embeddings), in_dims, 3, flips=flips)


# E = 96: the widest the fused kernels take; widths 30 and 42 are not multiples of four floats, 24 is
WIDE3 = {'o_a': {'dim': 30, 'depth': 3}, 'o_b': {'dim': 24, 'depth': 1}, 'o_c': {'dim': 42, 'depth': 2}}


@pytest.mark.parametrize('sizes', [(1,), (7,), (129,), (1100,), (700, 300, 101)])
def test_three_observables_widths_to_96_vs_oracle(cuda, sizes):
    _run(WIDE3, [3, 5, 2], sizes, 21)


@pytest.mark.parametrize('depth', [1, 3])
def test_observable_depth_vs_oracle(cuda, depth):
    emb = {'o_a': {'dim': 16, 'depth': depth}, 'o_b': {'dim': 20, 'depth': depth}, 'o_c': {'dim': 28, 'depth': depth}}
    _run(emb, [4, 1, 7], (129, 7), 5 + depth)


# E = 160 is too wide to fuse; both chains have two or more layers at least 32 wide, and 'b' starts at column 64
TC2 = {'a': {'dim': 64, 'depth': 2}, 'b': {'dim': 96, 'depth': 3}}
# E = 120 is too wide to fuse, and the depth-1 chain rules out the tensor-core form
SIMT2 = {'a': {'dim': 100, 'depth': 1}, 'b': {'dim': 20, 'depth': 2}}
# E = 64 with a 64-wide hidden layer: the tensor-core form would take it too, the fused kernels must
BOTH1 = {'a': {'dim': 64}}


def _run_form(embeddings, in_dims, sizes, seed, form, flips=False):
    """_run, and the kernels of the step show which form ran: the fused kernels are obsmlp::k_fwd / k_bwd, and the
    tensor-core form's backward always starts with k_pack_rows_masked."""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _run(embeddings, in_dims, sizes, seed, flips)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    fused = [any('obsmlp::k_fwd' in n for n in names), any('obsmlp::k_bwd' in n for n in names)]
    tc = any('k_pack_rows_masked' in n for n in names)
    assert fused == [form == 'fused'] * 2 and tc == (form == 'tensor_core'), (form, sorted(set(names)))


@pytest.mark.parametrize('sizes', [(129,), (512, 300, 101), (700, 300, 101), (700, 300)])
def test_tensor_core_form_vs_oracle(cuda, sizes):
    _run_form(TC2, [40, 3], sizes, 31, 'tensor_core', flips=True)


@pytest.mark.parametrize('sizes', [(129,), (700, 300, 101)])
def test_simt_form_vs_oracle(cuda, sizes):
    _run_form(SIMT2, [3, 5], sizes, 41, 'simt')


def test_fused_form_preferred_over_tensor_core(cuda):
    _run_form(BOTH1, [64], (129,), 51, 'fused')


def test_fused_form_carves_no_tensor_core_images(cuda):
    # BOTH1 and its depth-1 twin (which only the fused form takes) differ by the 64-wide hidden activation and its
    # gradient, fp32 [256, 64] each; tile images of the observe-embedding layers would add several times that
    B = 256
    ws = []
    for emb in (BOTH1, {'a': {'dim': 64, 'depth': 1}}):
        net = synthetic.build_network(emb, [64], TABLE, lstm_dim=64, mixture_components=3, seed=0, precision=0)
        net._sync_native()
        ws.append(_lib.call('ppb_ic_workspace_bytes', net._handle, B, B, 1, 1, 1))
    assert ws[0] - ws[1] == 2 * B * 64 * 4, ws
