"""Fused observe-embedding MLP kernels (obs_mlp.cuh) at shapes the workload tests do not reach: three observables with
input dims above one, chain depths 1 to 3, widths up to 96 (rows that are and are not multiples of four floats), and
batches from one trace to more traces than there are SMs.  Loss and every gradient are checked against the oracle."""
import numpy as np
import pytest
import torch

from oracle import network as onet
from pyprob_b200 import synthetic

pytestmark = pytest.mark.gpu

TABLE = [('a_u', 'Uniform', 0), ('a_c', 'Categorical', 5), ('a_n', 'Normal', 0), ('a_p', 'Poisson', 0)]


def _check(net, batch, observe_names, observe_in_dims, K, rtol=1e-4):
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in batch.subs]
    want_loss, want_grads, _ = onet.loss_and_grads(params, tsubs, observe_names, observe_in_dims, K)
    ok, loss = net._loss(batch)
    assert ok
    assert abs(float(loss.detach()) - float(want_loss)) <= rtol * abs(float(want_loss))
    loss.backward()
    bad = {}
    for k, g in want_grads.items():
        got = net.grad_view(k).cpu()
        scale = max(float(g.abs().max()), 1e-6)
        err = float((got - g).abs().max())
        if err > rtol * scale + 1e-7:
            bad[k] = (err, scale)
    assert not bad, sorted(bad.items(), key=lambda kv: -kv[1][0] / kv[1][1])[:5]


def _run(embeddings, in_dims, sizes, seed):
    rng = np.random.default_rng(seed)
    net = synthetic.build_network(embeddings, in_dims, TABLE, lstm_dim=64, mixture_components=3, seed=seed, precision=0)
    seqs = ([0, 1, 2, 3], [2, 0], [1])
    subs = [synthetic.random_sub_batch(rng, [TABLE[i] for i in seqs[i % 3]], b, sum(in_dims)) for i, b in enumerate(sizes)]
    _check(net, synthetic.ArrayBatch(subs), list(embeddings), in_dims, 3)


# E = 96: the widest the fused kernels take; widths 30 and 42 are not multiples of four floats, 24 is
WIDE3 = {'o_a': {'dim': 30, 'depth': 3}, 'o_b': {'dim': 24, 'depth': 1}, 'o_c': {'dim': 42, 'depth': 2}}


@pytest.mark.parametrize('sizes', [(1,), (7,), (129,), (1100,), (700, 300, 101)])
def test_three_observables_widths_to_96_vs_oracle(cuda, sizes):
    _run(WIDE3, [3, 5, 2], sizes, 21)


@pytest.mark.parametrize('depth', [1, 3])
def test_observable_depth_vs_oracle(cuda, depth):
    emb = {'o_a': {'dim': 16, 'depth': depth}, 'o_b': {'dim': 20, 'depth': depth}, 'o_c': {'dim': 28, 'depth': depth}}
    _run(emb, [4, 1, 7], (129, 7), 5 + depth)
