"""Output layer of the proposal heads + NLL (csrc/net_tc.inc: run_head_nll) against the oracle on ragged sub-batches, segments
with padding rows behind them, and H = 64 / 128 / 256.  At these sizes the h2 phase runs as a cluster, so the NLL runs in its
reduce phase (net.cu: NllRowEpi).  Loss within 1e-4; at precision 0 every gradient within 1e-4 of its tensor's maximum."""
import numpy as np
import pytest
import torch

from oracle import network as onet
from pyprob_b200 import synthetic

pytestmark = pytest.mark.gpu

TABLE = [('a_u', 'Uniform', 0), ('a_c', 'Categorical', 5), ('a_n', 'Normal', 0), ('a_p', 'Poisson', 0),
         ('a_n2', 'Normal', 0), ('a_c2', 'Categorical', 3)]


def _case(seed, lstm_dim, spec, precision):
    rng = np.random.default_rng(seed)
    net = synthetic.build_network({'o0': {'dim': 12, 'depth': 2}, 'o1': {'dim': 6, 'depth': 3}}, [3, 1], TABLE,
                                  lstm_dim=lstm_dim, mixture_components=4, seed=seed, precision=precision)
    subs = [synthetic.random_sub_batch(rng, [TABLE[i] for i in seq], B, 4) for seq, B in spec]
    return net, subs


@pytest.mark.parametrize('precision', [0, 1])
@pytest.mark.parametrize('seed,lstm_dim,spec', [
    (21, 64, [([0, 1, 2, 3, 4, 5], 40), ([2], 3), ([0, 3], 64)]),
    (22, 128, [([5, 1, 4], 300), ([3], 129)]),          # segments with padding rows behind them
    (23, 256, [([2, 0, 4, 1], 140), ([3, 5], 20)]),
])
def test_head_output_and_nll_vs_oracle(cuda, seed, lstm_dim, spec, precision):
    net, subs = _case(seed, lstm_dim, spec, precision)
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
    want_loss, want_grads, _ = onet.loss_and_grads(params, tsubs, ['o0', 'o1'], [3, 1], 4)
    ok, loss = net._loss(synthetic.ArrayBatch(subs))
    assert ok
    err = abs(float(loss.detach()) - float(want_loss))
    assert err <= 1e-4 * abs(float(want_loss)), (err, float(want_loss))
    if precision == 0:
        loss.backward()
        for k, g in want_grads.items():
            got = net.grad_view(k).cpu()
            scale = max(float(g.abs().max()), 1e-6)
            err = float((got - g).abs().max())
            assert err <= 1e-4 * scale + 1e-7, (k, err, scale)
