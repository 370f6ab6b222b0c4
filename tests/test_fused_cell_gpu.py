"""LSTM steps with the cell fused into the recurrent GEMM (the default: cluster split-K with the cell in the reduce phase,
csrc/tc_cluster.cuh, or the per-step kernel without clusters, csrc/tc_lstm.cuh, when a step has few 32-element chunks or
many tiles): same order of additions and same activations as the unfused pair (PPB_FUSED_CELL=0: tcg::k_grouped +
k_cell_fwd), so loss and every gradient must agree to rounding (the cluster kernel sums its K-slices in a different order;
FMA contraction may differ); and the fused step must agree with the oracle."""
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


@pytest.mark.parametrize('level', ['3'])   # any value but 0 selects the default fused step
@pytest.mark.parametrize('precision', [0, 1])
@pytest.mark.parametrize('seed,lstm_dim,spec', [
    (2, 32, [([0, 1, 2, 3, 4, 5], 7), ([2], 1), ([0, 3], 64), ([1, 5, 4, 0], 3)]),
    (3, 64, [([2, 4], 130), ([5, 1, 5, 1, 5, 1, 0], 33), ([3], 257)]),
    (4, 128, [([0, 1, 2, 3, 4, 5, 0, 1, 2, 3], 300)]),
    (5, 256, [([2, 0, 4, 1], 140), ([3, 5], 20)]),
    (6, 256, [([2, 0, 4], 1100)]),   # 9 row tiles x 8 unit blocks = 72 tiles per step: k_lstm_step at deep K
])
def test_fused_cell_matches_the_unfused_step(cuda, monkeypatch, seed, lstm_dim, spec, precision, level):
    monkeypatch.setenv('PPB_FUSED_CELL', '0')      # read when the native network handle is created
    base, subs = _case(seed, lstm_dim, spec, precision)
    ok, loss0 = base._loss(synthetic.ArrayBatch(subs))
    assert ok
    loss0.backward()
    g0 = base._arena.grad.clone()
    monkeypatch.setenv('PPB_FUSED_CELL', level)
    fused, _ = _case(seed, lstm_dim, spec, precision)
    ok, loss1 = fused._loss(synthetic.ArrayBatch(subs))
    assert ok
    loss1.backward()
    assert torch.equal(fused._arena.data, base._arena.data)
    # identical up to the compiler's choice of FMA contraction in the cell arithmetic of the two kernels
    assert abs(float(loss1.detach()) - float(loss0.detach())) <= 2e-6 * abs(float(loss0.detach()))
    scale = float(g0.abs().max())
    assert float((fused._arena.grad - g0).abs().max()) <= 2e-5 * scale
    if precision == 0:
        params = {k: v.cpu() for k, v in fused.reference_state_dict().items()}
        tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
        want_loss, _, _ = onet.loss_and_grads(params, tsubs, ['o0', 'o1'], [3, 1], 4)
        assert abs(float(loss1.detach()) - float(want_loss)) <= 1e-4 * abs(float(want_loss))
