"""GPU: the step-input kernels of the LSTM training step when the one-pass dgates reduction does not apply.

k_dgates_reduce needs sample_embedding_dim <= 4 and 4 * lstm_dim <= 2048.  Beyond either limit the backward runs
k_step_colsum + k_smp_bwd_seg + k_wsmp_grad instead, at every precision.  Loss and every parameter gradient are checked
against the oracle on ragged sub-batches with T > 1, where Categorical and scalar addresses are both previous sites."""
import numpy as np
import pytest
import torch

from oracle import network as onet
from pyprob_b200 import synthetic

pytestmark = pytest.mark.gpu

TABLE = [('s_n', 'Normal', 0), ('s_c', 'Categorical', 5), ('s_u', 'Uniform', 0), ('s_p', 'Poisson', 0)]
OBS, IN_DIMS, K = ['o0', 'o1'], [3, 1], 4
# sub-batches: (address sequence, traces)
SPEC = [([0, 1, 2, 1], 37), ([1, 0], 130), ([3, 2, 0, 1, 3], 5)]
# The kernels under test are fp32 CUDA-core code, the same at every precision, and precisions 0 and 2 hold them to 1e-4.
# Precision 1 rounds every GEMM operand to tf32 (10-bit mantissa): sums over the batch that cancel to a few percent of their
# terms show that rounding (tests/test_t1_chain_gpu.py), so at 0.25 of a tensor's largest entry its case only checks that the
# tf32 pipeline feeds these kernels the right buffers; it would miss a dropped term smaller than that.
TOL = {0: (1e-4, 1e-4), 1: (2e-3, 0.25), 2: (1e-4, 1e-4)}
ATOL = {0: 1e-7, 1: 1e-6, 2: 1e-7}


@pytest.mark.parametrize('lstm_dim,sample_dim', [(64, 8), (544, 4)], ids=['S8', 'H544'])
@pytest.mark.parametrize('precision', [0, 1, 2])
def test_loss_and_grads_without_one_pass_reduction(cuda, lstm_dim, sample_dim, precision):
    assert sample_dim > 4 or 4 * lstm_dim > 2048
    rng = np.random.default_rng(lstm_dim + sample_dim)
    net = synthetic.build_network({'o0': {'dim': 12, 'depth': 2}, 'o1': {'dim': 6, 'depth': 1}}, IN_DIMS, TABLE,
                                  lstm_dim=lstm_dim, mixture_components=K, seed=5, precision=precision,
                                  sample_embedding_dim=sample_dim)
    subs = [synthetic.random_sub_batch(rng, [TABLE[i] for i in seq], B, 4) for seq, B in SPEC]
    params = {k: v.cpu() for k, v in net.reference_state_dict().items()}
    tsubs = [{k: (torch.from_numpy(v) if isinstance(v, np.ndarray) else v) for k, v in sb.items()} for sb in subs]
    want_loss, want_grads, _ = onet.loss_and_grads(params, tsubs, OBS, IN_DIMS, K)
    assert params['_layers_sample_embedding.s_c._layers.0.bias'].numel() == sample_dim
    success, loss = net._loss(synthetic.ArrayBatch(subs))
    assert success
    ltol, gtol = TOL[precision]
    assert abs(float(loss.detach()) - float(want_loss)) <= ltol * abs(float(want_loss))
    loss.backward()
    for k, g in want_grads.items():
        got = net.grad_view(k).cpu()
        scale = max(float(g.abs().max()), 1e-6)
        err = float((got - g).abs().max())
        assert err <= gtol * scale + ATOL[precision], (k, err, scale)
