"""The single-GPU Adam step (ppb_adam_step_dev) on every path that runs it: the scalar fallback on unaligned arrays, the
network's device state across a checkpoint, and ppb_ic_train_step_host with and without its cached CUDA graph."""
import numpy as np
import pytest
import torch

from pyprob_b200 import synthetic
from pyprob_b200._lib import call, ptr, stream
from pyprob_b200.util import Optimizer

pytestmark = pytest.mark.gpu


def test_adam_step_dev_on_unaligned_arrays_vs_torch(cuda):
    """Every array offset by one float and n not a multiple of 4: no float4 access, every element takes the scalar loop."""
    gen = torch.Generator().manual_seed(1)
    n = 50001
    p = torch.randn(n + 1, generator=gen).to(cuda)
    ref_p = p[1:].clone().requires_grad_(True)
    opt = torch.optim.Adam([ref_p], lr=1e-3, weight_decay=1e-2)
    g = torch.zeros(n + 1, device=cuda)
    m, v = torch.zeros(n + 1, device=cuda), torch.zeros(n + 1, device=cuda)
    hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 1e-2, 1.0], device=cuda)
    state = torch.zeros(2, dtype=torch.int64, device=cuda)
    for _ in range(3):
        g[1:] = torch.randn(n, generator=gen).to(cuda)
        ref_p.grad = g[1:].clone()
        opt.step()
        call('ppb_adam_step_dev', ptr(p[1:]), ptr(g[1:]), ptr(m[1:]), ptr(v[1:]), n, ptr(hyper), ptr(state), stream())
    torch.testing.assert_close(p[1:], ref_p.data, rtol=1e-5, atol=1e-6)
    assert int(state[0]) == 3


def _train(net, grads, lrs):
    for g, lr in zip(grads, lrs):
        net._arena.grad = g.clone()
        net._learning_rate = lr
        net.optimizer_step()
    assert net._seg is None   # every step ran the flat kernel


def test_flat_adam_resumes_bit_identically_from_a_checkpoint(cuda, tmp_path):
    """k flat steps, save, load, then k more steps on the original and on the loaded copy: the loaded copy starts a new
    device state block whose counter comes from the checkpoint's step count, so both continue with the same bias
    corrections.  The learning rate changes every step, as under a polynomial schedule; fixed gradients keep the
    comparison free of the loss's atomic reductions."""
    k = 3
    net = synthetic.gum_network(lstm_dim=64, precision=0, seed=2)
    net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM, 1e-3, 1e-5
    net._auto_skip_absent = False
    net._create_optimizer()
    gen = torch.Generator().manual_seed(4)
    grads = [torch.randn(net._arena.numel(), generator=gen).to(cuda) for _ in range(2 * k)]
    lrs = [1e-3 * (1.0 - 0.1 * i) for i in range(2 * k)]
    _train(net, grads[:k], lrs[:k])
    path = str(tmp_path / 'resume.network')
    net._save(path)
    loaded = type(net)._load(path)
    assert loaded._optimizer_step == k
    _train(net, grads[k:], lrs[k:])
    _train(loaded, grads[k:], lrs[k:])
    assert net._optimizer_step == loaded._optimizer_step == 2 * k
    assert torch.equal(net._arena.data, loaded._arena.data)
    assert torch.equal(net._exp_avg, loaded._exp_avg)
    assert torch.equal(net._exp_avg_sq, loaded._exp_avg_sq)


def _host_steps(net, batches, cuda):
    net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM, 1e-3, 0.0
    net._create_optimizer()
    net._sync_native()
    encs = [b.encode(net) for b in batches]
    hosts = [torch.from_numpy(e.pack().copy()) for e in encs]
    img_dev = torch.empty(max(h.numel() for h in hosts), dtype=hosts[0].dtype, device=cuda)
    need = net._ensure_workspace(encs[0])
    grad = torch.zeros_like(net._arena.data)
    loss_host = torch.zeros(1).pin_memory()
    status_host = torch.zeros(1, dtype=torch.int32).pin_memory()
    losses = []
    for step in range(1, 7):
        h = hosts[(step - 1) % len(hosts)]
        call('ppb_ic_train_step_host', net._handle, ptr(net._arena.data), ptr(grad), ptr(net._exp_avg), ptr(net._exp_avg_sq),
             net._arena.numel(), h.data_ptr(), h.numel(), ptr(img_dev), ptr(net._workspace), net._workspace.numel(), 0,
             1e-3 * (1.0 - 0.1 * step), 0.9, 0.999, 1e-8, 0.0, step, loss_host.data_ptr(), status_host.data_ptr(),
             stream())
        assert int(status_host[0]) == 0
        losses.append(float(loss_host[0]))
    return losses


def test_host_step_eager_matches_graph_replay(cuda, monkeypatch):
    """ppb_ic_train_step_host on a net created under PPB_HOST_STEP_GRAPH=0 (every call issued without capture) against
    the default (first call eager, second captured, later ones replayed), over six steps with a changing learning rate:
    both modes run the same Adam.  The loss and its gradient use atomic reductions, so two runs of the same mode already
    differ in the last bits (a few 1e-8 on the arena); the tolerance is that of test_host_step_gpu."""
    rng = np.random.default_rng(6)
    batches = [synthetic.gum_batch(rng, 1) for _ in range(3)]
    monkeypatch.setenv('PPB_HOST_STEP_GRAPH', '0')
    eager = synthetic.gum_network(lstm_dim=64, precision=0, seed=8)
    eager._sync_native()   # ppb_net_create reads the variable
    monkeypatch.delenv('PPB_HOST_STEP_GRAPH')
    graph = synthetic.gum_network(lstm_dim=64, precision=0, seed=8)
    assert torch.equal(eager._arena.data, graph._arena.data)
    eager_losses = _host_steps(eager, batches, cuda)
    graph_losses = _host_steps(graph, batches, cuda)
    np.testing.assert_allclose(eager_losses, graph_losses, rtol=1e-6)
    for a, b in ((eager._arena.data, graph._arena.data), (eager._exp_avg, graph._exp_avg),
                 (eager._exp_avg_sq, graph._exp_avg_sq)):
        torch.testing.assert_close(a, b, rtol=1e-6, atol=1e-7)
