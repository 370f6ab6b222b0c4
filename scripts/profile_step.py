"""Per-kernel device times of the bench training step in a normal (non-ncu) run, via CUPTI (torch.profiler)."""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pyprob_b200 import _lib, synthetic
from pyprob_b200._lib import call, ptr
from pyprob_b200.util import Optimizer
from pyprob_b200.network import BatchStruct

prec = int(sys.argv[1]) if len(sys.argv) > 1 else 0
cfg = sys.argv[2] if len(sys.argv) > 2 else 'gum'
B = int(sys.argv[3]) if len(sys.argv) > 3 else 256
dev = torch.device('cuda:0')
rng = np.random.default_rng(0)
if cfg == 'gum':
    net = synthetic.gum_network(lstm_dim=512, precision=prec); batch = synthetic.gum_batch(rng, B)
else:
    T = int(cfg[1:]) if cfg.startswith('s') and len(cfg) > 1 else 50
    net = synthetic.synthetic50_network(precision=prec, T=T); batch = synthetic.synthetic50_batch(rng, B, T=T)
net._optimizer_type, net._learning_rate_init, net._weight_decay = Optimizer.ADAM, 1e-3, 0.0
net._create_optimizer(); net._sync_native()
enc = batch.encode(net)
grad = torch.zeros_like(net._arena.data); net._arena.grad = grad
img = torch.from_numpy(enc.pack().copy()).pin_memory(); dimg = img.to(dev)
bs = BatchStruct(); call('ppb_batch_from_image', img.data_ptr(), dimg.data_ptr(), img.numel(), C.byref(bs))
need = net._ensure_workspace(enc)
st = torch.cuda.current_stream().cuda_stream
loss = torch.empty((), device=dev); status = torch.zeros(1, dtype=torch.int32, device=dev)
hyper = torch.tensor([1e-3, 0.9, 0.999, 1e-8, 0.0, 1.0], dtype=torch.float32, device=dev)
adam_state = torch.zeros(2, dtype=torch.int64, device=dev)
def step():
    st = torch.cuda.current_stream().cuda_stream
    grad.zero_()
    call('ppb_ic_loss_forward', net._handle, ptr(net._arena.data), C.byref(bs), ptr(net._workspace), need, prec, ptr(loss), ptr(status), None, 1, st)
    call('ppb_ic_loss_backward', net._handle, ptr(net._arena.data), ptr(grad), C.byref(bs), ptr(net._workspace), need, prec, 1.0, st)
    call('ppb_adam_step_dev', ptr(net._arena.data), ptr(grad), ptr(net._exp_avg), ptr(net._exp_avg_sq), net._arena.numel(), ptr(hyper), ptr(adam_state), st)
for _ in range(5): step()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(50): step()
e1.record(); torch.cuda.synchronize()
print('avg step (no L2 flush, back-to-back): %.1f us  | rows %d params %d' % (e0.elapsed_time(e1) * 1000 / 50, enc.n_rows, net._arena.numel()))
if len(sys.argv) > 4 and sys.argv[4] == 'quick':   # A/B mode: eager and graph-replay step time only
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        step()
    for _ in range(5): g.replay()
    torch.cuda.synchronize()
    best = 1e9
    for _ in range(5):
        e0.record()
        for _ in range(20): g.replay()
        e1.record(); torch.cuda.synchronize()
        best = min(best, e0.elapsed_time(e1) * 1000 / 20)
    print('graph replay: %.1f us per step (best of 5 x 20)' % best)
    sys.exit(0)
from torch.profiler import profile, ProfilerActivity
with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU]) as prof:
    for _ in range(5): step()
    torch.cuda.synchronize()
rows = [(e.key[:70], e.count, e.device_time_total / max(e.count, 1), e.device_time_total) for e in prof.key_averages() if e.device_time_total > 0]
tot = sum(r[3] for r in rows)
for k, c, avg, t in sorted(rows, key=lambda r: -r[3])[:25]:
    print('%-72s n=%4d avg=%8.1f us total=%9.1f us %5.1f%%' % (k, c, avg, t, 100 * t / tot))
print('device total per step: %.1f us' % (tot / 5))

# per-launch phase stamps of the tensor-core GEMM kernels (CTA 0 of each launch of one step)
NTR = 256
tr = torch.zeros(NTR * 16, dtype=torch.int64, device=dev)
call('ppb_debug_trace', ptr(tr))
step()
torch.cuda.synchronize()
call('ppb_debug_trace', None)
def dump(t, title):
    print(title)
    prev_end = None
    for i in range(NTR):
        if t[i, 0] == 0: break
        r = t[i]
        kind = int(r[13]); name = 'grouped' if kind == 0 else ('cluster' if kind % 16 == 1 else 'lstm_cl') + 'x%d' % (kind // 16)
        vis = (r[7] - r[0]) if r[7] else -1
        print('tc launch %3d %-10s: M%5d N%5d K%5d grid%4d chunks%3d | setup %5d first_data %5d mma_issued %5d acc_ready %5d cluster_vis %5d loads_done %5d epi_done %5d end %5d ns | start %+7d ns after previous end' % (
            i, name, r[8], r[9], r[10], r[11], r[12], r[1]-r[0], r[2]-r[0], r[3]-r[0], r[4]-r[0], vis, (r[14]-r[0]) if r[14] else -1, r[5]-r[0], r[6]-r[0],
            (r[0] - prev_end) if prev_end is not None else 0))
        prev_end = r[6]
dump(tr.cpu().numpy().reshape(NTR, 16), '== eager launches')

# the same step as one CUDA graph (the production form): the stamps of a replay show the gaps between dependent graph nodes
tr.zero_()
call('ppb_debug_trace', ptr(tr))
g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):
    step()
call('ppb_debug_trace', None)
for _ in range(3): g.replay()
torch.cuda.synchronize()
e0.record()
for _ in range(20): g.replay()
e1.record(); torch.cuda.synchronize()
print('graph replay: %.1f us per step' % (e0.elapsed_time(e1) * 1000 / 20))
dump(tr.cpu().numpy().reshape(NTR, 16), '== graph replay (stamps of the last replay)')
