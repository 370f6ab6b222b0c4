import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pyprob_b200 import _lib
from pyprob_b200._lib import call, ptr, stream
dev = torch.device('cuda:0')
def pack(x, mn=False):
    rows, K = x.shape
    nfl = _lib.call('ppb_packed_floats', rows, K)
    hi = torch.empty(nfl, device=dev); lo = torch.empty(nfl, device=dev)
    call('ppb_pack_tf32_mn' if mn else 'ppb_pack_tf32', ptr(x), rows, K, x.stride(0), ptr(hi), ptr(lo), stream())
    return hi, lo
def timeit(fn, n=200):
    for _ in range(10): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000 / n
for (M, N, K) in [(128, 128, 32), (128, 128, 512), (256, 2048, 64), (256, 2048, 512), (256, 271, 512), (4096, 2048, 512)]:
    a = torch.randn(M, K, device=dev); b = torch.randn(N, K, device=dev); c = torch.empty(M, N, device=dev)
    ah, al = pack(a); bh, bl = pack(b)
    for prec in (0, 1):
        t = timeit(lambda: call('ppb_gemm_packed', ptr(ah), ptr(al), ptr(bh), ptr(bl), ptr(c), M, N, K, N, None, 0, prec, stream()))
        fl = 2.0 * M * N * K * (3 if prec == 0 else 1)
        print('NT M%5d N%5d K%5d prec%d: %8.1f us  %7.2f TF/s (issued)' % (M, N, K, prec, t, fl / t / 1e6))
for (M, N, R) in [(2048, 64, 256), (271, 512, 256), (2048, 512, 4096)]:
    x = torch.randn(R, M, device=dev); y = torch.randn(R, N, device=dev); c = torch.empty(M, N, device=dev)
    xh, xl = pack(x, True); yh, yl = pack(y, True)
    t = timeit(lambda: call('ppb_gemm_packed_tn', ptr(xh), ptr(xl), ptr(yh), ptr(yl), ptr(c), M, N, R, N, 0, stream()))
    print('TN M%5d N%5d R%5d prec0: %8.1f us' % (M, N, R, t))
t = timeit(lambda: torch.empty(1, device=dev).zero_())
print('torch tiny kernel launch: %.1f us' % t)

# device-side durations (CUPTI) of the bring-up kernel for tiny problems: the fixed cost of one tensor-core tile
from torch.profiler import profile, ProfilerActivity
for (M, N, K) in [(128, 128, 32), (128, 128, 128), (128, 128, 512), (256, 2048, 64)]:
    a = torch.randn(M, K, device=dev); b = torch.randn(N, K, device=dev); c = torch.empty(M, N, device=dev)
    ah, al = pack(a); bh, bl = pack(b)
    for _ in range(3):
        call('ppb_gemm_packed', ptr(ah), ptr(al), ptr(bh), ptr(bl), ptr(c), M, N, K, N, None, 0, 0, stream())
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(20):
            call('ppb_gemm_packed', ptr(ah), ptr(al), ptr(bh), ptr(bl), ptr(c), M, N, K, N, None, 0, 0, stream())
        torch.cuda.synchronize()
    for e in prof.key_averages():
        if 'gemm_packed' in e.key:
            print('device time M%d N%d K%d x3: %.2f us' % (M, N, K, e.device_time_total / e.count))
