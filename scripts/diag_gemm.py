"""Bring-up diagnostic: 3xTF32 / TF32 error of the wgmma packed GEMM vs fp64, as a function of shape."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
from pyprob_b200 import _lib
from pyprob_b200._lib import call, ptr, stream

def pack(x):
    rows, K = x.shape
    nfl = _lib.call('ppb_packed_floats', rows, K)
    hi = torch.empty(nfl, device=x.device); lo = torch.empty(nfl, device=x.device)
    call('ppb_pack_tf32', ptr(x), rows, K, x.stride(0), ptr(hi), ptr(lo), stream())
    return hi, lo

dev = torch.device('cuda:0')
for (M, N, K) in [(128,128,32),(128,128,64),(128,128,96),(128,128,128),(128,128,160),(128,128,256),(128,128,1024),(256,128,64),(128,256,64),(256,256,64),(256,256,96)]:
    g = torch.Generator().manual_seed(1)
    a = torch.randn(M, K, generator=g); b = torch.randn(N, K, generator=g)
    want = a.double() @ b.double().t()
    f32 = (a @ b.t()).double()
    ah, al = pack(a.to(dev)); bh, bl = pack(b.to(dev))
    res = {}
    for prec in (0, 1):
        c = torch.zeros(M, N, device=dev)
        call('ppb_gemm_packed', ptr(ah), ptr(al), ptr(bh), ptr(bl), ptr(c), M, N, K, N, None, 0, prec, stream())
        torch.cuda.synchronize()
        e = (c.cpu().double() - want)
        res[prec] = (e.abs().max().item(), e.mean().item())
    e32 = (f32 - want).abs().max().item()
    print('M%5d N%5d K%5d | x3 max %.3e mean %+.3e | tf32 max %.3e | cpu-fp32 max %.3e | |want|max %.1f' % (M, N, K, res[0][0], res[0][1], res[1][0], e32, want.abs().max().item()))
