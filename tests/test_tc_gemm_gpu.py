"""GPU: tensor-core building blocks — operand packing (bit-exact layout + TF32 split) and the packed GEMM
against an fp64 CPU matmul.  3xTF32 must be fp32-faithful (<= 2e-6 relative to the fp64 result scale);
single-pass TF32 is only held to TF32 accuracy."""
import numpy as np
import pytest
import torch

from pyprob_b200 import _lib
from pyprob_b200._lib import call, ptr, stream

pytestmark = pytest.mark.gpu


def _pack(x, mn=False):
    rows, K = x.shape
    nfl = _lib.call('ppb_packed_floats', rows, K)
    hi = torch.empty(nfl, device=x.device)
    lo = torch.empty(nfl, device=x.device)
    call('ppb_pack_tf32_mn' if mn else 'ppb_pack_tf32', ptr(x), rows, K, x.stride(0), ptr(hi), ptr(lo), stream())
    return hi, lo


def _packed_index(rows, K):
    KB = (K + 31) // 32
    r, k = np.meshgrid(np.arange(rows), np.arange(K), indexing='ij')
    rt, rr128, kb, kk = r >> 7, r & 127, k >> 5, k & 31
    atom, rr, c, j = rr128 >> 3, rr128 & 7, kk >> 2, kk & 3
    return (rt * KB + kb) * 4096 + atom * 256 + rr * 32 + ((c ^ rr) << 2) + j


def test_pack_layout_and_split(cuda):
    rows, K = 200, 77
    x = torch.randn(rows, K, device=cuda)
    hi, lo = _pack(x)
    idx = torch.as_tensor(_packed_index(rows, K), device=cuda)
    h, l = hi[idx], lo[idx]
    # hi is x rounded to TF32 (low 13 mantissa bits zero), hi+lo reproduces x to ~2^-21
    assert (h.view(torch.int32) & 0x1FFF).abs().sum().item() == 0
    assert (l.view(torch.int32) & 0x1FFF).abs().sum().item() == 0
    assert ((h + l - x).abs() <= x.abs() * 2.0 ** -20 + 1e-30).all()
    # padding is zero
    mask = torch.ones_like(hi, dtype=torch.bool)
    mask[idx.view(-1)] = False
    assert hi[mask].abs().sum().item() == 0 and lo[mask].abs().sum().item() == 0


@pytest.mark.parametrize('persistent', ['0', '1'])   # PPB_PERSISTENT: one CTA per SM walking the tiles (tc_persist.cuh)
@pytest.mark.parametrize('M,N,K', [(128, 128, 32), (128, 128, 64), (256, 256, 128), (100, 70, 50), (300, 2048, 724),
                                   (1024, 512, 512), (2000, 1500, 96), (4096, 2048, 512), (1300, 1300, 40)])
@pytest.mark.parametrize('precision', [0, 1])
def test_gemm_packed(cuda, monkeypatch, M, N, K, precision, persistent):
    monkeypatch.setenv('PPB_PERSISTENT', persistent)
    gen = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    a = torch.randn(M, K, generator=gen)
    b = torch.randn(N, K, generator=gen)
    bias = torch.randn(N, generator=gen)
    want = (a.double() @ b.double().t() + bias.double()).clamp(min=0).numpy()
    ah, al = _pack(a.to(cuda))
    bh, bl = _pack(b.to(cuda))
    c = torch.full((M, N), float('nan'), device=cuda)
    call('ppb_gemm_packed', ptr(ah), ptr(al), ptr(bh), ptr(bl), ptr(c), M, N, K, N, ptr(bias.to(cuda)), 1, precision,
         stream())
    torch.cuda.synchronize()
    got = c.cpu().double().numpy()
    scale = np.sqrt(K)  # typical |dot product|
    err = np.abs(got - want).max() / scale
    assert np.isfinite(got).all()
    # fp32-faithful: within ~2x of a CPU fp32 sgemm (the tensor core accumulates with truncation; see tc_gemm.cu)
    assert err < (8e-6 if precision == 0 else 3e-3), err


@pytest.mark.parametrize('M,N,R', [(128, 128, 32), (128, 128, 256), (100, 30, 77), (271, 512, 300), (2048, 64, 256),
                                   (512, 2048, 1000)])
@pytest.mark.parametrize('precision', [0, 1])
def test_gemm_packed_tn(cuda, M, N, R, precision):
    """Weight-gradient form: C = X^T Y with both operands read MN-major from the row-major-packed images."""
    gen = torch.Generator().manual_seed(M + N + R)
    x = torch.randn(R, M, generator=gen)
    y = torch.randn(R, N, generator=gen)
    want = (x.double().t() @ y.double()).numpy()
    xh, xl = _pack(x.to(cuda), mn=True)
    yh, yl = _pack(y.to(cuda), mn=True)
    c = torch.full((M, N), float('nan'), device=cuda)
    call('ppb_gemm_packed_tn', ptr(xh), ptr(xl), ptr(yh), ptr(yl), ptr(c), M, N, R, N, precision, stream())
    torch.cuda.synchronize()
    got = c.cpu().double().numpy()
    err = np.abs(got - want).max() / np.sqrt(R)
    assert np.isfinite(got).all()
    assert err < (8e-6 if precision == 0 else 3e-3), err


@pytest.mark.parametrize('M,N,K,cs', [(128, 128, 64, 2), (512, 2048, 512, 2), (512, 512, 2048, 8), (256, 271, 512, 8),
                                      (100, 70, 500, 4), (300, 96, 271, 4), (256, 30, 300, 2), (129, 257, 96, 2),
                                      (256, 271, 30, 8), (128, 64, 40, 4)])   # K shorter than the cluster: empty splits
@pytest.mark.parametrize('precision', [0, 1])
def test_gemm_packed_cluster_split_k(cuda, M, N, K, cs, precision):
    """Cluster split-K (tc_cluster.cuh): the reduction of every output tile is divided over `cs` CTAs of one thread-block
    cluster and the partial tiles meet in distributed shared memory — same result as the single-CTA kernel."""
    gen = torch.Generator().manual_seed(M * 5 + N * 3 + K + cs)
    a = torch.randn(M, K, generator=gen)
    b = torch.randn(N, K, generator=gen)
    bias = torch.randn(N, generator=gen)
    want = (a.double() @ b.double().t() + bias.double()).clamp(min=0).numpy()
    ah, al = _pack(a.to(cuda))
    bh, bl = _pack(b.to(cuda))
    c = torch.full((M, N), float('nan'), device=cuda)
    call('ppb_gemm_packed_cluster', ptr(ah), ptr(al), ptr(bh), ptr(bl), ptr(c), M, N, K, N, ptr(bias.to(cuda)), 1, precision,
         cs, stream())
    torch.cuda.synchronize()
    got = c.cpu().double().numpy()
    assert np.isfinite(got).all()
    err = np.abs(got - want).max() / np.sqrt(K)
    assert err < (8e-6 if precision == 0 else 3e-3), err
