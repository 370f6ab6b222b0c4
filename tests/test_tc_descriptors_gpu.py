"""GPU: the tensor-core GEMM kernels descriptor by descriptor against the float64 restatement of tests/tc_fp64.py, through
ppb_tc_run_problems (the network's phase runners): tcg::k_grouped, its chunk-table instantiation, the persistent
tcp::k_grouped_persistent (more tiles than SMs) and the cluster split-K tcc::k_cluster (CS = 2, 4, 8), with epilogues
0 (fp32 store), 1 (fp32 red.add) and 2 (tile images), at both precisions.

Every launch asserts, from the kernel names torch.profiler records, the form and precision it ran, and every launch is
checked four ways:
  * each fp32 output element within the per-element bound tau (sum_k |A_eff B_eff| + |bias| + |C prefill|) of tc_fp64
    (derived there from the kernels' arithmetic, not fitted), exactly 0 where the epilogue zeroes it (rows at or beyond
    m_valid under kZeroInvalid, mask not > 0), never NaN;
  * each output image bit for bit the rna split of the kernel's own fp32 value where C is written, else within the bound
    plus the split error;
  * the image padding columns (N up to the next 32) exactly +0 in both parts;
  * every float outside the descriptors' write sets keeps its sentinel bits.
Operand images are NaN everywhere outside the blocks the descriptors read as data: the M and N padding of every tile, the
unused image rows and columns around the offsets.  The K padding of the last chunk is zero in both operands, which is the
caller's contract.  Single-pass TF32 launches pass null operand lo pointers.  Before any launch the float ranges every
descriptor reads and writes (tc_fp64.touched_ranges) are checked to lie inside the buffers the test allocated.

Largest error / bound seen on one NVIDIA H100 80GB HBM3 (printed per launch with `-s`; tf32x3 / tf32):
  grouped     epilogue 0: 0.025 / 0.042   epilogue 1: 0.033 / 0.052   epilogue 2: 0.031 / 0.044
  chunk table epilogue 0: 0.014 / 0.023
  persistent  epilogue 0: 0.025 / 0.035   epilogue 1: 0.033 / 0.052   epilogue 2: 0.031 / 0.044
  cluster 2   epilogue 0: 0.018 / 0.029   epilogue 2: 0.021 / 0.026
  cluster 4   epilogue 0: 0.019 / 0.032   epilogue 2: 0.020 / 0.028
  cluster 8   epilogue 0: 0.022 / 0.032   epilogue 2: 0.021 / 0.026
"""
import contextlib
import re

import numpy as np
import pytest
import torch

from pyprob_b200 import _lib
from tests import tc_fp64 as T

pytestmark = pytest.mark.gpu

F32 = np.float32
RATIOS = {}
MASK_VALUES = np.array([1.0, -1.0, 0.0, -0.0, np.nan, 1e-40, -1e-40, 2.5], dtype=F32)   # 1e-40: denormal


# ---- operand and output builders ------------------------------------------------------------------------------------------
def kop(rng, img, rows, K, row0, col0):
    """K-major operand: random [rows, K] block at (row0, col0), zero K padding up to the chunk"""
    x = rng.standard_normal((rows, 32 * ((K + 31) // 32))).astype(F32)
    x[:, K:] = 0
    img.put(x, row0, col0)
    return T.Op(img, row0, col0)


def mnop(rng, img, rows, K, row0, col0, origins=None):
    """MN-major operand: random [K, rows] block (image rows = reduction index) at (row0, col0), or chunk c at image rows
    origins[c] ..; zero K padding"""
    KC = (K + 31) // 32
    x = rng.standard_normal((32 * KC, rows)).astype(F32)
    x[K:, :] = 0
    if origins is None:
        img.put(x, row0, col0)
        return T.Op(img, row0, col0)
    for c, r0 in enumerate(origins):
        img.put(x[32 * c:32 * c + 32], r0, col0)
    return T.Op(img, row0, col0, np.asarray(origins, dtype=np.int32))


def table_origins(rng, KC, spare=2):
    """row origins (multiples of 32) of KC chunks in an image of 32 (KC + spare) rows, not monotone when KC > 1"""
    perm = rng.permutation(KC + spare)[:KC]
    if KC > 1 and (np.diff(perm) > 0).all():
        perm = perm[::-1]
    return [32 * int(p) for p in perm], 32 * (KC + spare)


def cbuf(M, ldc):
    return np.full(M * ldc + 2 * ldc + 64, T.SENTINEL, dtype=np.uint32).view(F32)


def out_img(rows, kb, mn):
    return T.Image(rows, kb, mn, fill=T.SENTINEL)


def mask_img(rng, rows, kb):
    im = T.Image(rows, kb, False)
    im.hi[:] = rng.choice(MASK_VALUES, im.hi.size)
    return im


# ---- one launch ---------------------------------------------------------------------------------------------------------------
FORM_RE = [('persistent', re.compile(r'tcp::k_grouped_persistent<(\w+), (\d)>')),
           ('grouped', re.compile(r'tcg::k_grouped<(\w+), (\d), (\w+)>')),
           ('cluster', re.compile(r'tcc::k_cluster<(\w+), (\d+), (\d)'))]


def _forms(names):
    out = set()
    for n in names:
        for form, rx in FORM_RE:
            m = rx.search(n)
            if not m:
                continue
            x3 = m.group(1) == 'true'
            if form == 'grouped':
                out.add(('ktab' if m.group(3) == 'true' else 'grouped', x3, int(m.group(2))))
            elif form == 'cluster':
                out.add(('cluster{}'.format(m.group(2)), x3, int(m.group(3))))
            else:
                out.add((form, x3, int(m.group(2))))
    return out


@contextlib.contextmanager
def kernel_forms(*expected):
    """one profiler session around a test's launches: the tensor-core kernels it ran must be exactly `expected`
    ((form, 3xTF32, epilogue) each)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        yield
        torch.cuda.synchronize()
    names = [e.key for e in prof.key_averages() if e.device_time_total > 0]
    assert _forms(names) == set(expected), names


def launch(descs, epi, x3, cs=1, ktab=False, prefill=None):
    """Runs descs as one ppb_tc_run_problems launch and returns {(id(buffer), part): host copy after the launch}.
    prefill: {id(desc): [M, N] array} written into C (epilogue 1) before the launch."""
    for d in descs:
        for obj, part, lo, hi in T.touched_ranges(d, x3, epi):
            assert 0 <= lo < hi <= T.size_of(obj, part), ('descriptor reaches outside its buffer', lo, hi)
    for d in descs:
        if prefill and id(d) in prefill:
            d.c[T.c_offsets(d)] = prefill[id(d)].astype(F32)
    dev = {}

    def ptr(obj, part):
        key = (id(obj), part)
        if key not in dev:
            arr = obj.hi if part == 'hi' else obj.lo if part == 'lo' else obj
            dev[key] = torch.from_numpy(np.ascontiguousarray(arr)).cuda()
        return dev[key].data_ptr()
    probs = (T.Problem * len(descs))(*[T.to_problem(d, ptr, x3) for d in descs])
    _lib.call('ppb_tc_run_problems', probs, len(descs), epi, cs, int(ktab), 0 if x3 else 1, _lib.stream())
    torch.cuda.synchronize()
    return {k: t.cpu().numpy() for k, t in dev.items()}


def check(descs, out, epi, x3, form, cs=1, prefill=None):
    """the four checks of the module docstring; returns the largest error / bound"""
    worst = 0.0
    for d in descs:
        val, bound, zero = T.reference(d, x3, cs, (prefill or {}).get(id(d)))
        got_c = None
        if d.c is not None:
            got_c = out[(id(d.c), None)][T.c_offsets(d)]
            g = got_c.astype(np.float64)
            assert np.isfinite(g).all()
            err = np.abs(g - val)
            assert (err <= bound).all(), (d.M, d.N, d.K, float((err / np.maximum(bound, 1e-300)).max()))
            assert (g[zero] == 0).all()
            worst = max(worst, float((err / np.maximum(bound, 1e-300)).max()))
        if epi != 2:
            continue
        for im, mn in ((d.o_k, False), (d.o_mn, True)):
            if im is None:
                continue
            off = T.out_offsets(d, mn)
            hi, lo = out[(id(im), 'hi')][off], out[(id(im), 'lo')][off]
            assert not hi[:, d.N:].view(np.uint32).any() and not lo[:, d.N:].view(np.uint32).any(), 'padding columns'
            hi, lo = hi[:, :d.N], lo[:, :d.N]
            if got_c is not None:
                eh, el = T.split_tf32(got_c)
                np.testing.assert_array_equal(hi.view(np.uint32), eh.view(np.uint32))
                np.testing.assert_array_equal(lo.view(np.uint32), el.view(np.uint32))
            else:
                assert not (hi.view(np.uint32) & 0x1FFF).any() and not (lo.view(np.uint32) & 0x1FFF).any()
                v = hi.astype(np.float64) + lo
                assert np.isfinite(v).all()
                err = np.abs(v - val)
                allow = bound + 2.0 ** -21 * (np.abs(val) + bound)
                assert (err <= allow).all(), (d.M, d.N, d.K, float((err / np.maximum(allow, 1e-300)).max()))
                assert (v[zero] == 0).all()
                worst = max(worst, float((err / np.maximum(allow, 1e-300)).max()))
    for key, (_, _, offs) in T.write_sets(descs, epi).items():
        arr = out[key].view(np.uint32)
        rest = np.ones(arr.size, dtype=bool)
        rest[offs] = False
        assert (arr[rest] == T.SENTINEL).all(), 'a float outside the write set changed'
    k = (form, epi, 'tf32x3' if x3 else 'tf32')
    RATIOS[k] = max(RATIOS.get(k, 0.0), worst)
    print('\nerror/bound {} epilogue {} {}: {:.3g}'.format(*k, worst))
    return worst


def run_and_check(descs, epi, x3, form, cs=1, ktab=False, prefill=None):
    out = launch(descs, epi, x3, cs, ktab, prefill)
    check(descs, out, epi, x3, form, cs, prefill)
    return out


def same_bits(a, b):
    assert a.keys() == b.keys()
    for k in a:
        np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32))


# ---- the descriptor sets ------------------------------------------------------------------------------------------------------
def set_epi0(rng):
    """M in {1, 127, 128, 129, 300}, N in {1, 31, 33, 200}, K in {1, 31, 33, 200, 1000}; A K-major at nonzero (row0, col0) of
    one shared image, B MN-major at nonzero offsets of another; bias, ReLU, kZeroInvalid with m_valid 0 / inside a tile /
    >= M, ldc > N"""
    shapes = [(1, 1, 1, {}), (127, 31, 33, dict(bias=True, flags=T.RELU)), (128, 33, 200, dict(flags=T.ZERO_INVALID, m_valid=0)),
              (129, 200, 31, dict(flags=T.ZERO_INVALID, m_valid=70, ldc=217)),
              (300, 1, 1000, dict(flags=T.ZERO_INVALID, m_valid=400, bias=True)), (300, 200, 200, dict(flags=T.RELU, ldc=203))]
    A = T.Image(128 + sum((M + 127) // 128 * 128 for M, *_ in shapes), 36, False)
    B = T.Image(32 + sum(32 * ((K + 31) // 32) + 32 for *_, K, _ in shapes), 9, True)
    descs, ra, rb = [], 128, 32
    for i, (M, N, K, kw) in enumerate(shapes):
        a = kop(rng, A, M, K, ra, 32 * (1 + i % 3))
        b = mnop(rng, B, N, K, rb, 32 * (1 + i % 2))
        ra += (M + 127) // 128 * 128
        rb += 32 * ((K + 31) // 32) + 32
        ldc = kw.get('ldc', N)
        bias = rng.standard_normal(N).astype(F32) if kw.get('bias') else None
        descs.append(T.Desc(a, b, M, N, K, c=cbuf(M, ldc), ldc=ldc, bias=bias, flags=kw.get('flags', 0),
                            m_valid=kw.get('m_valid', 0)))
    return descs


def set_epi1(rng):
    """both operands MN-major through non-monotone row tables; k_splits 1, 2, 3, 7 and 5 > KC (empty splits); C prefilled"""
    shapes = [(100, 70, 200, 1), (129, 33, 96, 2), (64, 200, 320, 3), (31, 31, 500, 7), (200, 129, 64, 5)]
    descs, pre = [], {}
    for M, N, K, ks in shapes:
        KC = (K + 31) // 32
        oa, ra = table_origins(rng, KC)
        ob, rb = table_origins(rng, KC)
        a = mnop(rng, T.Image(ra, (32 + M + 31) // 32, True), M, K, 0, 32, oa)
        b = mnop(rng, T.Image(rb, (N + 31) // 32 + 1, True), N, K, 0, 0, ob)
        d = T.Desc(a, b, M, N, K, c=cbuf(M, N + 3), ldc=N + 3, k_splits=ks)
        descs.append(d)
        pre[id(d)] = 3 * rng.standard_normal((M, N))
    return descs, pre


def set_epi2(rng, cluster=False):
    """K and MN images at o_row0 = 256, o_col0 = 64 inside larger images, with and without C; two problems write adjacent
    column ranges of one image pair, a third the rows below; the mask image holds +, -, +0, -0, NaN and denormals; kZeroInvalid
    with ReLU"""
    OK, OMN, MK = out_img(896, 8, False), out_img(896, 8, True), mask_img(rng, 896, 8)
    A = T.Image(1024, 10, False)
    B = T.Image(512, 8, True)
    Bk = T.Image(256, 5, False)
    d0 = T.Desc(kop(rng, A, 200, 100, 256, 32), kop(rng, Bk, 70, 100, 128, 0), 200, 70, 100, c=cbuf(200, 70), ldc=70,
                bias=rng.standard_normal(70).astype(F32), flags=T.RELU | T.ZERO_INVALID | T.MASK_IMG, m_valid=150,
                o_k=OK, o_mn=OMN, mask=MK, o_row0=256, o_col0=64)
    d1 = T.Desc(kop(rng, A, 100, 33, 512, 64), mnop(rng, B, 33, 33, 32, 64), 100, 33, 33, flags=T.MASK_IMG,
                o_k=OK, o_mn=OMN, mask=MK, o_row0=256, o_col0=64 + 96)
    d2 = T.Desc(kop(rng, A, 129, 64 if not cluster else 224, 640, 0), mnop(rng, B, 128, 64 if not cluster else 224, 96, 128),
                129, 128, 64 if not cluster else 224, c=cbuf(129, 130), ldc=130, o_k=OK, o_row0=512, o_col0=64)
    d3 = T.Desc(kop(rng, A, 1, 1, 896, 0), mnop(rng, B, 1, 1, 480, 0), 1, 1, 1, flags=T.RELU, o_mn=OMN, mask=MK,
                o_row0=768, o_col0=32)
    return [d0, d1, d2, d3]


def set_ktab(rng):
    """the feed-forward d obs_emb GEMM: A K-major through (row block, column block) pairs out of order and repeated, B
    MN-major with a row origin per chunk"""
    descs = []
    for M, N, pairs in ((200, 100, [(256, 3), (0, 1), (256, 3), (0, 5), (256, 0)]), (77, 33, [(128, 2), (0, 2), (128, 4)])):
        KC = len(pairs)
        A = T.Image(max(p for p, _ in pairs) + 256, 6, False)
        x = rng.standard_normal((M, 32 * KC)).astype(F32)
        for c, (r0, cb) in enumerate(pairs):
            first = [i for i, p in enumerate(pairs) if p == (r0, cb)][0]
            A.put(x[:, 32 * first:32 * first + 32], r0, 32 * cb)   # a repeated pair reads the same block
        a = T.Op(A, 0, 0, np.array(pairs, dtype=np.int32).ravel())
        ob, rb = table_origins(rng, KC)
        b = mnop(rng, T.Image(rb, (N + 31) // 32 + 1, True), N, 32 * KC, 0, 32, ob)
        descs.append(T.Desc(a, b, M, N, 32 * KC, c=cbuf(M, N), ldc=N))
    return descs


def set_persistent(rng, epi):
    """more tiles than SMs (133, 265 and 505 tiles for epilogues 0, 1, 2); chunk counts 3, 5, 7 (not multiples of the 2 or 4
    stages of the ring) so that the stage parity wraps inside a tile; one single-tile problem per launch"""
    descs, pre = [], {}
    if epi == 0:
        shapes = [(1000, 1000, 65, {}), (600, 900, 150, dict(flags=T.ZERO_INVALID, m_valid=555)),
                  (300, 1100, 200, dict(bias=True, flags=T.RELU)), (50, 20, 1, {}), (128, 128, 33, {})]
        for M, N, K, kw in shapes:
            a = kop(rng, T.Image(M + 128, (K + 31) // 32 + 1, False), M, K, 128, 32)
            b = mnop(rng, T.Image(32 * ((K + 31) // 32) + 64, (N + 31) // 32 + 1, True), N, K, 64, 32)
            bias = rng.standard_normal(N).astype(F32) if kw.get('bias') else None
            descs.append(T.Desc(a, b, M, N, K, c=cbuf(M, N), ldc=N, bias=bias, flags=kw.get('flags', 0),
                                m_valid=kw.get('m_valid', 0)))
    elif epi == 1:
        for M, N, K, ks in [(1000, 1000, 96, 1), (1000, 1000, 160, 1), (700, 900, 224, 1), (500, 500, 100, 3),
                            (640, 1000, 33, 1), (1, 1, 1, 1)]:
            KC = (K + 31) // 32
            oa, ra = table_origins(rng, KC)
            ob, rb = table_origins(rng, KC)
            a = mnop(rng, T.Image(ra, (M + 31) // 32, True), M, K, 0, 0, oa)
            b = mnop(rng, T.Image(rb, (N + 31) // 32 + 1, True), N, K, 0, 32, ob)
            d = T.Desc(a, b, M, N, K, c=cbuf(M, N), ldc=N, k_splits=ks)
            descs.append(d)
            pre[id(d)] = rng.standard_normal((M, N))
    else:
        shapes = [(1024, 2048, 33, 'c k'), (1024, 2048, 65, 'mn mask'), (1000, 2000, 100, 'c k mn zi'), (900, 1900, 150, 'mn'),
                  (3, 5, 7, 'c k mn mask')]
        for M, N, K, what in shapes:
            w = what.split()
            a = kop(rng, T.Image(M + 128, (K + 31) // 32 + 1, False), M, K, 128, 32)
            b = kop(rng, T.Image(N + 256, (K + 31) // 32, False), N, K, 256, 0)
            rows, kb = M + 128, (N + 31) // 32 + 2
            descs.append(T.Desc(a, b, M, N, K, c=cbuf(M, N) if 'c' in w else None, ldc=N,
                                flags=(T.MASK_IMG if 'mask' in w else 0) | (T.ZERO_INVALID | T.RELU if 'zi' in w else 0),
                                m_valid=M - 300, o_k=out_img(rows, kb, False) if 'k' in w else None,
                                o_mn=out_img(rows, kb, True) if 'mn' in w else None,
                                mask=mask_img(rng, rows, kb) if 'mask' in w else None, o_row0=128, o_col0=64))
    return descs, pre


def set_cluster0(rng):
    """at most 8 tiles (tiles x CS <= 66 at CS = 8): KC 16, 2 (< CS 4 and 8: empty slices), 5 and 7 (not divisible by CS); A
    K-major, B MN-major (the d_hid form) and K-major"""
    A = T.Image(1024, 20, False)
    B = T.Image(1024, 10, True)
    Bk = T.Image(256, 8, False)
    return [T.Desc(kop(rng, A, 256, 500, 128, 32), mnop(rng, B, 256, 500, 32, 32), 256, 256, 500, c=cbuf(256, 256), ldc=256),
            T.Desc(kop(rng, A, 100, 33, 384, 0), kop(rng, Bk, 70, 33, 128, 32), 100, 70, 33, c=cbuf(100, 75), ldc=75,
                   bias=rng.standard_normal(70).astype(F32), flags=T.RELU),
            T.Desc(kop(rng, A, 129, 150, 512, 64), mnop(rng, B, 31, 150, 576, 0), 129, 31, 150, c=cbuf(129, 31), ldc=31,
                   flags=T.ZERO_INVALID, m_valid=100),
            T.Desc(kop(rng, A, 1, 224, 768, 0), mnop(rng, B, 1, 224, 768, 288), 1, 1, 224, c=cbuf(1, 1), ldc=1)]


PREC = pytest.mark.parametrize('x3', [True, False], ids=['tf32x3', 'tf32'])


# ---- cases ----------------------------------------------------------------------------------------------------------------------
@PREC
def test_grouped_epilogue0(cuda, x3):
    descs = set_epi0(np.random.default_rng(10))
    with kernel_forms(('grouped', x3, 0)):
        first = run_and_check(descs, 0, x3, 'grouped')
        same_bits(first, launch(descs, 0, x3))     # deterministic


@PREC
def test_grouped_epilogue1_split_k_into_prefilled_c(cuda, x3):
    descs, pre = set_epi1(np.random.default_rng(11))
    with kernel_forms(('grouped', x3, 1)):
        run_and_check(descs, 1, x3, 'grouped', prefill=pre)


@PREC
def test_grouped_epilogue2_images(cuda, x3):
    descs = set_epi2(np.random.default_rng(12))
    with kernel_forms(('grouped', x3, 2)):
        first = run_and_check(descs, 2, x3, 'grouped')
        same_bits(first, launch(descs, 2, x3))


@PREC
def test_chunk_table(cuda, x3):
    descs = set_ktab(np.random.default_rng(13))
    with kernel_forms(('ktab', x3, 0)):
        first = run_and_check(descs, 0, x3, 'ktab', ktab=True)
        same_bits(first, launch(descs, 0, x3, ktab=True))


@PREC
@pytest.mark.parametrize('cs', [2, 4, 8])
def test_cluster_epilogue0(cuda, x3, cs):
    descs = set_cluster0(np.random.default_rng(30 + cs))
    assert sum(((d.M + 127) // 128) * ((d.N + 127) // 128) for d in descs) * cs <= 66
    with kernel_forms(('cluster{}'.format(cs), x3, 0)):
        first = run_and_check(descs, 0, x3, 'cluster{}'.format(cs), cs=cs)
        same_bits(first, launch(descs, 0, x3, cs=cs))


@PREC
@pytest.mark.parametrize('cs', [2, 4, 8])
def test_cluster_epilogue2(cuda, x3, cs):
    descs = set_epi2(np.random.default_rng(40 + cs), cluster=True)
    assert sum(((d.M + 127) // 128) * ((d.N + 127) // 128) for d in descs) * cs <= 66
    with kernel_forms(('cluster{}'.format(cs), x3, 2)):
        first = run_and_check(descs, 2, x3, 'cluster{}'.format(cs), cs=cs)
        same_bits(first, launch(descs, 2, x3, cs=cs))


@PREC
@pytest.mark.parametrize('form', ['grouped', 'cluster2'])
def test_nan_padding_never_reaches_a_stored_value(cuda, x3, form):
    """mostly padding: every tile row beyond M of the K-major operands and every column beyond N of the MN-major ones is
    NaN (Image's fill), K padding zero; every stored value must be finite"""
    rng = np.random.default_rng(50)
    OK, OMN = out_img(256, 4, False), out_img(256, 4, True)
    descs = []
    for i, (M, N, K) in enumerate([(1, 1, 1), (5, 3, 40), (127, 97, 7)]):
        a = kop(rng, T.Image(128, 2, False), M, K, 0, 0)
        b = mnop(rng, T.Image(64, 4, True), N, K, 0, 0) if i != 1 else kop(rng, T.Image(128, 2, False), N, K, 0, 0)
        descs.append(T.Desc(a, b, M, N, K, c=cbuf(M, N), ldc=N, o_k=OK, o_mn=OMN, o_row0=(0, 0, 128)[i], o_col0=(0, 32, 0)[i]))
    cs = 2 if form == 'cluster2' else 1
    with kernel_forms((form, x3, 2)):
        out = launch(descs, 2, x3, cs=cs)
    for d in descs:
        assert np.isfinite(out[(id(d.c), None)][T.c_offsets(d)]).all()
    check(descs, out, 2, x3, form, cs=cs)


@PREC
@pytest.mark.parametrize('epi', [0, 1, 2])
def test_persistent_matches_grouped_bit_for_bit(cuda, monkeypatch, x3, epi):
    """tc_persist.cuh: same arithmetic and epilogues as k_grouped, so identical results (epilogue 1: where k_splits = 1;
    split problems add their partial sums in whatever order the CTAs finish)"""
    descs, pre = set_persistent(np.random.default_rng(20 + epi), epi)
    assert sum(((d.M + 127) // 128) * ((d.N + 127) // 128) * d.k_splits for d in descs) > 132
    with kernel_forms(('persistent', x3, epi), ('grouped', x3, epi)):
        monkeypatch.setenv('PPB_PERSISTENT', '1')
        pers = run_and_check(descs, epi, x3, 'persistent', prefill=pre)
        if epi != 1:
            same_bits(pers, launch(descs, epi, x3))
        monkeypatch.setenv('PPB_PERSISTENT', '0')
        grouped = run_and_check(descs, epi, x3, 'grouped', prefill=pre)
    exact = {(id(d.c), None) for d in descs if d.k_splits == 1 and d.c is not None} if epi == 1 else set(pers)
    for k in exact:
        np.testing.assert_array_equal(pers[k].view(np.uint32), grouped[k].view(np.uint32))


def test_zz_report_ratios():
    """the largest error / bound per form, epilogue and precision over the cases above (printed with -s)"""
    for k in sorted(RATIOS):
        print('error/bound max {:12s} epilogue {} {:7s} {:.3g}'.format(*k, RATIOS[k]))
    assert all(v < 1 for v in RATIOS.values())
