"""CPU: the float64 restatement of the tensor-core GEMM descriptors (tests/tc_fp64.py) — its ctypes mirror of tcg::Problem
against the compiled struct, its image packer against the layout helpers of tc.cuh, its gather against the dense blocks the
images were built from, its bound against an fp32 matmul — and the descriptor checks of ppb_tc_run_problems, which refuse
every combination the kernels do not implement before anything is uploaded or launched."""
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from tests import tc_fp64 as T

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'pyprob_b200', 'csrc')
NVCC = os.environ.get('NVCC') or shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
ROWS, KB = 300, 3

PROGRAM = r'''
#include <stddef.h>
#include <stdio.h>
#include "tc_grouped.cuh"
#define OP(p, f) printf(#p "." #f " %%zu\n", offsetof(tcg::Problem, p) + offsetof(tcg::Operand, f));
#define PR(f) printf(#f " %%zu\n", offsetof(tcg::Problem, f));
int main() {
  printf("sizeof.Operand %%zu\nsizeof.Problem %%zu\n", sizeof(tcg::Operand), sizeof(tcg::Problem));
  OP(a, hi) OP(a, lo) OP(a, k_rows) OP(a, kb) OP(a, mn) OP(a, row0) OP(a, col0)
  OP(b, hi) OP(b, lo) OP(b, k_rows) OP(b, kb) OP(b, mn) OP(b, row0) OP(b, col0)
  PR(M) PR(N) PR(K) PR(m_valid) PR(flags) PR(c) PR(ldc) PR(bias) PR(o_k_hi) PR(o_k_lo) PR(o_mn_hi) PR(o_mn_lo) PR(mask_hi)
  PR(o_kb) PR(o_row0) PR(o_col0) PR(tile_start) PR(tiles_m) PR(tiles_n) PR(k_splits)
  for (int64_t row = 0; row < %(rows)d; ++row)
    for (int64_t k = 0; k < 32 * %(kb)d; ++k)
      printf("off %%lld %%lld\n", (long long)tc::packed_offset(row, k, %(kb)d), (long long)tc::packed_offset_mn(row, k, %(kb)d));
  return 0;
}
''' % {'rows': ROWS, 'kb': KB}


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip('nvcc not available')
    d = tmp_path_factory.mktemp('tc_fp64')
    src, exe = d / 'structs.cu', d / 'structs'
    src.write_text(PROGRAM)
    subprocess.check_call([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-std=c++17', '-I', CSRC, '-o', str(exe),
                           str(src)])
    fields, offs = {}, []
    for line in subprocess.check_output([str(exe)]).decode().splitlines():
        w = line.split()
        if w[0] == 'off':
            offs.append((int(w[1]), int(w[2])))
        else:
            fields[w[0]] = int(w[1])
    return fields, np.array(offs, dtype=np.int64).reshape(ROWS, 32 * KB, 2)


def test_ctypes_mirror_matches_the_compiled_structs(compiled):
    fields, _ = compiled
    assert fields.pop('sizeof.Operand') == C_sizeof(T.Operand) == 40
    assert fields.pop('sizeof.Problem') == C_sizeof(T.Problem) == 200
    assert fields == T.field_offsets()
    assert (fields['a.hi'], fields['b.hi'], fields['M'], fields['c'], fields['mask_hi'], fields['k_splits']) == \
        (0, 40, 80, 104, 160, 192)


def C_sizeof(t):
    import ctypes
    return ctypes.sizeof(t)


def test_packer_offsets_match_the_layout_helpers(compiled):
    _, offs = compiled
    row, col = np.meshgrid(np.arange(ROWS), np.arange(32 * KB), indexing='ij')
    np.testing.assert_array_equal(T.packed_offset(row, col, KB, False), offs[..., 0])
    np.testing.assert_array_equal(T.packed_offset(row, col, KB, True), offs[..., 1])


def test_rna_split():
    bits = np.array([0x3F801000, 0xBF801000, 0x3F800FFF, 0x3F803000, 0x7F7FF000, 0x00000001, 0x80000000, 0x3FFFF000],
                    dtype=np.uint32)
    want = np.array([0x3F802000, 0xBF802000, 0x3F800000, 0x3F804000, 0x7F800000, 0x00000000, 0x80000000, 0x40000000],
                    dtype=np.uint32)
    np.testing.assert_array_equal(T.rna_tf32(bits.view(np.float32)).view(np.uint32), want)
    x = np.random.default_rng(1).standard_normal(10000).astype(np.float32) * np.float32(1e3)
    hi, lo = T.split_tf32(x)
    assert not (hi.view(np.uint32) & 0x1FFF).any() and not (lo.view(np.uint32) & 0x1FFF).any()
    err = np.abs(hi.astype(np.float64) + lo - x)
    assert (err <= 2.0 ** -22 * np.abs(x)).all()


def test_image_put_places_the_split_at_the_layout_offsets():
    rng = np.random.default_rng(2)
    for mn in (False, True):
        im = T.Image(260, 4, mn)
        x = rng.standard_normal((100, 70)).astype(np.float32)
        im.put(x, 131, 33)
        r, c = np.meshgrid(np.arange(100) + 131, np.arange(70) + 33, indexing='ij')
        off = T.packed_offset(r, c, 4, mn)
        hi, lo = T.split_tf32(x)
        np.testing.assert_array_equal(im.hi[off], hi)
        np.testing.assert_array_equal(im.lo[off], lo)
        rest = np.ones(im.hi.size, dtype=bool)
        rest[off.ravel()] = False
        assert (im.hi.view(np.uint32)[rest] == T.NAN_FILL).all()


@pytest.mark.parametrize('x3', [True, False])
def test_gather_returns_the_dense_blocks(x3):
    """every operand mode: K-major at (row0, col0), K-major through a chunk table, MN-major at (row0, col0), MN-major
    through a row table"""
    rng = np.random.default_rng(3)
    M, K = 150, 70
    KC = 3
    X = rng.standard_normal((M, 32 * KC)).astype(np.float32)
    X[:, K:] = 0
    hi, lo = T.split_tf32(X)
    want = hi.astype(np.float64) + (lo if x3 else 0)

    im = T.Image(512, 6, False)
    im.put(X, 128, 64)
    np.testing.assert_array_equal(T.gather(T.Op(im, 128, 64), M, KC, x3), want)

    pairs = [(256, 5), (0, 1), (256, 2)]      # chunk c: (row block origin, column block); out of order
    im = T.Image(512, 6, False)
    for c, (r0, cb) in enumerate(pairs):
        im.put(X[:, 32 * c:32 * c + 32], r0, 32 * cb)
    kr = np.array(pairs, dtype=np.int32).ravel()
    np.testing.assert_array_equal(T.gather(T.Op(im, k_rows=kr), M, KC, x3), want)

    im = T.Image(200, 7, True)
    im.put(X.T, 32, 64)
    np.testing.assert_array_equal(T.gather(T.Op(im, 32, 64), M, KC, x3), want)

    origins = [160, 32, 96]                    # chunk c at image rows origins[c] ..
    im = T.Image(200, 7, True)
    for c, r0 in enumerate(origins):
        im.put(X[:, 32 * c:32 * c + 32].T, r0, 32)
    np.testing.assert_array_equal(T.gather(T.Op(im, 0, 32, np.array(origins, dtype=np.int32)), M, KC, x3), want)


@pytest.mark.parametrize('K', [1, 31, 200, 1000, 4096])
def test_bound_exceeds_an_fp32_matmul(K):
    """the per-element bound holds for an fp32 matmul of the same operands (sequential fp32 sums: K roundings, more than the
    kernels' KC), so it is not tighter than fp32 arithmetic itself"""
    rng = np.random.default_rng(K)
    A = rng.standard_normal((64, K)).astype(np.float32)
    B = rng.standard_normal((48, K)).astype(np.float32)
    want = A.astype(np.float64) @ B.T.astype(np.float64)
    mag = np.abs(A.astype(np.float64)) @ np.abs(B.T.astype(np.float64))
    got = (A @ B.T).astype(np.float64)
    seq = np.zeros((64, 48), dtype=np.float32)
    for k in range(0, K, max(1, K // 64)):         # a sequential fp32 sum over slices
        seq += A[:, k:k + max(1, K // 64)] @ B[:, k:k + max(1, K // 64)].T
    for x3 in (True, False):
        bound = T.tau(x3, (K + 31) // 32) * mag
        assert (np.abs(got - want) <= bound).all()
        assert (np.abs(seq.astype(np.float64) - want) <= bound).all()


def test_write_sets_and_ranges():
    a = T.Image(256, 2, False)
    b = T.Image(64, 4, True)
    c = np.zeros(10 * 40, dtype=np.float32)
    ok = T.Image(512, 5, False)
    d = T.Desc(T.Op(a, 128, 32), T.Op(b, 32, 64), M=10, N=33, K=20, c=c, ldc=40, o_k=ok, o_row0=256, o_col0=64)
    ws = T.write_sets([d], 2)
    assert len(ws[(id(c), None)][2]) == 10 * 33 and int(ws[(id(c), None)][2].max()) == 9 * 40 + 32
    assert len(ws[(id(ok), 'hi')][2]) == 10 * 64
    for obj, part, lo, hi in T.touched_ranges(d, True, 2):
        assert 0 <= lo < hi <= T.size_of(obj, part)


# ---- descriptor checks of ppb_tc_run_problems ------------------------------------------------------------------------------
# Run in a child process that sees no CUDA device: a check that failed to refuse would reach cudaMalloc and fail there with
# a CUDA error (not the check's message), never launch a kernel on fake pointers.
CHILD = r'''
import ctypes, json, os, sys
sys.path.insert(0, %(root)r)
from pyprob_b200 import _lib
from tests import tc_fp64 as T
lib = _lib.load()
F = 0x100000   # fake, never dereferenced: every call below is refused on the host, or fails on the missing device

def base(**kw):
    p = T.Problem()
    p.a = T.Operand(F, F, None, 4, 0, 0, 0); p.b = T.Operand(F, F, None, 4, 0, 0, 0)
    p.M, p.N, p.K, p.c, p.ldc = 100, 100, 100, F, 100
    for k, v in kw.items():
        obj = p
        *path, last = k.split('__')
        for s in path:
            obj = getattr(obj, s)
        setattr(obj, last, v)
    return p

out = []
for name, kw, epi, cs, ktab, prec in json.loads(sys.argv[1]):
    arr = (T.Problem * 2)(base(**kw) if name.startswith('valid') else base(), base(**kw))
    n0 = lib.ppb_launch_count()
    rc = lib.ppb_tc_run_problems(ctypes.byref(arr), 2 if name != 'no problems' else 0, epi, cs, ktab, prec, None)
    out.append([name, rc, _lib.last_error(), lib.ppb_launch_count() - n0])
print(json.dumps(out))
'''

F = 0x100000   # the child's fake address
ZI, RELU, MASK = T.ZERO_INVALID, T.RELU, T.MASK_IMG
# name, fields of the second problem (operand fields as a__x / b__x), epi, cluster size, chunk table, precision, message
REJECTED = [
    ('epilogue 3', {}, 3, 1, 0, 0, 'epilogue must be 0'),
    ('epilogue -1', {}, -1, 1, 0, 0, 'epilogue must be 0'),
    ('precision 2', {}, 0, 1, 0, 2, 'precision must be'),
    ('cluster size 3', {}, 0, 3, 0, 0, 'cluster size must be'),
    ('no problems', {}, 0, 1, 0, 0, 'no problems'),
    ('cluster with epilogue 1', {}, 1, 2, 0, 0, 'the cluster form has no red.add'),
    ('cluster with k_splits', {'k_splits': 2}, 0, 4, 0, 0, 'the cluster form splits the reduction'),
    ('cluster with a chunk table', {'a__k_rows': F}, 0, 8, 1, 0, 'the cluster form has no red.add epilogue and no chunk'),
    ('chunk table with epilogue 2', {'a__k_rows': F, 'o_k_hi': F, 'o_k_lo': F, 'o_kb': 4}, 2, 1, 1, 0,
     'the chunk table runs with epilogue 0'),
    ('chunk table with epilogue 1', {'a__k_rows': F}, 1, 1, 1, 0, 'the chunk table runs with epilogue 0'),
    ('chunk table without k_rows', {}, 0, 1, 1, 0, 'needs a K-major A with k_rows'),
    ('chunk table with an MN-major A', {'a__mn': 1, 'a__k_rows': F}, 0, 1, 1, 0, 'needs a K-major A with k_rows'),
    ('K-major k_rows without the chunk table', {'a__k_rows': F}, 0, 1, 0, 0, 'read by the chunk table only'),
    ('K-major B with k_rows', {'b__k_rows': F}, 0, 1, 0, 0, 'a K-major B has no chunk table'),
    ('k_splits with epilogue 0', {'k_splits': 2}, 0, 1, 0, 0, 'k_splits > 1 adds partial sums'),
    ('k_splits with images', {'k_splits': 3, 'o_k_hi': F, 'o_k_lo': F, 'o_kb': 4}, 2, 1, 0, 0,
     'k_splits > 1 adds partial sums'),
    ('k_splits with bias', {'k_splits': 2, 'bias': F}, 1, 1, 0, 0, 'k_splits > 1 adds partial sums'),
    ('k_splits with ReLU', {'k_splits': 2, 'flags': RELU}, 1, 1, 0, 0, 'k_splits > 1 adds partial sums'),
    ('k_splits with the mask', {'k_splits': 2, 'flags': MASK, 'mask_hi': F, 'o_kb': 4}, 1, 1, 0, 0,
     'k_splits > 1 adds partial sums'),
    ('k_splits with kZeroInvalid', {'k_splits': 7, 'flags': ZI, 'm_valid': 50}, 1, 1, 0, 0, 'k_splits > 1 adds partial sums'),
    ('images with epilogue 1', {'o_mn_hi': F, 'o_mn_lo': F, 'o_kb': 4}, 1, 1, 0, 0, 'images and the mask need epilogue 2'),
    ('mask with epilogue 0', {'flags': MASK, 'mask_hi': F, 'o_kb': 4}, 0, 1, 0, 0, 'images and the mask need epilogue 2'),
    ('mask flag without a mask image', {'flags': MASK, 'o_k_hi': F, 'o_k_lo': F, 'o_kb': 4}, 2, 1, 0, 0,
     'kMaskImg without a mask image'),
    ('unknown flag 2', {'flags': 2}, 0, 1, 0, 0, 'unknown flags'),
    ('epilogue 0 without c', {'c': None}, 0, 1, 0, 0, 'epilogues 0 and 1 need c'),
    ('epilogue 1 without c', {'c': None}, 1, 1, 0, 0, 'epilogues 0 and 1 need c'),
    ('epilogue 2 without any output', {'c': None}, 2, 2, 0, 0, 'epilogue 2 without any output'),
    ('ldc below N', {'ldc': 99}, 0, 1, 0, 0, 'ldc < N'),
    ('K image hi without lo', {'o_k_hi': F, 'o_kb': 4}, 2, 1, 0, 0, 'needs both its hi and lo'),
    ('MN image hi without lo', {'o_mn_hi': F, 'o_kb': 4}, 2, 4, 0, 0, 'needs both its hi and lo'),
    ('3xTF32 without A lo', {'a__lo': None}, 0, 1, 0, 0, '3xTF32 needs the operand lo parts'),
    ('3xTF32 without B lo', {'b__lo': None}, 0, 2, 0, 0, '3xTF32 needs the operand lo parts'),
    ('no A image', {'a__hi': None}, 0, 1, 0, 1, 'operand without an image'),
    ('empty M', {'M': 0}, 0, 1, 0, 0, 'M, N and K must be positive'),
    ('K-major row0 % 128', {'a__row0': 64}, 0, 1, 0, 0, 'operand offset off the layout'),
    ('K-major col0 % 32', {'b__col0': 16}, 0, 1, 0, 0, 'operand offset off the layout'),
    ('MN-major row0 % 32', {'a__mn': 1, 'a__row0': 16}, 0, 1, 0, 0, 'operand offset off the layout'),
    ('MN-major col0 % 32', {'b__mn': 1, 'b__col0': 8}, 0, 1, 0, 0, 'operand offset off the layout'),
    ('o_row0 % 128', {'o_k_hi': F, 'o_k_lo': F, 'o_kb': 4, 'o_row0': 32}, 2, 1, 0, 0, 'output image geometry off the layout'),
    ('o_col0 % 32', {'o_mn_hi': F, 'o_mn_lo': F, 'o_kb': 4, 'o_col0': 48}, 2, 2, 0, 0, 'output image geometry off the layout'),
    ('no o_kb', {'o_k_hi': F, 'o_k_lo': F}, 2, 1, 0, 0, 'output image geometry off the layout'),
]
ACCEPTED = [('valid epilogue 0', {}, 0, 1, 0, 0), ('valid split-K', {'k_splits': 9}, 1, 1, 0, 0),
            ('valid cluster images', {'c': None, 'o_mn_hi': F, 'o_mn_lo': F, 'o_kb': 4, 'o_row0': 128, 'o_col0': 32,
                                      'flags': MASK | RELU | ZI, 'mask_hi': F}, 2, 8, 0, 1),
            ('valid chunk table', {'a__k_rows': F, 'b__mn': 1, 'b__k_rows': F, 'a__lo': None, 'b__lo': None}, 0, 1, 1, 1)]


def _child(cases):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES='')
    out = subprocess.check_output([sys.executable, '-c', CHILD % {'root': ROOT},
                                   json.dumps([c[:6] for c in cases])], env=env, cwd=ROOT)
    return json.loads(out.decode().strip().splitlines()[-1])


def test_rejected_descriptors_are_refused_before_any_launch():
    for (name, rc, msg, launches), case in zip(_child(REJECTED), REJECTED):
        assert rc != 0 and msg.startswith('check_problems: ') and case[6] in msg, (name, rc, msg)
        assert launches == 0, name


def test_valid_descriptors_pass_the_checks():
    """the same calls with a supported combination get past every check (and then fail on the missing device)"""
    for name, rc, msg, launches in _child(ACCEPTED):
        assert rc != 0 and not msg.startswith('check_problems'), (name, msg)
        assert launches == 0, name
