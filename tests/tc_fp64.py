"""Float64 restatement of the tensor-core GEMM descriptors (tcg::Problem, csrc/tc_grouped.cuh) for the descriptor tests.

Everything here is built on the host, independently of the library: the tf32 tile images (DESIGN.md, tc.cuh: tile (rt, cb)
at float (rt * KB + cb) * 4096, row r of a tile at r * 32, the 16-byte chunk c16 of a K-format row at c16 ^ (r & 7), the
32-byte chunk c32 of an MN-format row at c32 ^ (r & 3)), the tf32 split (cvt.rna: round half away from zero at bit 13,
lo = rna(x - hi)), the operands as each kernel reads them, the epilogues, the write set of every descriptor and the float
ranges it reads and writes.

Error bound.  Per output element the kernels compute sum_k A_eff[m, k] B_eff[n, k] (+ bias, + prefilled C) where A_eff, B_eff
are the operands as read: hi + lo in 3xTF32, hi alone in TF32.  Against that exact sum the arithmetic of DESIGN.md
§Tensor-core GEMM makes these errors (u = 2^-24, S = sum_k |A_eff B_eff| + |bias| + |C prefill|):
  * products: a tf32 x tf32 product has 22 significant bits and is exact in fp32.  3xTF32 drops a_lo b_lo; |a_lo| <=
    2^-11 (1 + 2^-11) |a_hi| and |a_hi| <= |A_eff| / (1 - 2^-10), so the dropped term is at most 2^-22 (1 + 2^-8) of
    |A_eff B_eff| (the lo parts are read as stored: their own rounding is inside A_eff, not an error);
  * one 32-element chunk is accumulated by the tensor core into a zeroed fragment in J wgmma k8 steps (J = 12 in 3xTF32:
    cross terms and hi hi for each of the four k8 slices; J = 4 in TF32), each adding 8 products to the running fragment.
    The tensor core aligns the addends to the largest one and truncates: each of the 9 addends loses less than one unit in
    the last place (2u of the largest addend), and the normalised result loses less than one more.  Every addend and every
    partial result is at most the chunk's term sum S_c (plus higher-order terms), so one step errs by less than
    10 * 2u * S_c and the chunk by less than 20 J u S_c;
  * the chunk sums are added to the fp32 accumulator with round-to-nearest: KC additions, each within u of a partial sum,
    at most KC u S;
  * the cluster form adds its CS partial tiles (CS more additions), the epilogue adds the bias (one), epilogue 1 adds the
    k_splits partial results into C with red.add (k_splits more);
  so |got - exact| <= tau S with tau = (1 + 2^-10) (20 J u + (KC + CS + 1 + k_splits) u + [3xTF32] 2^-22 (1 + 2^-8)),
  the leading factor covering the second-order terms.  That is 240 u + ... in 3xTF32 (about 1.5e-5 + KC 6e-8) and 80 u
  + ... in TF32.  Nothing in tau is fitted to observed errors; the truncation term is the loose one (an addend loses a full
  unit only in the worst alignment), so observed ratios error / bound sit far below 1.

The caller's contract, which every test image keeps: the K padding of the last reduction chunk (K-major columns, MN-major
rows at or beyond K) is zero in both operands.  Padding in M and N (rows of a K-major tile beyond M, columns of an MN-major
block beyond N) may hold anything, NaN included; the tests fill it with NaN.
"""
import ctypes as C
from dataclasses import dataclass, field

import numpy as np

U = 2.0 ** -24
NAN_FILL = 0x7FC0F00D     # quiet NaN of the operand padding
SENTINEL = 0x7FC0DEAD     # quiet NaN in every output float outside the write set

# tcg flags (tc_grouped.cuh)
RELU, MASK_IMG, ZERO_INVALID = 1, 4, 8


class Operand(C.Structure):
    _fields_ = [('hi', C.c_void_p), ('lo', C.c_void_p), ('k_rows', C.c_void_p), ('kb', C.c_int), ('mn', C.c_int),
                ('row0', C.c_int), ('col0', C.c_int)]


class Problem(C.Structure):
    _fields_ = [('a', Operand), ('b', Operand), ('M', C.c_int), ('N', C.c_int), ('K', C.c_int), ('m_valid', C.c_int),
                ('flags', C.c_int), ('c', C.c_void_p), ('ldc', C.c_int64), ('bias', C.c_void_p),
                ('o_k_hi', C.c_void_p), ('o_k_lo', C.c_void_p), ('o_mn_hi', C.c_void_p), ('o_mn_lo', C.c_void_p),
                ('mask_hi', C.c_void_p), ('o_kb', C.c_int), ('o_row0', C.c_int), ('o_col0', C.c_int),
                ('tile_start', C.c_int), ('tiles_m', C.c_int), ('tiles_n', C.c_int), ('k_splits', C.c_int)]


def field_offsets():
    """{'a.hi': offset, ...} of every field of Problem, nested operand fields as 'a.<name>' / 'b.<name>'"""
    out = {}
    for name, _ in Problem._fields_:
        off = getattr(Problem, name).offset
        if name in ('a', 'b'):
            for sub, _ in Operand._fields_:
                out[name + '.' + sub] = off + getattr(Operand, sub).offset
        else:
            out[name] = off
    return out


# ---- tf32 split and the tile-image layout ---------------------------------------------------------------------------------
def rna_tf32(x):
    """cvt.rna.tf32.f32: round the fp32 magnitude to 10 mantissa bits, ties away from zero"""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def split_tf32(x):
    x = np.asarray(x, dtype=np.float32)
    hi = rna_tf32(x)
    return hi, rna_tf32(x - hi)


def ceil32(n):
    return (n + 31) // 32 * 32


def img_floats(rows, kb):
    return (rows + 127) // 128 * kb * 4096


def packed_offset(row, col, kb, mn):
    """float offset of image element (row, col) in an image with kb column blocks, K format (mn False) or MN format"""
    row, col = np.asarray(row, dtype=np.int64), np.asarray(col, dtype=np.int64)
    r, c = row % 128, col % 32
    span = ((row // 128) * kb + col // 32) * 4096 + r * 32
    if mn:
        return span + (((c // 8) ^ (r % 4)) * 8) + c % 8
    return span + (((c // 4) ^ (r % 8)) * 4) + c % 4


class Image:
    """Host tf32 tile image (hi and lo parts) of rows x (32 kb) logical elements in one format; every float starts as `fill`."""

    def __init__(self, rows, kb, mn, fill=NAN_FILL):
        self.rows, self.kb, self.mn = (rows + 127) // 128 * 128, kb, bool(mn)
        n = img_floats(rows, kb)
        self.hi = np.full(n, fill, dtype=np.uint32).view(np.float32)
        self.lo = np.full(n, fill, dtype=np.uint32).view(np.float32)

    def put(self, x, row0=0, col0=0):
        """store the rna split of the dense fp32 block x at image rows row0.., columns col0.."""
        x = np.asarray(x, dtype=np.float32)
        r, c = np.meshgrid(np.arange(x.shape[0]) + row0, np.arange(x.shape[1]) + col0, indexing='ij')
        assert r.max() < self.rows and c.max() < 32 * self.kb
        off = packed_offset(r, c, self.kb, self.mn)
        hi, lo = split_tf32(x)
        self.hi[off], self.lo[off] = hi, lo

    def value(self, off, x3):
        """fp64 value at float offsets off as a kernel reads it: hi + lo (x3) or hi"""
        v = self.hi[off].astype(np.float64)
        return v + self.lo[off].astype(np.float64) if x3 else v


# ---- descriptors ----------------------------------------------------------------------------------------------------------
@dataclass(eq=False)
class Op:
    img: Image
    row0: int = 0
    col0: int = 0
    k_rows: np.ndarray = None      # int32: MN-major row origin per chunk, or K-major (row block origin, column block) pairs


@dataclass(eq=False)
class Desc:
    """One tcg::Problem with host objects in place of device pointers (c: fp32 array of at least (M - 1) ldc + N floats)."""
    a: Op
    b: Op
    M: int
    N: int
    K: int
    c: np.ndarray = None
    ldc: int = 0
    bias: np.ndarray = None
    flags: int = 0
    m_valid: int = 0
    o_k: Image = None
    o_mn: Image = None
    mask: Image = None
    o_row0: int = 0
    o_col0: int = 0
    k_splits: int = 1
    o_kb: int = field(init=False, default=0)

    def __post_init__(self):
        for im in (self.o_k, self.o_mn, self.mask):
            if im is not None:
                assert self.o_kb in (0, im.kb), 'output and mask images share one geometry'
                self.o_kb = im.kb

    @property
    def KC(self):
        return (self.K + 31) // 32


def to_problem(d, ptr, x3):
    """ctypes Problem of d; ptr(obj, part) gives the device address of a host object ('hi' / 'lo' of an Image, else None).
    Operand lo parts are passed in 3xTF32 only: the single-pass path must not read them."""
    def op(o, mn):
        return Operand(ptr(o.img, 'hi'), ptr(o.img, 'lo') if x3 else None, ptr(o.k_rows, None) if o.k_rows is not None else None,
                       o.img.kb, int(mn), o.row0, o.col0)
    p = Problem()
    p.a, p.b = op(d.a, d.a.img.mn), op(d.b, d.b.img.mn)
    p.M, p.N, p.K, p.m_valid, p.flags = d.M, d.N, d.K, d.m_valid, d.flags
    p.c = ptr(d.c, None) if d.c is not None else None
    p.ldc = d.ldc
    p.bias = ptr(d.bias, None) if d.bias is not None else None
    if d.o_k is not None:
        p.o_k_hi, p.o_k_lo = ptr(d.o_k, 'hi'), ptr(d.o_k, 'lo')
    if d.o_mn is not None:
        p.o_mn_hi, p.o_mn_lo = ptr(d.o_mn, 'hi'), ptr(d.o_mn, 'lo')
    if d.mask is not None:
        p.mask_hi = ptr(d.mask, 'hi')
    p.o_kb, p.o_row0, p.o_col0, p.k_splits = d.o_kb, d.o_row0, d.o_col0, d.k_splits
    return p


# ---- the operands as the kernels read them --------------------------------------------------------------------------------
def operand_offsets(o, n_rows, KC):
    """[n_rows, 32 KC] float offsets into o.img of operand element (row, k) as the loader reads it (load_operand)"""
    kk = np.arange(32 * KC)
    c, j = kk // 32, kk % 32
    m = np.arange(n_rows)[:, None]
    if not o.img.mn:
        if o.k_rows is not None:   # chunk table: chunk c = rows k_rows[2c] + m of column block k_rows[2c + 1]
            t = np.asarray(o.k_rows, dtype=np.int64)
            return packed_offset(t[2 * c][None, :] + m, (32 * t[2 * c + 1] + j)[None, :], o.img.kb, False)
        return packed_offset(o.row0 + m, (o.col0 + kk)[None, :], o.img.kb, False)
    r0 = np.asarray(o.k_rows, dtype=np.int64)[c] if o.k_rows is not None else o.row0 + 32 * c
    return packed_offset((r0 + j)[None, :], o.col0 + m, o.img.kb, True)


def gather(o, n_rows, KC, x3):
    """dense fp64 [n_rows, 32 KC] operand as read: A_eff (n_rows = M) or B_eff (n_rows = N)"""
    return o.img.value(operand_offsets(o, n_rows, KC), x3)


def tau(x3, KC, cs=1, k_splits=1):
    """per-element bound factor (module docstring)"""
    J = 12 if x3 else 4
    t = 20 * J * U + (KC + cs + 1 + k_splits) * U + (2.0 ** -22 * (1 + 2.0 ** -8) if x3 else 0.0)
    return t * (1 + 2.0 ** -10)


def reference(d, x3, cs=1, c_prefill=None):
    """(value, bound, forced_zero) of every output element [M, N] of descriptor d: the epilogue in fp64 on the operands as
    read, |got - value| <= bound, and the elements the epilogue must set to exactly 0 (rows at or beyond m_valid under
    kZeroInvalid, mask not > 0).  c_prefill: the [M, N] C that epilogue 1 adds into."""
    A, B = gather(d.a, d.M, d.KC, x3), gather(d.b, d.N, d.KC, x3)
    val = A @ B.T
    mag = np.abs(A) @ np.abs(B).T
    if d.bias is not None:
        val = val + d.bias[:d.N].astype(np.float64)[None, :]
        mag = mag + np.abs(d.bias[:d.N].astype(np.float64))[None, :]
    if d.flags & RELU:
        val = np.maximum(val, 0.0)
    zero = np.zeros((d.M, d.N), dtype=bool)
    if d.flags & ZERO_INVALID:
        zero[max(d.m_valid, 0):, :] = True
    if d.flags & MASK_IMG:
        mk = d.mask.hi[out_offsets(d, False)[:, :d.N]]
        zero |= ~(mk > 0)
    val = np.where(zero, 0.0, val)
    if c_prefill is not None:
        val = val + c_prefill
        mag = mag + np.abs(c_prefill)
    return val, tau(x3, d.KC, cs, d.k_splits) * mag, zero


# ---- write sets and the ranges a descriptor touches -----------------------------------------------------------------------
def c_offsets(d):
    """[M, N] float offsets of C"""
    return np.arange(d.M)[:, None] * d.ldc + np.arange(d.N)[None, :]


def out_offsets(d, mn):
    """[M, ceil32(N)] float offsets of the output image positions (o_row0 + m, o_col0 + n), padding columns included"""
    r = d.o_row0 + np.arange(d.M)[:, None]
    c = d.o_col0 + np.arange(ceil32(d.N))[None, :]
    return packed_offset(r, c, d.o_kb, mn)


def write_sets(descs, epi):
    """{id(buffer): (buffer, 'hi' / 'lo' / None, sorted unique float offsets written)} over all descriptors of one launch"""
    acc = {}

    def add(obj, part, off):
        key = (id(obj), part)
        acc.setdefault(key, (obj, part, []))[2].append(np.asarray(off).ravel())
    for d in descs:
        if d.c is not None:
            add(d.c, None, c_offsets(d))
        if epi == 2:
            for im, mn in ((d.o_k, False), (d.o_mn, True)):
                if im is not None:
                    add(im, 'hi', out_offsets(d, mn))
                    add(im, 'lo', out_offsets(d, mn))
    return {k: (o, p, np.unique(np.concatenate(v))) for k, (o, p, v) in acc.items()}


def tiles(n):
    return (n + 127) // 128


def touched_ranges(d, x3, epi):
    """[(buffer, part, lo, hi)]: every read and write of d lies in floats (or ints) [lo, hi) of the buffer.  The K-major loader
    fetches whole tiles (row tiles of M or N, column block per chunk); the MN-major loader 32-row pieces of the four column
    blocks of a 128-wide tile that lie below kb."""
    out = []

    def operand(o, n_rows):
        im, KC = o.img, d.KC
        starts = []
        if not im.mn:
            for c in range(KC):
                if o.k_rows is not None:
                    rt0, cb = int(o.k_rows[2 * c]) // 128, int(o.k_rows[2 * c + 1])
                else:
                    rt0, cb = o.row0 // 128, o.col0 // 32 + c
                assert cb < im.kb, 'K-major chunk beyond the image width'
                for t in range(tiles(n_rows)):
                    starts.append(((rt0 + t) * im.kb + cb) * 4096)
            lo, hi = min(starts), max(starts) + 4096
        else:
            for c in range(KC):
                r0 = int(o.k_rows[c]) if o.k_rows is not None else o.row0 + 32 * c
                for t in range(tiles(n_rows)):
                    for j in range(4):
                        cb = o.col0 // 32 + 4 * t + j
                        if cb < im.kb:
                            starts.append(((r0 >> 7) * im.kb + cb) * 4096 + ((r0 & 127) >> 3) * 256)
            assert o.col0 // 32 + (n_rows + 31) // 32 <= im.kb, 'MN-major operand beyond the image width'
            lo, hi = min(starts), max(starts) + 1024
        out.append((im, 'hi', lo, hi))
        if x3:
            out.append((im, 'lo', lo, hi))
        if o.k_rows is not None:
            out.append((o.k_rows, None, 0, (2 if not im.mn else 1) * KC))
    operand(d.a, d.M)
    operand(d.b, d.N)
    if d.c is not None:
        out.append((d.c, None, 0, int(c_offsets(d).max()) + 1))
    if d.bias is not None:
        out.append((d.bias, None, 0, d.N))
    if epi == 2:
        assert d.o_col0 // 32 + ceil32(d.N) // 32 <= d.o_kb, 'output beyond the image width'
        for im, mn, parts in ((d.o_k, False, ('hi', 'lo')), (d.o_mn, True, ('hi', 'lo')), (d.mask, False, ('hi',))):
            if im is not None and (im is not d.mask or d.flags & MASK_IMG):
                off = out_offsets(d, mn)
                for p in parts:
                    out.append((im, p, int(off.min()), int(off.max()) + 1))
    return out


def size_of(obj, part):
    if isinstance(obj, Image):
        return (obj.hi if part == 'hi' else obj.lo).size
    return np.asarray(obj).size
