"""The tf32 tile-image layout helpers of tc.cuh (img_span, k_swz, mn_swz, packed_offset, packed_offset_mn), evaluated on
the host by a small program built with nvcc, against the layout as DESIGN.md states it: tile (rt, cb) at float
(rt * KB + cb) * 4096, row r of a tile at r * 32, the 16-byte chunk c16 of a K-format row at c16 ^ (r & 7), the 32-byte
chunk c32 of an MN-format row at c32 ^ (r & 3)."""
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, 'pyprob_b200', 'csrc')
NVCC = os.environ.get('NVCC') or shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
ROWS, COLS = 384, 96

PROGRAM = r'''
#include <stdio.h>
#include "tc.cuh"
int main() {
  const int64_t kbs[2] = {1, 3};
  for (int64_t KB : kbs)
    for (int64_t row = 0; row < %(rows)d; ++row)
      for (int64_t k = 0; k < 32 * KB; ++k)
        printf("%%lld %%lld %%lld %%lld %%lld\n", (long long)tc::packed_offset(row, k, KB),
               (long long)tc::packed_offset_mn(row, k, KB), (long long)tc::img_span(row, k >> 5, KB),
               (long long)tc::k_swz(row, (int)(k & 31)), (long long)tc::mn_swz(row, (int)(k & 31)));
  return 0;
}
''' % {'rows': ROWS}


@pytest.fixture(scope='module')
def helpers(tmp_path_factory):
    if not os.path.exists(NVCC):
        pytest.skip('nvcc not available')
    d = tmp_path_factory.mktemp('tile_layout')
    src, exe = d / 'layout.cu', d / 'layout'
    src.write_text(PROGRAM)
    subprocess.check_call([NVCC, '-gencode', 'arch=compute_90a,code=sm_90a', '-std=c++17', '-I', CSRC, '-o', str(exe),
                           str(src)])
    out = np.array(subprocess.check_output([str(exe)]).split(), dtype=np.int64).reshape(-1, 5)
    res, at = {}, 0
    for KB in (1, 3):
        n = ROWS * 32 * KB
        res[KB] = out[at:at + n].reshape(ROWS, 32 * KB, 5)
        at += n
    assert at == len(out)
    return res


def layout(KB):
    """(K-format offset, MN-format offset, span, position in a K span, position in an MN span) of every (row, col)"""
    row, col = np.meshgrid(np.arange(ROWS), np.arange(32 * KB), indexing='ij')
    rt, r, cb, c = row // 128, row % 128, col // 32, col % 32
    span = (rt * KB + cb) * 4096 + r * 32
    pos_k = ((c // 4) ^ (r % 8)) * 4 + c % 4
    pos_mn = ((c // 8) ^ (r % 4)) * 8 + c % 8
    return span + pos_k, span + pos_mn, span, pos_k, pos_mn


@pytest.mark.parametrize('KB', [1, 3])
def test_helpers_match_the_documented_layout(helpers, KB):
    got = helpers[KB]
    for i, want in enumerate(layout(KB)):
        np.testing.assert_array_equal(got[..., i], want)


@pytest.mark.parametrize('KB', [1, 3])
@pytest.mark.parametrize('flavour', [0, 1], ids=['k', 'mn'])
def test_each_flavour_is_a_bijection_onto_each_tile(helpers, KB, flavour):
    off = helpers[KB][..., flavour]
    for rt in range(ROWS // 128):
        for cb in range(KB):
            tile = off[rt * 128:(rt + 1) * 128, cb * 32:(cb + 1) * 32].ravel()
            base = (rt * KB + cb) * 4096
            np.testing.assert_array_equal(np.sort(tile), base + np.arange(4096))
