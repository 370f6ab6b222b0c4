"""GPU: ppb_pack_tf32 / ppb_pack_tf32_mn on ragged shapes (rows not a multiple of 128, K not a multiple of 32) against
the tile-image layout as DESIGN.md states it: every element where the layout puts it, hi + lo = x to tf32-split
accuracy, and every padding position of the image zero."""
import numpy as np
import pytest
import torch

from pyprob_b200 import _lib
from pyprob_b200._lib import call, ptr, stream

pytestmark = pytest.mark.gpu


def _layout(rows, K, mn):
    KB = (K + 31) // 32
    row, col = np.meshgrid(np.arange(rows), np.arange(K), indexing='ij')
    r, c = row % 128, col % 32
    span = ((row // 128) * KB + col // 32) * 4096 + r * 32
    if mn:
        return span + ((c // 8) ^ (r % 4)) * 8 + c % 8
    return span + ((c // 4) ^ (r % 8)) * 4 + c % 4


@pytest.mark.parametrize('mn', [False, True], ids=['k', 'mn'])
@pytest.mark.parametrize('rows,K', [(1, 1), (77, 45), (200, 77), (129, 33), (300, 100)])
def test_pack_places_every_element_and_zero_fills_the_padding(cuda, rows, K, mn):
    torch.manual_seed(rows * 1000 + K)
    x = torch.randn(rows, K + 3, device=cuda)[:, :K]   # ldx > K
    nfl = _lib.call('ppb_packed_floats', rows, K)
    assert nfl == -(-rows // 128) * -(-K // 32) * 4096
    hi = torch.full((nfl,), float('nan'), device=cuda)
    lo = torch.full((nfl,), float('nan'), device=cuda)
    call('ppb_pack_tf32_mn' if mn else 'ppb_pack_tf32', ptr(x), rows, K, x.stride(0), ptr(hi), ptr(lo), stream())
    torch.cuda.synchronize()
    idx = torch.as_tensor(_layout(rows, K, mn), device=cuda)
    h, l = hi[idx], lo[idx]
    # hi is x rounded to tf32 (low 13 mantissa bits zero), lo the rounded rest; hi + lo reproduces x to ~2^-21
    assert (h.view(torch.int32) & 0x1FFF).abs().sum().item() == 0
    assert (l.view(torch.int32) & 0x1FFF).abs().sum().item() == 0
    assert ((h + l - x).abs() <= x.abs() * 2.0 ** -20 + 1e-30).all()
    pad = torch.ones(nfl, dtype=torch.bool, device=cuda)
    pad[idx.ravel()] = False
    assert int(pad.sum()) == nfl - rows * K       # the layout is one-to-one
    assert (hi[pad] == 0).all() and (lo[pad] == 0).all()
