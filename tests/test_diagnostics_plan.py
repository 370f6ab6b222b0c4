"""CPU: the diagnostics kernels' workspace sizes (include/pyprob_b200.h section 8) stay bounded for the requests a user
makes: a per-iteration R-hat curve, every lag, many chains; and invalid arguments are refused without a GPU."""
import ctypes

import numpy as np

from pyprob_b200 import _lib

F32, F64 = 0, 1


def _rhat_bytes(S, C, V, iters):
    it = np.ascontiguousarray(np.asarray(iters, dtype=np.int64))
    return _lib.call('ppb_diag_rhat_workspace_bytes', S, C, V, it.ctypes.data_as(ctypes.c_void_p), len(it))


def test_rhat_workspace_does_not_grow_per_chain_with_the_iterations():
    S, C = 10000, 65536
    default = _rhat_bytes(S, C, 1, np.unique(np.logspace(0, np.log10(S)).astype(int)))
    every = _rhat_bytes(S, C, 1, np.arange(1, S + 1))
    # segment statistics: at most max(256 MiB, (2^17 + C V) x 16 B); partials: 32 B per (iteration, variable, 256 chains)
    assert default <= (256 << 20) + (4 << 20)
    assert every <= (2 ** 17 + C) * 16 + S * (C // 256) * 32 + (1 << 20)
    assert every < 100 << 20          # the values themselves are 2.6 GB at fp32


def test_autocorrelation_workspace_is_bounded():
    for S, C, V, n_lags in ((10000, 65536, 4, 40), (10007, 1000, 3, 10008), (10 ** 6, 4, 1, 50)):
        for dt in (F32, F64):
            b = _lib.call('ppb_diag_autocorr_workspace_bytes', dt, S, C, V, n_lags)
            assert 0 < b <= (1 << 30) + 64 * C * V + (8 << 20), (S, C, V, n_lags, b)


def test_invalid_arguments_are_refused():
    assert _rhat_bytes(10, 1, 1, [5]) == -1          # one chain
    assert _rhat_bytes(10, 4, 1, [0, 5]) == -1       # an iteration below 1
    assert _lib.call('ppb_diag_autocorr_workspace_bytes', 2, 10, 4, 1, 3) == -1     # dtype
    assert _lib.call('ppb_diag_autocorr_workspace_bytes', F32, 10, 4, 1, 0) == -1   # no lags
