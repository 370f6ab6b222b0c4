"""Time pyprob_b200.diagnostics.gelman_rubin and autocorrelation at their default iters / lags (CUDA events after
warm-up), with the achieved HBM rate of R-hat (it reads C * S * V values once) against 3.35 TB/s and the fp64 rate of
the autocorrelation (2 * C * V * sum over lags of (S - lag) FLOPs) beside the data-sheet fp64 figure, which is not
claimed as reached; and the numpy oracle on the host at a size it finishes in well under a minute.

    python scripts/bench_diagnostics.py [--reps 10]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import diagnostics as odiag  # noqa: E402
from pyprob_b200 import diagnostics  # noqa: E402
from pyprob_b200.empirical import Empirical  # noqa: E402

HBM_BYTES_S = 3.35e12
FP64_FLOPS = 67e12      # H100 SXM data sheet, fp64 tensor core; 34 TFLOP/s without


def _card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception as e:   # noqa: BLE001
        return '{} (power limit not read: {})'.format(torch.cuda.get_device_name(0), e)


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    rows = []
    for C, S, V in ((65536, 1000, 1), (65536, 1000, 4), (65536, 10000, 1), (65536, 10000, 4), (4, 10 ** 6, 1)):
        x = torch.randn(S * C, V, device='cuda').squeeze(-1)
        post = Empirical(x, None)
        post.add_metadata(op='posterior', num_chains=C)
        lags = np.unique(np.logspace(0, np.log10(S / 2)).astype(int))
        ms_r = _time(lambda: diagnostics.gelman_rubin(post), args.reps)
        ms_a = _time(lambda: diagnostics.autocorrelation(post), args.reps)
        flops = 2.0 * C * V * float(np.sum(S - lags))
        rows.append(dict(C=C, S=S, V=V, rhat_ms=round(ms_r, 4),
                         rhat_hbm_share=round(C * S * V * 4 / (ms_r * 1e-3) / HBM_BYTES_S, 4),
                         acf_ms=round(ms_a, 4), acf_fp64_tflops=round(flops / (ms_a * 1e-3) / 1e12, 3),
                         # every product reads its partner value through L1 / L2: the rate of those reads
                         acf_partner_read_tb_s=round(flops / 2 * 4 / (ms_a * 1e-3) / 1e12, 3)))
        print(json.dumps(rows[-1]), flush=True)
        del post, x
    # the numpy oracle on the host (the reference's formulas, vectorised over chains)
    C, S = 1024, 1000
    xs = np.random.default_rng(0).standard_normal((C, S))
    t0 = time.perf_counter()
    odiag.r_hats(xs, np.unique(np.logspace(0, np.log10(S)).astype(int)))
    t1 = time.perf_counter()
    odiag.autocorrelation(xs, np.unique(np.logspace(0, np.log10(S / 2)).astype(int)))
    t2 = time.perf_counter()
    host = dict(C=C, S=S, V=1, oracle_rhat_ms=round((t1 - t0) * 1e3, 2), oracle_acf_ms=round((t2 - t1) * 1e3, 2))
    print(json.dumps(host))
    print(json.dumps({'card': _card(), 'fp64_datasheet_tflops': FP64_FLOPS / 1e12, 'rows': rows, 'host': host}))


if __name__ == '__main__':
    main()
