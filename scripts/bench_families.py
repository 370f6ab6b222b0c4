"""Device-event timings of the Exponential .. VonMises log_prob kernels and samplers, with Normal's as the point of
comparison.

    python scripts/bench_families.py [--sizes 20 24] [--iters 50] [--json out.json]

For every family and n = 2^k particles: the log_prob kernel with shared (stride-0) and per-particle parameters, and the
sampler (with lp_out).  Reports the mean time per launch over --iters launches after warm-up, the achieved bytes/s
(algorithmic bytes per particle: value + lp_out, 4 B each, + 4 B per per-particle parameter; a sampler writes value and
lp_out and reads its parameters) against the H100 SXM's 3.35 TB/s, and draws/s for samplers.  The GPU name and power
limit are read in the same run.  Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pyprob_b200 import ops  # noqa: E402

HBM_BYTES_PER_S = 3.35e12

# family -> (log_prob, sampler, per-particle parameter generator, shared parameters)
FAMILIES = {
    'normal': (ops.normal_log_prob, ops.normal_sample, lambda n: [torch.randn(n), torch.rand(n) + 0.5], [0.3, 1.2]),
    'exponential': (ops.exponential_log_prob, ops.exponential_sample, lambda n: [torch.rand(n) + 0.5], [1.5]),
    'gamma': (ops.gamma_log_prob, ops.gamma_sample, lambda n: [torch.rand(n) * 5 + 0.1, torch.rand(n) + 0.5],
              [2.7, 1.2]),
    'lognormal': (ops.lognormal_log_prob, ops.lognormal_sample, lambda n: [torch.randn(n), torch.rand(n) + 0.5],
                  [0.5, 0.8]),
    'weibull': (ops.weibull_log_prob, ops.weibull_sample, lambda n: [torch.rand(n) + 0.5, torch.rand(n) * 3 + 0.5],
                [1.1, 1.5]),
    'beta': (ops.beta_log_prob, ops.beta_sample,
             lambda n: [torch.rand(n) * 5 + 0.1, torch.rand(n) * 5 + 0.1, torch.zeros(n), torch.ones(n)],
             [2.0, 5.0, 0.0, 1.0]),
    'binomial': (ops.binomial_log_prob, ops.binomial_sample,
                 lambda n: [torch.randint(1, 100, (n,)).float(), torch.rand(n)], [40.0, 0.3]),
    'von_mises': (ops.von_mises_log_prob, ops.von_mises_sample, lambda n: [torch.randn(n), torch.rand(n) * 10 + 0.1],
                  [0.5, 2.0]),
}


def gpu_info():
    info = {'name': torch.cuda.get_device_name(0)}
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm', '--format=csv,noheader'],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info['power_limit'], info['max_sm_clock'] = [s.strip() for s in out.split(',')]
    except Exception as e:       # the timings stand without it, but say why it is missing
        info['power_limit'] = 'unavailable ({})'.format(type(e).__name__)
    return info


def time_ms(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    start.record()
    for _ in range(iters):
        fn()
    stop.record()
    torch.cuda.synchronize()
    return start.elapsed_time(stop) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--sizes', type=int, nargs='+', default=[20, 24], help='log2 of the particle counts')
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_families.py needs a CUDA device')
    torch.manual_seed(0)
    info = gpu_info()
    print('# {} power limit {}'.format(info['name'], info.get('power_limit')))
    rows = []
    for k in args.sizes:
        n = 1 << k
        for fam, (score, draw, per_particle, shared) in FAMILIES.items():
            params = [p.cuda() for p in per_particle(n)]
            value, _ = draw(*shared, n, 1, 0, with_log_prob=True)
            lp = torch.empty(n, device='cuda')
            cases = [('log_prob shared', lambda: score(value, *shared, lp_out=lp), 8),
                     ('log_prob per-particle', lambda: score(value, *params, lp_out=lp), 8 + 4 * len(params))]
            offset = [0]

            def sample(ps):
                offset[0] += 1
                return draw(*ps, n, 1, offset[0], with_log_prob=True)
            cases += [('sample shared', lambda: sample(shared), 8),
                      ('sample per-particle', lambda: sample(params), 8 + 4 * len(params))]
            for what, fn, bytes_per in cases:
                ms = time_ms(fn, args.iters)
                row = {'family': fam, 'kernel': what, 'n': n, 'ms': ms, 'bytes_per_particle': bytes_per,
                       'GB_per_s': bytes_per * n / ms / 1e6, 'hbm_fraction': bytes_per * n / (ms * 1e-3) / HBM_BYTES_PER_S}
                if what.startswith('sample'):
                    row['Gdraws_per_s'] = n / ms / 1e6
                rows.append(row)
                print('{:12s} {:22s} n=2^{:<2d} {:8.4f} ms  {:7.1f} GB/s  {:5.1%} of 3.35 TB/s{}'.format(
                    fam, what, k, ms, row['GB_per_s'], row['hbm_fraction'],
                    '  {:6.2f} Gdraws/s'.format(row['Gdraws_per_s']) if 'Gdraws_per_s' in row else ''))
    out = {'gpu': info, 'iters': args.iters, 'rows': rows}
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
