"""Device-event timings of the Poisson, Uniform and truncated-Normal-mixture samplers (with lp_out), the samplers the
importance-sampling proposals draw from.

    python scripts/bench_samplers.py [--log2n 24] [--iters 20] [--json out.json]

Poisson at rates 4 (inversion), 37 and 1e5 (PTRS: the double-precision acceptance test runs only on draws that miss
the squeeze), Uniform(1000, 1001), and the K = 10 truncated mixture on the Poisson proposal window [0, 40] with shared
rows.  Every launch draws a new offset.  Reports the mean time per launch over --iters launches after warm-up, and the
GPU name and power limit read in the same run.  Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench_families import gpu_info, time_ms  # noqa: E402
from pyprob_b200 import ops  # noqa: E402


def cases():
    k = torch.arange(10, dtype=torch.float32)
    means, stddevs, probs = (-2 + 47 * k / 9).cuda(), (2 + k / 3).cuda(), (1 + (k * 5) % 7).cuda()
    out = [('poisson rate {:g}'.format(r), lambda n, o, r=r: ops.poisson_sample(r, n, 1, o, with_log_prob=True))
           for r in (4.0, 37.0, 1e5)]
    out.append(('uniform (1000, 1001)', lambda n, o: ops.uniform_sample(1000.0, 1001.0, n, 1, o, with_log_prob=True)))
    out.append(('truncated mixture K=10 [0, 40]',
                lambda n, o: ops.mixture_truncated_normal_sample(means, stddevs, probs, 0.0, 40.0, n, 1, o,
                                                                 with_log_prob=True)))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--log2n', type=int, default=24)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_samplers.py needs a CUDA device')
    info = gpu_info()
    print('# {} power limit {}'.format(info['name'], info.get('power_limit')))
    n = 1 << args.log2n
    rows = []
    for name, draw in cases():
        offset = [0]

        def fn():
            offset[0] += 1
            draw(n, offset[0])
        ms = time_ms(fn, args.iters)
        rows.append({'sampler': name, 'n': n, 'ms': ms, 'Gdraws_per_s': n / ms / 1e6})
        print('{:32s} n=2^{:<2d} {:8.4f} ms  {:6.2f} Gdraws/s'.format(name, args.log2n, ms, n / ms / 1e6))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump({'gpu': info, 'iters': args.iters, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
