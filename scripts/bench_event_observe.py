"""Device-event timings of the event-shaped observation path.

    python scripts/bench_event_observe.py [--iters 50] [--json out.json]

1. The event log_prob kernel (acc only) at n D = 2^24 and 2^26 for D in {8, 100, 784}, for Normal, Poisson, Bernoulli and
   Gamma, with the first parameter one event per particle ([n, D]), the others scalars, and one shared value row.
   Algorithmic bytes: 4 B per element of the per-particle parameter, the shared row once (4 D B) and the fp64 accumulator
   read and written (16 B per particle); GB/s and the share of the H100 SXM's 3.35 TB/s follow from them.
2. IS posterior particles/s of a Bayesian linear regression (w, b ~ Normal(0, 1); y_j ~ Normal(w x_j + b, 0.5)) at
   n = 65,536 and D = 100 and 1,000: one vector observe against D scalar observes of the same data.
The GPU name and power limit are read in the same run.  Needs a CUDA device; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyprob_b200 as pyprob  # noqa: E402
from pyprob_b200 import Model, ops  # noqa: E402
from pyprob_b200.distributions import Normal  # noqa: E402
from pyprob_b200.util import TraceMode  # noqa: E402

HBM_BYTES_PER_S = 3.35e12

# family -> (per-particle first parameter [n, D], the other parameters as scalars, a shared value row [1, D])
FAMILIES = {
    'Normal': (lambda n, D: torch.randn(n, D, device='cuda'), [1.3], lambda D: torch.randn(1, D, device='cuda')),
    'Poisson': (lambda n, D: torch.rand(n, D, device='cuda') * 20 + 0.1, [],
                lambda D: torch.randint(0, 30, (1, D), device='cuda').float()),
    'Bernoulli': (lambda n, D: torch.rand(n, D, device='cuda'), [],
                  lambda D: (torch.rand(1, D, device='cuda') < 0.5).float()),
    'Gamma': (lambda n, D: torch.rand(n, D, device='cuda') * 4 + 0.5, [1.5],
              lambda D: torch.rand(1, D, device='cuda') * 3 + 0.01),
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
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


class RegressionVector(Model):
    def __init__(self, x):
        super().__init__()
        self.x = x

    def forward(self):
        w = pyprob.sample(Normal(0.0, 1.0), name='w')
        b = pyprob.sample(Normal(0.0, 1.0), name='b')
        pyprob.observe(Normal(w.view(-1, 1) * self.x.view(1, -1) + b.view(-1, 1), 0.5), name='y')
        return w


class RegressionScalars(Model):
    def __init__(self, x):
        super().__init__()
        self.x = x.tolist()

    def forward(self):
        w = pyprob.sample(Normal(0.0, 1.0), name='w')
        b = pyprob.sample(Normal(0.0, 1.0), name='b')
        for j, xj in enumerate(self.x):
            pyprob.observe(Normal(w * xj + b, 0.5), name='y{}'.format(j))
        return w


def regression_rate(model, n, observe, reps):
    def run():
        model._run_batched(n, trace_mode=TraceMode.POSTERIOR, observe=observe)
    run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        run()
    torch.cuda.synchronize()
    return n * reps / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    info = gpu_info()
    print('# {} power limit {}'.format(info['name'], info.get('power_limit')))
    rows = []
    for total_log2 in (24, 26):
        for D in (8, 100, 784):
            n = (1 << total_log2) // D
            for fam, (per_particle, scalars, value) in FAMILIES.items():
                fid = ops.EVENT_FAMILIES[fam]
                params = [per_particle(n, D)] + scalars
                v = value(D)
                acc = torch.zeros(n, dtype=torch.float64, device='cuda')
                ms = time_ms(lambda: ops.event_log_prob(fid, v, params, n, D, acc=acc), args.iters)
                nbytes = 4 * n * D + 4 * D + 16 * n
                gbs = nbytes / (ms * 1e-3) / 1e9
                row = {'kernel': 'event_log_prob', 'family': fam, 'n': n, 'D': D, 'elements': n * D, 'ms': ms,
                       'GB/s': gbs, 'hbm_share': gbs * 1e9 / HBM_BYTES_PER_S}
                rows.append(row)
                print('event_log_prob {:9s} nD=2^{} D={:4d} n={:8d}  {:8.4f} ms  {:7.1f} GB/s  {:5.1%} of HBM'.format(
                    fam, total_log2, D, n, ms, gbs, row['hbm_share']))
    pyprob.set_verbosity(0)
    n = 65536
    for D in (100, 1000):
        x = torch.linspace(-1, 1, D, device='cuda')
        y = 0.7 * x - 0.2 + 0.5 * torch.randn(D, device='cuda')
        vec = regression_rate(RegressionVector(x), n, {'y': y}, reps=20)
        sca = regression_rate(RegressionScalars(x), n, {'y{}'.format(j): float(y[j]) for j in range(D)}, reps=3)
        rows.append({'kernel': 'is_regression', 'n': n, 'D': D, 'vector_particles_per_s': vec,
                     'scalar_particles_per_s': sca})
        print('IS regression n={} D={:5d}: one vector observe {:.3e} particles/s, {} scalar observes {:.3e} '
              'particles/s ({:.1f}x)'.format(n, D, vec, D, sca, vec / sca))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump({'gpu': info, 'rows': rows}, f, indent=1)


if __name__ == '__main__':
    main()
