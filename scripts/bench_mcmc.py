"""Throughput of the lock-step Metropolis-Hastings chains (LMH) through Model.posterior.

    python scripts/bench_mcmc.py [--chains 1 1024 16384 65536] [--steps 200] [--warmup 20] [--json out.json]

For GUM (one Normal site, two observes), the lock-step Marsaglia model (a while_loop of Uniform pairs) and the lock-step
HMM of the reference's tests (17 Categorical sites, 16 observes), at every chain count: --steps MH steps of every chain,
each recorded (thinning 1), after a separate run of --warmup steps.  Reports chain-steps/s (chains x steps / wall time)
and recorded states/s.  Wall time runs from the call to the end of a device synchronisation, so it includes the host's
launch overhead, which dominates at small chain counts.  The GPU name and power limit are read (nvidia-smi
--query-gpu, read-only) in the same run.  Needs a CUDA device.
"""
import argparse
import json
import math
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pyprob_b200 as pyprob  # noqa: E402
from pyprob_b200 import InferenceEngine, Model, util  # noqa: E402
from pyprob_b200.distributions import Categorical, Normal, Uniform  # noqa: E402

HMM_OBS = [0.9, 0.8, 0.7, 0.0, -0.025, -5.0, -2.0, -0.1, 0.0, 0.13, 0.45, 6, 0.2, 0.3, -1, -1]


class GUM(Model):
    def forward(self):
        mu = pyprob.sample(Normal(1, math.sqrt(5)))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


class Marsaglia(Model):
    def forward(self):
        def body(s):
            x = pyprob.sample(Uniform(-1, 1))
            y = pyprob.sample(Uniform(-1, 1))
            return {'x': x, 'y': y, 's': x * x + y * y}
        st = pyprob.while_loop(lambda s: s['s'] >= 1, body, {'x': 0.0, 'y': 0.0, 's': 2.0})
        mu = 1 + math.sqrt(5) * (st['x'] * torch.sqrt(-2 * torch.log(st['s']) / st['s']))
        likelihood = Normal(mu, math.sqrt(2))
        pyprob.observe(likelihood, name='obs0')
        pyprob.observe(likelihood, name='obs1')
        return mu


class HMM(Model):
    def __init__(self):
        super().__init__('HMM')
        self.T = torch.tensor([[0.1, 0.5, 0.4], [0.2, 0.2, 0.6], [0.15, 0.15, 0.7]], device='cuda')
        self.means = torch.tensor([-1.0, 1.0, 0.0], device='cuda')

    def forward(self):
        states = [pyprob.sample(Categorical([1, 1, 1]))]
        for i in range(len(HMM_OBS)):
            s = pyprob.sample(Categorical(self.T[states[-1].long()]))
            pyprob.observe(Normal(self.means[s.long()], 1.0), name='obs{}'.format(i))
            states.append(s)
        return torch.stack(states, dim=1)


MODELS = {'gum': (GUM, {'obs0': 8, 'obs1': 9}), 'marsaglia': (Marsaglia, {'obs0': 8, 'obs1': 9}),
          'hmm': (HMM, {'obs{}'.format(i): v for i, v in enumerate(HMM_OBS)})}


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in q.split(',')]
        return {'gpu': name, 'power_limit': power}
    except Exception as e:     # noqa: BLE001 - report what could not be read, keep measuring
        return {'gpu': torch.cuda.get_device_name(), 'power_limit': 'unknown ({})'.format(type(e).__name__)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--chains', type=int, nargs='+', default=[1, 1024, 16384, 65536])
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--models', nargs='+', default=list(MODELS))
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    info = gpu_info()
    print(json.dumps(info))
    rows = []
    for name in args.models:
        make, observe = MODELS[name]
        for C in args.chains:
            model = make()
            util.seed(1)
            model.posterior(args.warmup, inference_engine=InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS,
                            observe=observe, num_chains=C)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            post = model.posterior(args.steps, inference_engine=InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS,
                                   observe=observe, num_chains=C)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            row = dict(info, model=name, chains=C, steps=args.steps, seconds=round(dt, 4),
                       chain_steps_per_s=round(C * args.steps / dt, 1), states_per_s=round(len(post) / dt, 1),
                       name=post.name)
            rows.append(row)
            print(json.dumps(row))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(rows, f, indent=1)


if __name__ == '__main__':
    main()
