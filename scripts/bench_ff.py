"""Feed-forward against LSTM inference network on the GPU: one JSON line.

  train : ms per training step (forward, backward, Adam) and traces/s of the GUM network (B = 256, T = 1, observe embeddings
          32 + 32, LSTM h = 512) and the synthetic50 network (B = 512, T = 50, E = 256, LSTM h = 512): the step replayed from
          the CUDA graph of ppb_ic_train_step_host, timed with device events, L2 flushed between steps (as in bench.py)
  launches_per_t1_step : kernel launches of one eager GUM step (forward + backward + Adam)
  ic_posterior : IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK particles/s on GUM at 64 k particles (bench.py's timing)
The two network types alternate within one run; --repeats runs the whole comparison that many times.

    python scripts/bench_ff.py [--steps 200] [--warmup 20] [--repeats 3]
"""
import argparse
import contextlib
import ctypes as C
import io
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pyprob_b200 import InferenceEngine, InferenceNetwork, _lib, synthetic  # noqa: E402
from pyprob_b200._lib import call, ptr  # noqa: E402

KINDS = (('feedforward', InferenceNetwork.FEEDFORWARD), ('lstm', InferenceNetwork.LSTM))


class _Step:
    """One network + batch, stepped through ppb_ic_train_step_host."""

    def __init__(self, net, batch):
        net._sync_native()
        self.net, self.enc = net, batch.encode(net)
        self.img = self.enc.pack().copy()
        self.dimg = torch.empty(self.img.nbytes, dtype=torch.uint8, device='cuda')
        need = net._ensure_workspace(self.enc)
        self.ws = torch.empty(need + 1024, dtype=torch.uint8, device='cuda')
        self.grad = torch.zeros_like(net._arena.data)
        self.m, self.v = torch.zeros_like(self.grad), torch.zeros_like(self.grad)
        self.loss, self.status, self.step = C.c_float(), C.c_int32(), 0

    def __call__(self):
        self.step += 1
        n = self.net
        call('ppb_ic_train_step_host', n._handle, ptr(n._arena.data), ptr(self.grad), ptr(self.m), ptr(self.v),
             n._arena.numel(), self.img.ctypes.data, self.img.nbytes, ptr(self.dimg), ptr(self.ws), self.ws.numel(), 0,
             1e-4, 0.9, 0.999, 1e-8, 0.0, self.step, C.byref(self.loss), C.byref(self.status),
             torch.cuda.current_stream().cuda_stream)


def _time(step, steps, warmup, flush):
    for _ in range(warmup):
        step()
    ms = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(steps):
        flush.zero_()
        e0.record()
        step()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def _launches(net, batch):
    os.environ['PPB_HOST_STEP_GRAPH'] = '0'   # read when the handle is created: plain stream launches
    net._handle = None
    st = _Step(net, batch)
    st()
    torch.cuda.synchronize()
    l0 = _lib.call('ppb_launch_count')
    st()
    torch.cuda.synchronize()
    del os.environ['PPB_HOST_STEP_GRAPH']
    return int(_lib.call('ppb_launch_count') - l0)


def _posterior(kind):
    import pyprob_b200 as pyprob
    pyprob.seed(2)
    pyprob.set_verbosity(0)
    m = bench._gum_model()
    with contextlib.redirect_stdout(io.StringIO()):
        m.learn_inference_network(num_traces=10 * 256, batch_size=256, inference_network=kind, lstm_dim=512,
                                  observe_embeddings={'obs0': {'dim': 32}, 'obs1': {'dim': 32}})
    value, ess, _ = bench._time_posterior(m, 65536, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK, 20)
    return value


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ff.py needs a CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device='cuda')
    rng = np.random.default_rng(0)
    shapes = {'gum_b256': (lambda k: synthetic.gum_network(lstm_dim=512, seed=0, inference_network=k),
                           synthetic.gum_batch(rng, 256), 256),
              'synthetic50_b512': (lambda k: synthetic.synthetic50_network(lstm_dim=512, seed=0, inference_network=k),
                                   synthetic.synthetic50_batch(rng, 512), 512)}
    steps = {(s, name): _Step(make(kind), batch) for s, (make, batch, _) in shapes.items() for name, kind in KINDS}
    runs = []
    for _ in range(a.repeats):
        r = {}
        for s, (_, _, B) in shapes.items():
            for name, _ in KINDS:    # the two network types alternate
                ms = _time(steps[(s, name)], a.steps, a.warmup, flush)
                r['{}_{}_ms'.format(s, name)] = ms
                r['{}_{}_traces_per_s'.format(s, name)] = B / (ms * 1e-3)
        for name, kind in KINDS:
            r['ic_posterior_gum_64k_{}_particles_per_s'.format(name)] = _posterior(kind)
        runs.append(r)
    launches = {name: _launches(synthetic.gum_network(lstm_dim=512, seed=0, inference_network=kind),
                                synthetic.gum_batch(np.random.default_rng(1), 256)) for name, kind in KINDS}
    print(json.dumps({'gpu': q, 'runs': runs, 'launches_per_t1_step': launches, 'steps': a.steps, 'warmup': a.warmup}))


if __name__ == '__main__':
    main()
