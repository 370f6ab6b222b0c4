"""Spread of the Marsaglia IC acceptance statistic (tests/test_model_gpu.py::test_marsaglia_inference_compilation) over seeds.

    python scripts/marsaglia_ess.py [--traces 600000] [--batch 256] [--lstm 128] [--seeds 5 6 7] [--draws 3] [--precision 0]

For every seed: one training run, then --draws independent posteriors of 8192 proposals; prints each draw's ESS, their
median (what the test holds against the reference floor 0.016 * 8192), the posterior means and the best training loss.
--precision selects the network arithmetic (0 = 3xTF32 tensor cores, 1 = TF32, 2 = exact-fp32 SIMT GEMMs)."""
import argparse
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))
import pyprob_b200 as pyprob  # noqa: E402
from pyprob_b200 import InferenceEngine, InferenceNetwork  # noqa: E402
from pyprob_b200 import network as pnet  # noqa: E402
from test_model_gpu import GaussianUnknownMeanMarsaglia  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--traces', type=int, default=600000)
ap.add_argument('--batch', type=int, default=256)
ap.add_argument('--lstm', type=int, default=128)
ap.add_argument('--seeds', type=int, nargs='+', default=[5, 6, 7])
ap.add_argument('--draws', type=int, default=3)
ap.add_argument('--precision', type=int, default=0, choices=[0, 1, 2])
args = ap.parse_args()

if args.precision:
    _init = pnet.InferenceNetworkLSTM.__init__

    def _init_with_precision(self, *a, **kw):
        kw['precision'] = args.precision
        _init(self, *a, **kw)
    pnet.InferenceNetworkLSTM.__init__ = _init_with_precision

pyprob.set_verbosity(0)
floor = 0.016 * 8192
print('budget %d traces, batch %d, h %d, precision %d, env %s' % (
    args.traces, args.batch, args.lstm, args.precision,
    ' '.join('%s=%s' % kv for kv in sorted(os.environ.items()) if kv[0].startswith('PPB_')) or '-'), flush=True)
for seed in args.seeds:
    pyprob.seed(seed)
    m = GaussianUnknownMeanMarsaglia()
    t0 = time.time()
    m.learn_inference_network(num_traces=args.traces, batch_size=args.batch, inference_network=InferenceNetwork.LSTM,
                              lstm_dim=args.lstm, observe_embeddings={'obs0': {'dim': 16}, 'obs1': {'dim': 16}})
    t1 = time.time()
    ess, means = [], []
    for _ in range(args.draws):
        post = m.posterior_results(8192, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                   observe={'obs0': 8, 'obs1': 9})
        ess.append(float(post.effective_sample_size))
        means.append(float(post.mean))
    med = sorted(ess)[len(ess) // 2]
    print('seed %d: train %.1f s, loss %.4f, ESS %s median %.1f (floor %.1f%s), means %s' % (
        seed, t1 - t0, m._inference_network._loss_min, ' / '.join('%.1f' % e for e in ess), med, floor,
        '' if med > floor else ' FAIL', ' / '.join('%.3f' % x for x in means)), flush=True)
