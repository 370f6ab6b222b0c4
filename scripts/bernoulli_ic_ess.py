"""Spread of the Bernoulli-switch inference-compilation acceptance test (tests/test_bernoulli_gpu.py) over seeds.

    python scripts/bernoulli_ic_ess.py --traces 40000 --seeds 1 2 3 4 5 --draws 3

Prints, for every seed, the final training loss and, for every posterior draw, P(z = 1 | x) and the ESS fraction."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pyprob_b200 as pyprob  # noqa: E402
from pyprob_b200 import InferenceEngine, InferenceNetwork  # noqa: E402
from tests.test_bernoulli_gpu import X_OBS, BinarySwitch, _closed_form  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--traces', type=int, default=40000)
    ap.add_argument('--seeds', type=int, nargs='+', default=[1, 2, 3, 4, 5])
    ap.add_argument('--draws', type=int, default=3)
    ap.add_argument('--n', type=int, default=8192)
    a = ap.parse_args()
    print('closed form P(z = 1 | x) = {:.4f}'.format(_closed_form()))
    for seed in a.seeds:
        pyprob.seed(seed)
        pyprob.set_verbosity(0)
        model = BinarySwitch()
        model.learn_inference_network(num_traces=a.traces, batch_size=256, inference_network=InferenceNetwork.LSTM,
                                      lstm_dim=64, observe_embeddings={'x': {'dim': 16}})
        net = model._inference_network
        rows = []
        for _ in range(a.draws):
            post = model.posterior_results(a.n, InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK,
                                           observe={'x': X_OBS})
            rows.append('{:.4f}/{:.3f}'.format(float(post.mean), float(post.effective_sample_size) / a.n))
        print('seed {} loss init {:.4f} final {:.4f} | mean/ESS fraction: {}'.format(
            seed, net._loss_init, net._history_train_loss[-1], ' '.join(rows)), flush=True)


if __name__ == '__main__':
    main()
