"""One launch of every scoring / sampling / normalisation kernel at 2^24 particles (per-particle parameters, every operand
array 64 MiB: far beyond the 50 MB L2 together) — the target of the `ncu --set full` capture whose dram__bytes and
throughput numbers go to profiles/ (scripts/summarise_ncu.py).  Warm-up launches first; ncu is told to skip them."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pyprob_b200 import ops  # noqa: E402

dev = torch.device('cuda:0')
n, K, C = 1 << 24, 10, 8
g = torch.Generator(device=dev).manual_seed(0)
v = torch.randn(n, device=dev, generator=g)
mu = torch.randn(n, device=dev, generator=g)
sd = torch.rand(n, device=dev, generator=g) + 0.5
lo, hi = mu - 2.0, mu + 2.0
rate = sd * 4
cnt = torch.poisson(rate, generator=g)
probs = torch.rand(n, C, device=dev, generator=g) + 0.01
cat = torch.randint(0, C, (n,), device=dev, generator=g).float()
m = torch.randn(n, K, device=dev, generator=g)
s = torch.rand(n, K, device=dev, generator=g) + 0.1
p = torch.rand(n, K, device=dev, generator=g) + 0.01
lw = torch.randn(n, device=dev, generator=g) * 5 - 40
out = torch.empty(n, device=dev)
cases = [
    lambda: ops.normal_log_prob(v, mu, sd, lp_out=out),
    lambda: ops.uniform_log_prob(v, lo, hi, lp_out=out),
    lambda: ops.poisson_log_prob(cnt, rate, lp_out=out),
    lambda: ops.categorical_log_prob(cat, probs, lp_out=out),
    lambda: ops.mixture_normal_log_prob(v, m, s, p, lp_out=out),
    lambda: ops.mixture_truncated_normal_log_prob(v, m, s, p, lo, hi, lp_out=out),
    lambda: ops.normal_sample(mu, sd, n, 1, 2),
    lambda: ops.weights_finalize(lw),
]
for rep in range(2):      # first pass = warm-up
    for fn in cases:
        fn()
    torch.cuda.synchronize()
print('done')
