"""A/B timing of the opt-in kernels against the defaults, each arm in its own process (the switches are read once per
process):
  PPB_MIXTURE_STAGED=1 mixture-of-Normals / mixture-of-TruncatedNormals log_prob at 2^24 particles, K=10
Prints one JSON object.  Timings only — correctness is the job of tests/test_scoring_staged_gpu.py."""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_MIX = r'''
import sys, json, torch
sys.path.insert(0, %r)
from pyprob_b200 import ops
n, K = 1 << 24, 10
g = torch.Generator(device='cuda').manual_seed(0)
means = torch.randn(n, K, device='cuda', generator=g); sd = torch.rand(n, K, device='cuda', generator=g) + 0.2
probs = torch.rand(n, K, device='cuda', generator=g); v = torch.randn(n, device='cuda', generator=g)
lo, hi = v - 1.0, v + 1.0
lp = torch.empty(n, device='cuda')
out = {}
for name, fn in (('mixture_normal', lambda: ops.mixture_normal_log_prob(v, means, sd, probs, lp_out=lp)),
                 ('mixture_truncated_normal', lambda: ops.mixture_truncated_normal_log_prob(v, means, sd, probs, lo, hi, lp_out=lp))):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): fn()
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 10
    bytes_per = (3 * K + (2 if name == 'mixture_normal' else 4)) * 4
    out[name] = {'ms': ms, 'gbs': n * bytes_per / (ms * 1e-3) / 1e9, 'checksum': float(lp.double().sum())}
print(json.dumps(out))
''' % ROOT


def run(script, env_extra):
    env = dict(os.environ)
    env.pop('PPB_MIXTURE_STAGED', None)
    env.update(env_extra)
    r = subprocess.run([sys.executable, '-c', script], env=env, capture_output=True, text=True, timeout=180)
    if r.returncode != 0:
        return {'error': r.stderr.strip().splitlines()[-1] if r.stderr.strip() else 'failed'}
    return json.loads(r.stdout.strip().splitlines()[-1])


if __name__ == '__main__':
    res = {'mixture_scoring': {'default': run(_MIX, {}), 'staged': run(_MIX, {'PPB_MIXTURE_STAGED': '1'})}}
    print(json.dumps(res, indent=1))
