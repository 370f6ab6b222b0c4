"""Reference traces -> TraceColumns.from_reference_traces -> trace file -> OfflineDataset.batch must describe the same
minibatch as the reference's own Batch: the oracle loss on the re-read arrays equals the UNMODIFIED reference's _loss on the
traces.  The traces, the network parameters, the reference's grouping and its loss are stored in tests/golden/bridge_golden.npz
(tests/golden/make_bridge_golden.py); the traces are rebuilt here as duck-typed objects with the attributes the bridge reads."""
import json
import os
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _distribution(v):
    fam = v['family']
    if fam == 'Categorical':
        d = SimpleNamespace(num_categories=v['num_categories'])
    elif fam == 'Normal':
        d = SimpleNamespace(mean=v['mean'], stddev=v['stddev'])
    elif fam == 'Uniform':
        d = SimpleNamespace(low=v['low'], high=v['high'])
    else:
        d = SimpleNamespace()
    return type(fam, (), dict(vars(d)))()


def _trace(rec):
    ctrl = [SimpleNamespace(address=v['address'], value=np.float32(v['value']), distribution=_distribution(v))
            for v in rec['variables']]
    named = {nm: SimpleNamespace(value=np.asarray(val, np.float32)) for nm, val in rec['observed'].items()}
    return SimpleNamespace(variables_controlled=ctrl, named_variables=named)


def test_reference_traces_survive_the_columnar_store(tmp_path):
    from oracle import network as onet
    from pyprob_b200 import offline

    g = np.load(os.path.join(ROOT, 'tests', 'golden', 'bridge_golden.npz'))
    meta = json.loads(bytes(g['meta']).decode())
    traces = [_trace(t) for t in meta['traces']]
    names = meta['observe_names']
    cols = offline.TraceColumns.from_reference_traces(traces, names)
    offline.save_columns(str(tmp_path), cols)
    data = offline.OfflineDataset(str(tmp_path))
    assert len(data) == 40 and data.num_trace_types == len(meta['sub_batch_sizes'])
    arr = data.batch(list(range(40)))
    # same grouping as the reference Batch: sub-batches in order of first appearance, same sizes
    assert [sb['values'].shape[1] for sb in arr.subs] == meta['sub_batch_sizes']
    assert [sb['addresses'] for sb in arr.subs] == meta['sub_batch_addresses']
    params = {k[len('param/'):]: torch.from_numpy(g[k]) for k in g.files if k.startswith('param/')}
    tsubs = [{k: (torch.from_numpy(np.ascontiguousarray(v)) if isinstance(v, np.ndarray) else v) for k, v in sb.items()}
             for sb in arr.subs]
    got, _ = onet.loss(params, tsubs, names, [1, 1], 3)
    ref_loss = meta['ref_loss']
    assert abs(float(got) - ref_loss) <= 2e-6 * abs(ref_loss)
