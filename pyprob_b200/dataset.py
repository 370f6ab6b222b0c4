"""Online training data: prior traces generated on the GPU in lock-step, grouped into sub-batches.

``TraceBatch`` is the batched counterpart of the reference's ``Batch`` (pyprob/nn/dataset.py:21-47) and
``OnlineDataset`` of its ``OnlineDataset`` (:50-62): every minibatch is one execution of the user's
``forward`` over ``batch_size`` particles in TraceMode.PRIOR_FOR_INFERENCE_NETWORK (observes are sampled).
"""
import numpy as np
import torch

from .distributions import Categorical, set_shard_first_index
from .encoding import EncodedBatch, SubBatch
from .util import PriorInflation, TraceMode


class TraceBatch:
    def __init__(self, trace):
        self.trace = trace
        self.size = trace.n
        self.groups = trace.sub_batches()  # [(controlled sites, particle index tensor or None)]
        sizes = [trace.n if idx is None else int(idx.numel()) for _, idx in self.groups]
        self.mean_length_controlled = sum(len(s) * b for (s, _), b in zip(self.groups, sizes)) / self.size
        self.num_sub_batches = len(self.groups)
        self._encoded = None

    def __len__(self):
        return self.size

    @property
    def sub_batches(self):
        return self.groups

    def address_signature(self):
        seen, out = set(), []
        for sites, _ in self.groups:
            for s in sites:
                if s.address not in seen:
                    seen.add(s.address)
                    d = s.distribution
                    out.append((s.address, d.name, d.num_categories if isinstance(d, Categorical) else 0))
        return out

    def encode(self, net):
        """-> EncodedBatch (index tensors + packed image), or None if an address is unknown to the network."""
        if self._encoded is not None:
            return self._encoded
        n = self.trace.n
        cols, plan = [], []

        def push(t):
            cols.append(t.reshape(n).float())
            return len(cols) - 1

        def param(p):
            return push(p if torch.is_tensor(p) else torch.full((n,), float(p), device='cuda'))
        # observables: D columns each (an event-shaped observable's [n, *E] value, flattened), in _observe_names order
        obs_mat = torch.cat([self.trace.named_variables[name].value.reshape(n, -1).float()
                             for name in net._observe_names], dim=1)
        for sites, idx in self.groups:
            ids, vc, p0c, p1c = [], [], [], []
            for s in sites:
                if s.address not in net._addresses:
                    print('Address unknown by inference network: {}'.format(s.address))
                    return None
                ids.append(net._addresses[s.address]['id'])
                vc.append(push(s.value))
                p0, p1 = s.distribution._prior_params()
                p0c.append(-1 if p0 is None else param(p0)); p1c.append(-1 if p1 is None else param(p1))
            plan.append((ids, vc, p0c, p1c, idx))
        ncols = len(cols)
        host = torch.cat([torch.stack(cols, dim=0), obs_mat.t()], dim=0).cpu().numpy()  # one device->host copy
        zeros = np.zeros(n, dtype=np.float32)
        subs = []
        for ids, vc, p0c, p1c, idx in plan:
            sel = slice(None) if idx is None else idx.cpu().numpy()

            def rows(cs):
                return np.stack([(zeros if c < 0 else host[c])[sel] for c in cs], axis=0)
            obs = np.ascontiguousarray(host[ncols:, sel].T)
            subs.append(SubBatch(ids, rows(vc), rows(p0c), rows(p1c), obs))
        self._encoded = EncodedBatch(subs, row_align=net.row_align)
        return self._encoded

    def to_sub_batches(self, observe_names):
        """Host copy of the minibatch as plain arrays, one dict per sub-batch (the form synthetic.ArrayBatch and
        offline.TraceColumns.from_sub_batches take): addresses/families/num_categories per step, values, prior0,
        prior1 [T, B] and obs [B, sum of observable sizes]."""
        n = self.trace.n
        obs = torch.cat([self.trace.named_variables[name].value.reshape(n, -1).float() for name in observe_names],
                        dim=1).cpu().numpy()

        def host(x):
            return (x.reshape(n).float().cpu().numpy() if torch.is_tensor(x) else np.full(n, float(x), np.float32))
        zeros = np.zeros(n, np.float32)
        subs = []
        for sites, idx in self.groups:
            sel = slice(None) if idx is None else idx.cpu().numpy()
            addresses, families, cats, vals, p0, p1 = [], [], [], [], [], []
            for s in sites:
                d = s.distribution
                addresses.append(s.address)
                families.append(d.name)
                cats.append(d.num_categories if isinstance(d, Categorical) else 0)
                vals.append(host(s.value)[sel])
                q0, q1 = d._prior_params()
                p0.append((zeros if q0 is None else host(q0))[sel])
                p1.append((zeros if q1 is None else host(q1))[sel])
            subs.append({'addresses': addresses, 'families': families, 'num_categories': cats,
                         'values': np.stack(vals, 0), 'prior0': np.stack(p0, 0), 'prior1': np.stack(p1, 0),
                         'obs': obs[sel]})
        return subs


def rank_first_index(batch_size):
    """Global Philox index of this rank's first trace within one distributed minibatch draw."""
    from . import parallel
    world, rank = parallel.world_info()
    return rank * int(batch_size) if world > 1 else 0


class OnlineDataset:
    def __init__(self, model, length=None, prior_inflation=PriorInflation.DISABLED):
        self._model = model
        self._length = int(1e6) if length is None else length
        self._prior_inflation = prior_inflation
        self._example = None

    def __len__(self):
        return self._length

    def next_batch(self, batch_size):
        """One minibatch of prior traces.  Under torch.distributed every rank draws a DISJOINT index range of the same
        Philox stream (rank r takes particles [r * batch_size, (r + 1) * batch_size) of this draw), so that the world's
        minibatches together are one global batch of world * batch_size independent traces — the reference's ranks draw
        independently because each process seeds its own torch generator (inference_network.py:296-333)."""
        first = rank_first_index(batch_size)
        set_shard_first_index(first)
        try:
            trace = self._model._run_batched(batch_size, trace_mode=TraceMode.PRIOR_FOR_INFERENCE_NETWORK,
                                             prior_inflation=self._prior_inflation)
        finally:
            set_shard_first_index(0)
        return TraceBatch(trace)

    def example_trace(self):
        if self._example is None:
            self._example = self._model._run_batched(1, trace_mode=TraceMode.PRIOR_FOR_INFERENCE_NETWORK,
                                                     prior_inflation=self._prior_inflation)
        return self._example

    def save_dataset(self, dataset_dir, num_traces, num_traces_per_file, observe_names, batch_size=None):
        """Generate prior traces on the GPU and write them as columnar trace files (reference:
        OnlineDataset.save_dataset, pyprob/nn/dataset.py:121-137 — one file per num_traces_per_file traces)."""
        from . import offline
        names = []
        written = 0
        while written < num_traces:
            count = num_traces_per_file   # like the reference, every file is full: ceil(num_traces / per file) files
            chunks, have = [], 0
            while have < count:
                b = min(batch_size or count, count - have)
                batch = self.next_batch(b)
                subs = batch.to_sub_batches(observe_names)
                dims = [int(np.prod(batch.trace.value_shape(batch.trace.named_variables[nm])))
                        for nm in observe_names]
                chunks.append(offline.TraceColumns.from_sub_batches(subs, observe_names, dims))
                have += b
            cols = chunks[0] if len(chunks) == 1 else offline.concat_columns(chunks)
            names.append(offline.save_columns(dataset_dir, cols))
            written += count
        return names
