"""Weighted sample container filled from device tensors.

Keeps the reference's ``Empirical`` semantics for the part of it that is on the hot path
(pyprob/distributions/empirical.py:298-340, :451-466, :759-766): fp32 log-weights, fp64 normalisation
(log-sum-exp), ESS = 1/sum p^2, expectations in fp64 — with the normalisation done by the CUDA reduce
kernels (ppb_weights_partials / ppb_weights_finalize).  Disk-backed modes, plotting, copying are out of scope.
"""
import copy

import torch

from . import ops


class Empirical:
    def __init__(self, values=None, log_weights=None, name='Empirical', sharded=False):
        """sharded=True: this rank holds one shard of the particles; normalisation statistics (log normaliser, ESS,
        logits) are global — the per-block partial triples of all ranks are all-gathered and combined exactly."""
        self.name = name
        self._sharded = sharded
        self._values = values                  # tensor [N, ...] on the GPU, or a python list
        n = len(values) if values is not None else 0
        if log_weights is None:
            log_weights = torch.zeros(n, dtype=torch.float32, device='cuda')
        self.log_weights = torch.as_tensor(log_weights, dtype=torch.float32).to('cuda').contiguous()
        self._finalized = False
        self._metadata = []
        self.finalize()

    def finalize(self):
        self._length = int(self.log_weights.numel())
        if self._length > 0:
            partials = None
            if getattr(self, '_sharded', False):
                from . import parallel
                partials = parallel.gather_weight_partials(ops.weights_partials(self.log_weights))
            self._stats, self._logits = ops.weights_finalize(self.log_weights, partials=partials)
        else:
            self._stats, self._logits = None, None
        self._probs = None
        self._finalized = True
        return self

    # ---- basic accessors ----------------------------------------------------------------------------------
    def __len__(self):
        return self._length

    length = property(lambda self: self._length)

    @property
    def values(self):
        return self._values

    def __getitem__(self, index):
        """An int gives the value; a slice gives a new Empirical of those values and weights with the metadata copied
        (reference empirical.py:415-422), e.g. ``posterior[burn_in:]``."""
        if isinstance(index, slice):
            values = self._values[index]
            ret = Empirical(values, self.log_weights[index], name=self.name)
            ret._metadata = copy.deepcopy(self._metadata)
            ret.add_metadata(op='slice', index='{}'.format(index))
            return ret
        return self._values[index]

    def values_numpy(self):
        return self._values.detach().cpu().numpy() if torch.is_tensor(self._values) else self._values

    def get_values(self):
        return self._values

    @property
    def logits(self):
        """Normalised log weights, fp64 (reference: Categorical(logits=log_weights.double()).logits)."""
        return self._logits

    @property
    def weights(self):
        if self._probs is None:
            self._probs = torch.exp(self._logits)
        return self._probs

    @property
    def log_normalizer(self):
        return float(self._stats[0])

    @property
    def effective_sample_size(self):
        return float(self._stats[1])

    @property
    def metadata(self):
        """The list of metadata dicts (e.g. ``op='posterior', num_chains=...``), oldest first."""
        return self._metadata

    def add_metadata(self, **kwargs):
        self._metadata.append(kwargs)

    def rename(self, name):
        self.name = name
        return self

    # ---- moments (fp64, like the reference's expectation()) --------------------------------------------------
    def _tensor_values(self):
        if not torch.is_tensor(self._values):
            raise NotImplementedError('moments need tensor-valued samples')
        return self._values.double().reshape(self._length, -1)

    def expectation(self, func):
        v = func(self._values) if torch.is_tensor(self._values) else torch.stack([func(x) for x in self._values])
        v = v.double().reshape(self._length, -1)
        return (v * self.weights.view(-1, 1)).sum(0).squeeze()

    @property
    def mean(self):
        return (self._tensor_values() * self.weights.view(-1, 1)).sum(0).squeeze()

    @property
    def variance(self):
        v = self._tensor_values()
        m = (v * self.weights.view(-1, 1)).sum(0, keepdim=True)
        return (((v - m) ** 2) * self.weights.view(-1, 1)).sum(0).squeeze()

    @property
    def stddev(self):
        return self.variance.sqrt()

    @property
    def mode(self):
        return self._values[int(torch.argmax(self._logits))]

    def sample(self, num_samples=1):
        idx = torch.multinomial(self.weights, num_samples, replacement=True)
        out = self._values[idx] if torch.is_tensor(self._values) else [self._values[int(i)] for i in idx]
        return out[0] if num_samples == 1 else out

    def unweighted(self):
        return Empirical(self._values, None, name=self.name)

    def resample(self, num_samples):
        idx = torch.multinomial(self.weights, num_samples, replacement=True)
        vals = self._values[idx] if torch.is_tensor(self._values) else [self._values[int(i)] for i in idx]
        return Empirical(vals, None, name=self.name)

    def __repr__(self):
        return 'Empirical(name:{}, length:{:,}, ESS:{:,.2f})'.format(self.name, self._length,
                                                                     self.effective_sample_size if self._length else 0)
