"""Metropolis-Hastings engines (LMH, RMH) as C lock-step chains (reference: pyprob/model.py:118-178,
pyprob/state.py:225-276, :328-336).

A single MH chain is sequential, but one MH step is one execution of the program, so C independent chains are the C
lanes of one lock-step execution.  This module owns the per-chain trace tables (format: include/pyprob_b200.h section 7):
an address -> column map that grows as addresses appear, device arrays [2, C, lda] holding the current and the candidate
trace of every chain, and per-chain fp64 accumulators and counters.  One step is

  ppb_mh_select   pick each chain's MH site among the columns of its current trace, reset the candidate accumulators
  forward()       every executed sample statement calls :meth:`Chains.site`: a fresh prior draw (the family's own
                  sampler), the current value and its rescoring (the family's own log_prob kernel), and ppb_mh_site,
                  which writes the candidate; observe / factor add into the candidate's log_prob_observed (trace.log_w)
  ppb_mh_accept   log alpha, accept, flip buffers, record map_func of the current trace

with no device -> host copy beyond those of while_loop.  Counters are read once, at the end.
"""
import warnings

import torch

from . import ops, state, util
from .distributions import Normal, Uniform, set_shard_first_index
from .empirical import Empirical
from .util import InferenceEngine, TraceMode

_INITIAL_COLUMNS = 16


class Chains:
    """Trace tables of C chains; rows first .. first + n - 1 execute together (n = C, or n = 1 per chain for models
    with python-scalar control flow)."""

    def __init__(self, num_chains, inference_engine, num_records):
        C = self.C = int(num_chains)
        self.rmh = inference_engine == InferenceEngine.RANDOM_WALK_METROPOLIS_HASTINGS
        self.num_records = num_records
        self.columns = {}                  # address -> column
        self.ncols, self.lda = 0, _INITIAL_COLUMNS
        dev = 'cuda'
        self.val = torch.zeros(2, C, self.lda, dtype=torch.float32, device=dev)
        self.lp = torch.zeros(2, C, self.lda, dtype=torch.float32, device=dev)
        self.stamp = torch.full((2, C, self.lda), -1, dtype=torch.int32, device=dev)
        self.reused = torch.zeros(2, C, self.lda, dtype=torch.uint8, device=dev)
        self.buf = torch.zeros(C, dtype=torch.int32, device=dev)
        self.cur_stamp = torch.full((C,), -2, dtype=torch.int32, device=dev)
        self.choice = torch.full((C,), -1, dtype=torch.int32, device=dev)
        self.cur_n = torch.zeros(C, dtype=torch.int32, device=dev)
        self.cand_n = torch.zeros(C, dtype=torch.int32, device=dev)
        self.cur_lpo = torch.zeros(C, dtype=torch.float64, device=dev)
        self.cand_lpo = torch.zeros(C, dtype=torch.float64, device=dev)
        self.reuse = torch.zeros(C, dtype=torch.float64, device=dev)
        self.trans = torch.zeros(C, dtype=torch.float64, device=dev)
        self.log_alpha = torch.zeros(C, dtype=torch.float64, device=dev)
        self.accepted = torch.zeros(C, dtype=torch.int64, device=dev)
        self.reused_count = torch.zeros(C, dtype=torch.int64, device=dev)
        self.sites_all = torch.zeros(C, dtype=torch.int64, device=dev)
        self.cur_map = self.cand_map = self.out = None
        self.map_words, self.map_dtype, self.map_width = 0, None, 0
        self.step = -1                     # stamp of the running step; the initial trace is step 0
        self.first = 0
        self.offsets = None                # Philox offsets (select, accept) of the last step

    # ---- tables ---------------------------------------------------------------------------------------------
    def column(self, address):
        col = self.columns.get(address)
        if col is None:
            col = self.columns[address] = self.ncols
            self.ncols += 1
            if col >= self.lda:
                self._grow(2 * self.lda)
        return col

    def _grow(self, lda):
        for name in ('val', 'lp', 'stamp', 'reused'):
            old = getattr(self, name)
            new = torch.full((2, self.C, lda), -1 if name == 'stamp' else 0, dtype=old.dtype, device=old.device)
            new[:, :, :self.lda] = old
            setattr(self, name, new)
        self.lda = lda

    def log_w_view(self, n):
        """The candidate's log_prob_observed accumulator of the executing rows (the trace's log_w)."""
        return self.cand_lpo[self.first:self.first + n]

    # ---- one sample statement ----------------------------------------------------------------------------------
    def site(self, distribution, address, n, mask):
        col = self.column(address)
        fresh, fresh_lp = distribution.sample(n, with_log_prob=True)
        mask_u8 = None if mask is None else mask.view(torch.uint8)
        old_v, old_lp, has = ops.mh_fetch(self, col, mask_u8, n, self.first)
        rescored = distribution.log_prob(old_v)
        kind, p0, p1, offset = 0, None, None, 0
        if self.rmh and isinstance(distribution, Normal):
            kind, p0, p1, offset = 1, distribution.loc, distribution.scale, util.next_draw_offset()
        elif self.rmh and isinstance(distribution, Uniform):
            kind, p0, p1, offset = 2, distribution.low, distribution.high, util.next_draw_offset()
        return ops.mh_site(self, kind, col, mask_u8, n, self.first, fresh, fresh_lp, old_v, old_lp, has,
                           rescored.reshape(-1), p0, p1, util._seed, offset)

    def _store_map(self, v, n):
        if not torch.is_tensor(v):
            v = torch.as_tensor(v, dtype=torch.float32, device='cuda')
        v = v.to('cuda')
        if v.dtype not in (torch.float32, torch.int32, torch.float64, torch.int64):
            v = v.to(torch.float32)
        v = v.reshape(n, -1) if v.numel() >= n else v.reshape(1, -1).expand(n, -1)
        words = v.contiguous().view(torch.int32)
        if self.cand_map is None:
            self.map_dtype, self.map_width, self.map_words = v.dtype, v.size(1), words.size(1)
            self.cand_map = torch.zeros(self.C, self.map_words, dtype=torch.int32, device='cuda')
            self.cur_map = torch.zeros_like(self.cand_map)
            self.out = torch.zeros(max(self.num_records, 1), self.C, self.map_words, dtype=torch.int32, device='cuda')
        elif words.size(1) != self.map_words or v.dtype != self.map_dtype:
            raise RuntimeError('map_func must return the same shape and dtype for every trace')
        self.cand_map[self.first:self.first + n] = words

    # ---- one MH step ---------------------------------------------------------------------------------------------
    def run_step(self, model, map_func, slot, scalar, args=(), kwargs=None):
        """One MH step of every chain (the initial trace when self.step is -1); records into out[slot] when slot >= 0."""
        kwargs = kwargs or {}
        self.step += 1
        initial = self.step == 0
        off_select = util.next_draw_offset()
        ops.mh_select(self, initial, util._seed, off_select)
        rows = [(c, 1) for c in range(self.C)] if scalar else [(0, self.C)]
        counter0 = top = util._draw_counter
        state._mcmc = self
        try:
            for first, n in rows:
                util._draw_counter = counter0     # every chain draws from the same offsets, as in one lock-step run
                self.first = first
                set_shard_first_index(first)
                trace = model._run_batched(n, init=False, *args, **kwargs)
                self._store_map(map_func(trace), n)
                top = max(top, util._draw_counter)
        finally:
            state._mcmc = None
            self.first = 0
            set_shard_first_index(0)
        util._draw_counter = top
        off_accept = util.next_draw_offset()
        ops.mh_accept(self, initial, slot, util._seed, off_accept)
        self.offsets = (off_select, off_accept)

    def values(self):
        """Recorded map_func rows in step-major order: [num_records * C] (or [num_records * C, width])."""
        v = self.out[:self.num_records].reshape(self.num_records * self.C, self.map_words).view(self.map_dtype)
        return v.squeeze(-1)


def _scalar_error(e):
    s = str(e)
    return ('convert' in s and 'calar' in s) or 'ambiguous' in s


def posterior(model, num_traces, inference_engine, map_func, observe, thinning_steps, likelihood_importance,
              num_chains=1, args=(), kwargs=None):
    """num_traces MH steps of num_chains chains -> (Empirical of map_func(current trace), Chains).

    The Empirical holds num_chains * ceil(num_traces / thinning_steps) unweighted states in step-major order: state
    k * num_chains + c is chain c after recorded step k, so ``posterior[burn_in * num_chains:]`` drops the burn-in of
    every chain."""
    thinning = 1 if thinning_steps is None else int(thinning_steps)
    if thinning < 1 or num_chains < 1:
        raise ValueError('thinning_steps and num_chains must be positive')
    num_records = -(-int(num_traces) // thinning)
    state._init_traces(model.forward, trace_mode=TraceMode.POSTERIOR, inference_engine=inference_engine,
                       observe=observe, likelihood_importance=likelihood_importance)
    while True:
        chains = Chains(num_chains, inference_engine, num_records)
        try:
            chains.run_step(model, map_func, -1, model._scalar_mode, args, kwargs)
            break
        except (ValueError, RuntimeError) as e:
            if model._scalar_mode or not _scalar_error(e):
                raise
            warnings.warn('Model uses python-scalar control flow on sampled values; running one chain per execution '
                          '(slow). Use pyprob_b200.while_loop for lock-step loops.')
            model._scalar_mode = True
    if int(chains.cur_n.min()) == 0:
        raise RuntimeError('Cannot run MCMC inference with empty initial trace. Make sure the model has at least one '
                           'pyprob.sample statement.')
    for i in range(int(num_traces)):
        chains.run_step(model, map_func, i // thinning if i % thinning == 0 else -1, model._scalar_mode, args, kwargs)
    post = Empirical(chains.values(), None)
    accepted, reused, sites = (int(x) for x in torch.stack([chains.accepted.sum(), chains.reused_count.sum(),
                                                             chains.sites_all.sum()]).tolist())
    steps = int(num_traces) * num_chains
    accept_pct = 100 * accepted / max(1, steps)
    reuse_pct = 100 * reused / max(1, sites)
    post.rename('Posterior, {}, traces: {:,}{}{}, accepted: {:,.2f}%, sample reuse: {:,.2f}%'.format(
        'RMH' if chains.rmh else 'LMH', post.length,
        '' if thinning == 1 else ' (thinning steps: {:,})'.format(thinning),
        '' if num_chains == 1 else ' (chains: {:,})'.format(num_chains), accept_pct, reuse_pct))
    post.add_metadata(op='posterior', num_traces=num_traces, inference_engine=str(inference_engine),
                      likelihood_importance=likelihood_importance, thinning_steps=thinning, num_chains=num_chains,
                      num_traces_accepted=accepted, num_samples_reuised=reused, num_samples=sites)
    return post, chains
