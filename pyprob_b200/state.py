"""Lock-step trace interpreter: ``sample`` / ``observe`` / ``tag`` / ``factor`` over n particles at once.

Per-site weight semantics follow the reference's IS and IC branches (pyprob/state.py:118-155, :192-219,
:280-288); the per-particle Python loop of pyprob/model.py:59-60 is replaced by one execution of the user's
``forward`` in which every sampled value is a length-n CUDA tensor.  Data-dependent control flow is written
with :func:`while_loop` (lanes leave the loop individually); a model that instead calls ``float()`` on a
sampled tensor still works — the engine falls back to one particle per execution (see model.py).
"""
import dis
import sys
import time
import warnings

import torch

from . import util
from .distributions import Bernoulli, Categorical, Distribution, Mixture, Normal, Poisson, Uniform
from .network import InferenceNetworkFeedForward
from .trace import BatchedTrace, Site
from .util import InferenceEngine, PriorInflation, TraceMode

_trace_mode = TraceMode.PRIOR
_inference_engine = InferenceEngine.IMPORTANCE_SAMPLING
_prior_inflation = PriorInflation.DISABLED
_likelihood_importance = 1.0
_current_trace = None
_root_function_name = None
_network = None
_previous_site = None
_observed = {}
_mask = None            # bool [n] of lanes executing the current statement, None = all
_mask_idx = None        # indices of the lanes of _mask (computed once per while_loop iteration), or None
_mask_parent = None     # the mask this one was narrowed from (while_loop: the previous iteration's mask)
_trace_start = None
_target_cache = {}
_NO_MASK_YET = object()


# ---- addressing (same information content as the reference's bytecode addresses, state.py:31-84) --------
def _assignment_target(code, lasti):
    """What the statement does with the value of the sample/observe call at bytecode offset `lasti` (reference
    `_extract_target_of_assignment`, pyprob/state.py:53-84): a variable name, 'return', ('subscr', base, index source) for
    ``base[i] = pyprob.sample(...)`` with a constant or local-variable index, or None."""
    key = (code, lasti)
    if key not in _target_cache:
        target = None
        ins = [i for i in dis.get_instructions(code) if i.offset > lasti and i.opname not in ('CACHE', 'PRECALL', 'NOP')]
        if ins:
            first = ins[0]
            if first.opname in ('STORE_FAST', 'STORE_NAME', 'STORE_GLOBAL', 'STORE_DEREF'):
                target = first.argval
            elif first.opname == 'RETURN_VALUE':
                target = 'return'
            elif (first.opname in ('LOAD_FAST', 'LOAD_NAME', 'LOAD_GLOBAL') and len(ins) >= 3
                  and ins[1].opname in ('LOAD_CONST', 'LOAD_FAST') and ins[2].opname == 'STORE_SUBSCR'):
                src = ('const', ins[1].argval) if ins[1].opname == 'LOAD_CONST' else ('fast', ins[1].argval)
                target = ('subscr', first.argval, src)
        _target_cache[key] = target
    return _target_cache[key]


def _extract_address(depth=2):
    frame = sys._getframe(depth)
    ip = frame.f_lasti
    target = _assignment_target(frame.f_code, ip)
    if isinstance(target, tuple):      # base[index] = ...: only integer indices name a target (reference :77-81)
        _, base, (kind, arg) = target
        index = arg if kind == 'const' else frame.f_locals.get(arg)
        target = '{}[{}]'.format(base, index) if type(index) is int else None
    names = []
    f = frame
    while f is not None:
        n = f.f_code.co_name
        if n.startswith('<') and n != '<listcomp>':
            break
        names.append(n)
        if n == _root_function_name:
            break
        f = f.f_back
    return '{}__{}__{}'.format(ip, '__'.join(reversed(names)), target if target is not None else '?')


def _addresses(distribution, address, depth):
    base = (_extract_address(depth + 1) if address is None else address) + '__' + distribution._address_suffix
    instance = _current_trace.next_instance(base)
    return base, instance, base + '__' + str(instance)


# ---- helpers -----------------------------------------------------------------------------------------------
def _inflate(distribution):
    if _prior_inflation == PriorInflation.ENABLED:
        if isinstance(distribution, Categorical):
            return Categorical(torch.full((distribution.num_categories,), 1.0 / distribution.num_categories))
        if isinstance(distribution, Normal):
            return Normal(distribution.loc, distribution.scale * 3)
    return None


def _broadcast_value(value, n):
    if isinstance(value, (int, float)):      # observed constants: filled on the device, no host->device copy (= no sync)
        return torch.full((n,), float(value), dtype=torch.float32, device='cuda')
    v = torch.as_tensor(value, dtype=torch.float32).to('cuda').reshape(-1)
    if v.numel() == 1 and n > 1:
        v = v.expand(n).contiguous()
    elif v.numel() != n:
        raise ValueError('pyprob_b200 scores scalar random variables: observed value has {} elements for {} '
                         'particles'.format(v.numel(), n))
    return v


def _accumulate(trace, fn):
    """Run fn(acc) (which adds weight terms into acc) for the lanes of the current mask only."""
    if _mask is None:
        fn(trace.log_w)
    else:
        term = torch.zeros_like(trace.log_w)
        fn(term)
        trace.log_w.add_(term.masked_fill_(~_mask, 0.0))   # masked-out lanes may hold junk (even NaN): dropped


def _prior_params(distribution):
    if isinstance(distribution, Normal):
        return distribution.loc, distribution.scale
    if isinstance(distribution, Uniform):
        return distribution.low, distribution.high
    return None, None


# ---- public statements ----------------------------------------------------------------------------------------
def tag(value, name=None, address=None):
    if _current_trace is None:
        return
    base = (_extract_address(2) if address is None else address) + '__None'
    instance = _current_trace.next_instance(base)
    _current_trace.add(Site(None, value, base, base + '__' + str(instance), instance, name=name, tagged=True,
                            mask=_mask))


def factor(log_prob=None, log_prob_func=None, name=None, address=None):
    """Add an arbitrary per-particle log-weight term (reference: state.py:113-115, distributions/factor.py)."""
    if _current_trace is None:
        return
    lp = log_prob_func() if log_prob is None else log_prob
    lp = _broadcast_value(lp, _current_trace.n).double() * _likelihood_importance
    _accumulate(_current_trace, lambda acc: acc.add_(lp))


def observe(distribution, value=None, name=None, address=None):
    trace = _current_trace
    if trace is None:
        return
    base, instance, addr = _addresses(distribution, address, 2)
    n = trace.n
    if name in _observed:
        value = _broadcast_value(_observed[name], n)
    elif value is not None:
        value = _broadcast_value(value, n)
    elif _trace_mode == TraceMode.PRIOR_FOR_INFERENCE_NETWORK:
        value = distribution.sample(n)
    if value is None:
        trace.add(Site(distribution, None, base, addr, instance, name=name, observed=False, mask=_mask))
        return None
    if _trace_mode == TraceMode.POSTERIOR:
        _accumulate(trace, lambda acc: distribution.score_into(value, acc, _likelihood_importance))
    trace.add(Site(distribution, value, base, addr, instance, name=name, observed=True, mask=_mask))
    return value


def sample(distribution, name=None, address=None, control=True):
    global _previous_site
    trace = _current_trace
    if trace is None:
        return distribution.sample()
    base, instance, addr = _addresses(distribution, address, 2)
    n = trace.n
    if name in _observed:
        value = _broadcast_value(_observed[name], n)
        if _trace_mode == TraceMode.POSTERIOR:
            _accumulate(trace, lambda acc: distribution.score_into(value, acc, _likelihood_importance))
        trace.add(Site(distribution, value, base, addr, instance, name=name, observed=True, mask=_mask))
        return value

    use_network = (_trace_mode == TraceMode.POSTERIOR and control and
                   _inference_engine == InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK)
    if use_network:
        value = _sample_from_proposal(trace, distribution, addr, n)
    else:
        inflated = _inflate(distribution)
        if inflated is None:
            value = distribution.sample(n)       # proposal == prior: weight term is exactly zero (state.py:198)
        else:
            value, q_lp = inflated.sample(n, with_log_prob=True)
            if _trace_mode == TraceMode.POSTERIOR or _trace_mode == TraceMode.PRIOR_FOR_INFERENCE_NETWORK:
                def fn(acc):
                    distribution.score_into(value, acc, 1.0)
                    acc.sub_(q_lp.double())
                _accumulate(trace, fn)
    site = Site(distribution, value, base, addr, instance, control=control, name=name, mask=_mask)
    trace.add(site)
    if use_network:
        _previous_site = site
    return value


def _lanes(x, idx):
    """Rows `idx` of a per-particle parameter (tensors only; scalars are shared by all particles)."""
    return x[idx] if (torch.is_tensor(x) and x.numel() > 1 and idx is not None) else x


def _sample_from_proposal(trace, distribution, addr, n):
    """IC branch (state.py:203-219): value ~ q(.|LSTM state); weight += log p(value) - log q(value).

    The proposal network only runs for the particles that execute this statement (the lanes of the current mask), packed
    densely, so a loop whose lanes drop out costs what its live lanes cost.  Every lane keeps its own LSTM state and its
    own previous site (address id + value): lanes that reached this statement from different sites are stepped in
    separate groups, like the per-trace `_current_trace_previous_variable` of the reference (state.py:212)."""
    net = _network
    K = net._proposal_mixture_components
    if isinstance(net, InferenceNetworkFeedForward):
        return _propose_and_weigh(trace, distribution, n, *_feedforward_params(net, distribution, addr, n, K))
    H = net._lstm_dim
    st = trace.ic_state
    if st is None:
        st = trace.ic_state = {'h': torch.zeros(n, H, device='cuda'), 'c': torch.zeros(n, H, device='cuda'),
                               'prev_id': torch.full((n,), -1, dtype=torch.int64, device='cuda'),
                               'prev_value': torch.zeros(n, device='cuda'),
                               'uniform_prev': -1}    # host copy of prev_id when all lanes are known to share it
    known = addr in net._addresses
    if not known:
        warnings.warn('Address unknown by inference network: {}'.format(addr))
    idx = None if _mask is None else (_mask_idx if _mask_idx is not None else torch.nonzero(_mask).view(-1))
    if idx is not None and idx.numel() == 0:     # nobody executes the statement: nothing to propose, nothing to weigh
        return distribution.sample(n)
    p0, p1 = _prior_params(distribution)
    # group the executing lanes by the site they came from.  Known on the host without a device round trip when every lane
    # shares its previous site, or when this mask is (a narrowing of) the mask of the previous proposal site: then all of its
    # lanes executed that site last.
    last_mask = st.get('last_mask', _NO_MASK_YET)
    if idx is None and st['uniform_prev'] is not None:
        groups = [(st['uniform_prev'], None)]
    elif idx is not None and st['uniform_prev'] is not None:
        groups = [(st['uniform_prev'], None)]
    elif idx is not None and last_mask is not _NO_MASK_YET and (_mask is last_mask or _mask_parent is last_mask):
        groups = [(st['last_id'], None)]
    else:
        ids = st['prev_id'] if idx is None else st['prev_id'][idx]
        uniq = torch.unique(ids).tolist()
        groups = [(u, None if len(uniq) == 1 else (ids == u)) for u in uniq]
    is_cat = isinstance(distribution, Categorical)
    width = distribution.num_categories if is_cat else 1 if isinstance(distribution, Bernoulli) else 3 * K
    params = None
    covered = True        # every executing lane got a proposal from the network
    by_id = net._address_by_id()
    for pid, sel in groups:
        if not known or pid == -2 or (pid >= 0 and pid not in by_id):
            covered = False
            continue
        lanes = idx if sel is None else (torch.nonzero(sel).view(-1) if idx is None else idx[sel])
        if lanes is None:
            h, c = st['h'], st['c']
            pv = st['prev_value']
        else:
            h, c = st['h'][lanes], st['c'][lanes]
            pv = st['prev_value'][lanes]
        out = net._infer_step_lanes(addr, None if pid < 0 else by_id[pid], None if pid < 0 else pv, _lanes(p0, lanes),
                                    _lanes(p1, lanes), h, c)
        if lanes is None:
            params = out
        else:
            st['h'].index_copy_(0, lanes, h)
            st['c'].index_copy_(0, lanes, c)
            if params is None:
                params = _default_params(distribution, n, K, width)
            params.index_copy_(0, lanes, out)
    has = None
    if not covered:   # lanes whose previous / current address the network does not know fall back to the prior
        has = torch.zeros(n, dtype=torch.bool, device='cuda')
        for pid, sel in groups:
            if known and pid != -2 and (pid < 0 or pid in by_id):
                lanes = idx if sel is None else (torch.nonzero(sel).view(-1) if idx is None else idx[sel])
                if lanes is None:
                    has.fill_(True)
                else:
                    has[lanes] = True
    value = _propose_and_weigh(trace, distribution, n, params, has)
    # this site becomes the previous site of the lanes that executed it
    new_id = net._addresses[addr]['id'] if known else -2
    if idx is None:
        st['prev_id'].fill_(new_id)
        st['prev_value'] = value.to(torch.float32).clone()
        st['uniform_prev'] = new_id
    else:
        st['prev_id'].index_fill_(0, idx, new_id)
        st['prev_value'].index_copy_(0, idx, value.to(torch.float32)[idx])
        st['uniform_prev'] = None
    st['last_mask'], st['last_id'] = _mask, new_id
    return value


def _feedforward_params(net, distribution, addr, n, K):
    """Feed-forward network (inference_network_feedforward.py:53-66): no LSTM state and no previous site, so the lanes
    that execute this statement are proposed for in ONE call.  -> (params [n, width] or None, None)."""
    idx = None if _mask is None else (_mask_idx if _mask_idx is not None else torch.nonzero(_mask).view(-1))
    if addr not in net._addresses:
        warnings.warn('Address unknown by inference network: {}'.format(addr))
        return None, None
    if idx is not None and idx.numel() == 0:
        return None, None
    p0, p1 = _prior_params(distribution)
    out = net._infer_step_lanes(addr, _lanes(p0, idx), _lanes(p1, idx), n if idx is None else idx.numel())
    if idx is None:
        return out, None
    is_cat = isinstance(distribution, Categorical)
    width = distribution.num_categories if is_cat else 1 if isinstance(distribution, Bernoulli) else 3 * K
    params = _default_params(distribution, n, K, width)
    params.index_copy_(0, idx, out)
    return params, None


def _propose_and_weigh(trace, distribution, n, params, has):
    """value ~ proposal(params) where `has` (None: every lane) marks the lanes the network proposed for, the prior
    elsewhere; the weight term log p(value) - log q(value) joins the trace's accumulator."""
    K = _network._proposal_mixture_components
    is_cat = isinstance(distribution, Categorical)
    if params is None:   # nobody could be proposed for: prior proposal, weight term exactly zero (reference warning path)
        value = distribution.sample(n)
    else:
        if is_cat:
            proposal = Categorical(probs=params)
        elif isinstance(distribution, Bernoulli):   # proposal_bernoulli_bernoulli.py: prior parameters are not inputs
            proposal = Bernoulli(probs=params[:, 0])
        elif isinstance(distribution, Normal):
            proposal = Mixture.from_rows(params[:, :K], params[:, K:2 * K], params[:, 2 * K:])
        elif isinstance(distribution, Uniform):
            proposal = Mixture.from_rows(params[:, :K], params[:, K:2 * K], params[:, 2 * K:], distribution.low,
                                         distribution.high)
        elif isinstance(distribution, Poisson):
            proposal = Mixture.from_rows(params[:, :K], params[:, K:2 * K], params[:, 2 * K:], 0.0, 40.0)
        else:
            raise RuntimeError('Distribution currently unsupported: {}'.format(distribution.name))
        value, q_lp = proposal.sample(n, with_log_prob=True)
        if has is not None:
            prior_value, prior_lp = distribution.sample(n, with_log_prob=True)
            value = torch.where(has, value, prior_value)
            q_lp = torch.where(has, q_lp, prior_lp)

        def fn(acc):
            distribution.score_into(value, acc, 1.0)
            acc.sub_(q_lp.double())
        _accumulate(trace, fn)
    return value


def _default_params(distribution, n, K, width):
    """Benign proposal parameters for lanes that do not execute the statement (their draws are discarded by the mask)."""
    p = torch.zeros(n, width, device='cuda')
    if isinstance(distribution, Categorical):
        p.fill_(1.0 / width)
    elif isinstance(distribution, Bernoulli):
        p.fill_(0.5)
    else:
        if isinstance(distribution, Uniform):
            lo, hi = distribution.low, distribution.high
            mid = (lo + hi) / 2
            p[:, :K] = mid.view(-1, 1) if torch.is_tensor(mid) else mid
        elif isinstance(distribution, Poisson):
            p[:, :K] = 1.0
        p[:, K:2 * K] = 1.0
        p[:, 2 * K:] = 1.0 / K
    return p


def while_loop(cond_fn, body_fn, state, max_iterations=10000):
    """Lock-step ``while cond(state): state = body(state)`` over particles.

    ``state`` is a dict of length-n tensors; ``cond_fn(state)`` returns a bool [n]; lanes whose condition is
    false stop executing sample/observe statements (their trace ends there) while the others continue."""
    global _mask, _mask_idx, _mask_parent
    trace = _current_trace
    n = trace.n if trace is not None else None
    outer, outer_idx, outer_parent = _mask, _mask_idx, _mask_parent
    state = {k: (v if torch.is_tensor(v) else torch.full((n,), float(v), device='cuda')) for k, v in state.items()}
    prev = None
    for _ in range(max_iterations):
        m = cond_fn(state)
        if outer is not None:
            m = m & outer
        if prev is not None:
            m = m & prev          # a lane that left the loop stays out (its state is frozen, so cond cannot change anyway)
        idx = torch.nonzero(m).view(-1)     # the one device round trip of the iteration: who is still in
        if idx.numel() == 0:
            break
        _mask, _mask_idx, _mask_parent = m, idx, (prev if prev is not None else outer)
        try:
            out = body_fn(state)
        finally:
            _mask, _mask_idx, _mask_parent = outer, outer_idx, outer_parent
        state = {k: torch.where(m, out[k].to(state[k].dtype), state[k]) for k in state}
        prev = m
    else:
        raise RuntimeError('while_loop: exceeded max_iterations')
    return state


# ---- trace life cycle (reference: state.py:296-354) -------------------------------------------------------------
def _init_traces(func, trace_mode=TraceMode.PRIOR, prior_inflation=PriorInflation.DISABLED,
                 inference_engine=InferenceEngine.IMPORTANCE_SAMPLING, inference_network=None, observe=None,
                 likelihood_importance=1.0):
    global _trace_mode, _inference_engine, _prior_inflation, _likelihood_importance
    global _root_function_name, _network, _observed
    if inference_engine in (InferenceEngine.LIGHTWEIGHT_METROPOLIS_HASTINGS,
                            InferenceEngine.RANDOM_WALK_METROPOLIS_HASTINGS):
        raise NotImplementedError('pyprob_b200 implements the importance-sampling engines only (MCMC is sequential '
                                  'and out of scope; use the reference for LMH/RMH)')
    _trace_mode, _inference_engine = trace_mode, inference_engine
    _prior_inflation, _likelihood_importance = prior_inflation, float(likelihood_importance)
    _root_function_name = func.__code__.co_name
    if observe is None:
        _observed = {}
    else:
        if any(v is None for v in observe.values()):
            raise RuntimeError('Observe has missing value(s): {}'.format(observe))
        _observed = observe
    _network = inference_network
    if _network is None:
        if inference_engine == InferenceEngine.IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK:
            raise ValueError('Cannot run trace with IMPORTANCE_SAMPLING_WITH_INFERENCE_NETWORK without an inference '
                             'network.')
    else:
        _network.eval()
        _network._infer_init(_observed)


def _begin_trace(n):
    global _current_trace, _previous_site, _trace_start, _mask
    _trace_start = time.time()
    _current_trace = BatchedTrace(n)
    _previous_site = None
    _mask = None
    if _network is not None:
        _network._infer_state = None


def _end_trace(result):
    global _current_trace
    trace = _current_trace
    trace.result = result
    trace.execution_time_sec = time.time() - _trace_start
    _current_trace = None
    return trace


__all__ = ['sample', 'observe', 'tag', 'factor', 'while_loop', 'Distribution']
