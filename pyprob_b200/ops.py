"""Tensor-level wrappers over the scoring / sampling / weight kernels (C-ABI sections 1-3).

Every function takes CUDA fp32 tensors and launches on the current torch stream.  Parameters may be
0-d / 1-element tensors (broadcast over particles) or length-n tensors.
"""
import ctypes

import numpy as np
import torch

from . import _lib
from ._lib import call, ptr, stream


_scalar_cache = {}


def _f32(t, device):
    if not torch.is_tensor(t):
        if isinstance(t, (int, float)):
            # python scalars (distribution parameters shared by all particles): a host->device copy of a pageable scalar is a
            # full stream synchronisation; keep one device constant per value instead (filled by a kernel, no copy)
            key = (float(t), str(device))
            c = _scalar_cache.get(key)
            if c is None:
                if len(_scalar_cache) > 4096:
                    _scalar_cache.clear()
                c = _scalar_cache[key] = torch.full((1,), float(t), dtype=torch.float32, device=device)
            return c
        t = torch.tensor(t, dtype=torch.float32, device=device)
    return t.to(device=device, dtype=torch.float32).contiguous()


def _param(t, n, device):
    """-> (tensor kept alive, pointer, stride)"""
    t = _f32(t, device)
    if t.numel() == 1:
        return t, ptr(t), 0
    if t.numel() != n:
        raise ValueError('parameter has {} elements, expected 1 or {}'.format(t.numel(), n))
    t = t.reshape(n)
    return t, ptr(t), 1


def _sink(n, device, lp_out, acc):
    if lp_out is None and acc is None:
        lp_out = torch.empty(n, dtype=torch.float32, device=device)
    if acc is not None and (acc.dtype != torch.float64 or acc.numel() != n or not acc.is_contiguous()):
        raise ValueError('acc must be a contiguous float64 tensor of length n')
    return lp_out, acc


# ---- the eleven families with an element-wise log_prob: the family-id entry points at D = 1 ----------------------------

EVENT_FAMILIES = {'Normal': 0, 'Uniform': 1, 'Poisson': 2, 'Bernoulli': 3, 'Exponential': 4, 'Gamma': 5,
                  'LogNormal': 6, 'Weibull': 7, 'Beta': 8, 'Binomial': 9, 'VonMises': 10}
EVENT_NUM_PARAMS = {0: 2, 1: 2, 2: 1, 3: 1, 4: 1, 5: 2, 6: 2, 7: 2, 8: 4, 9: 2, 10: 2}


def _slots(params, n, device):
    """-> (tensors kept alive, the four parameter pointers, the stride mask: bit k set where parameter k is per
    particle) of a D = 1 call"""
    held, ptrs, mask = [], [None, None, None, None], 0
    for k, x in enumerate(params):
        t, ptrs[k], stride = _param(x, n, device)
        held.append(t)
        mask |= stride << k
    return held, ptrs, mask


def _score(family, value, params, lp_out, acc, acc_scale):
    """log_prob of a family over the particle axis: value [n], each parameter a scalar or [n]."""
    value = _f32(value, value.device).reshape(-1)
    n = value.numel()
    held, p, mask = _slots(params, n, value.device)
    lp_out, acc = _sink(n, value.device, lp_out, acc)
    call('ppb_event_log_prob_d1', family, ptr(value), p[0], p[1], p[2], p[3], mask, ptr(lp_out), ptr(acc),
         float(acc_scale), n, stream())
    return lp_out


def normal_log_prob(value, mean, stddev, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Normal'], value, (mean, stddev), lp_out, acc, acc_scale)


def uniform_log_prob(value, low, high, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Uniform'], value, (low, high), lp_out, acc, acc_scale)


def poisson_log_prob(value, rate, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Poisson'], value, (rate,), lp_out, acc, acc_scale)


def bernoulli_log_prob(value, probs, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Bernoulli'], value, (probs,), lp_out, acc, acc_scale)


def exponential_log_prob(value, rate, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Exponential'], value, (rate,), lp_out, acc, acc_scale)


def gamma_log_prob(value, concentration, rate, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Gamma'], value, (concentration, rate), lp_out, acc, acc_scale)


def lognormal_log_prob(value, loc, scale, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['LogNormal'], value, (loc, scale), lp_out, acc, acc_scale)


def weibull_log_prob(value, scale, concentration, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Weibull'], value, (scale, concentration), lp_out, acc, acc_scale)


def beta_log_prob(value, concentration1, concentration0, low=0.0, high=1.0, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Beta'], value, (concentration1, concentration0, low, high), lp_out, acc, acc_scale)


def binomial_log_prob(value, total_count, probs, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['Binomial'], value, (total_count, probs), lp_out, acc, acc_scale)


def von_mises_log_prob(value, loc, concentration, lp_out=None, acc=None, acc_scale=1.0):
    return _score(EVENT_FAMILIES['VonMises'], value, (loc, concentration), lp_out, acc, acc_scale)


def _rows(t, n, device):
    """[C] shared or [n, C] per particle -> (tensor, row_stride, C)"""
    if torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 2 and t.stride(1) == 1 \
            and t.size(0) == n and t.stride(0) >= t.size(1):
        return t, t.stride(0), t.size(1)  # strided rows (e.g. a column block of the head output): no copy
    t = _f32(t, device)
    if t.dim() == 1:
        return t, 0, t.size(0)
    if t.dim() == 2 and t.size(0) == n:
        return t, t.size(1), t.size(1)
    if t.dim() == 2 and t.size(0) == 1:
        return t.reshape(-1), 0, t.size(1)
    raise ValueError('expected [C] or [n, C], got {}'.format(tuple(t.shape)))


def categorical_log_prob(value, probs, lp_out=None, acc=None, acc_scale=1.0):
    value = _f32(value, value.device).reshape(-1)
    n = value.numel()
    p, stride, C = _rows(probs, n, value.device)
    lp_out, acc = _sink(n, value.device, lp_out, acc)
    call('ppb_categorical_log_prob', ptr(value), ptr(p), stride, C, ptr(lp_out), ptr(acc), float(acc_scale), n,
         stream())
    return lp_out


def _mixture_rows(means, stddevs, probs, n, device):
    m, sm, K = _rows(means, n, device)
    s, ss, K2 = _rows(stddevs, n, device)
    p, sp, K3 = _rows(probs, n, device)
    if not (K == K2 == K3) or not (sm == ss == sp):
        raise ValueError('means/stddevs/probs must have identical shapes')
    return m, s, p, sm, K


def mixture_normal_log_prob(value, means, stddevs, probs, lp_out=None, acc=None, acc_scale=1.0):
    value = _f32(value, value.device).reshape(-1)
    n = value.numel()
    m, s, p, stride, K = _mixture_rows(means, stddevs, probs, n, value.device)
    lp_out, acc = _sink(n, value.device, lp_out, acc)
    call('ppb_mixture_normal_log_prob', ptr(value), ptr(m), ptr(s), ptr(p), stride, K, ptr(lp_out), ptr(acc),
         float(acc_scale), n, stream())
    return lp_out


def mixture_truncated_normal_log_prob(value, means, stddevs, probs, low, high, lp_out=None, acc=None, acc_scale=1.0):
    value = _f32(value, value.device).reshape(-1)
    n = value.numel()
    m, s, p, stride, K = _mixture_rows(means, stddevs, probs, n, value.device)
    lo, lop, los = _param(low, n, value.device)
    hi, hip, his = _param(high, n, value.device)
    lp_out, acc = _sink(n, value.device, lp_out, acc)
    call('ppb_mixture_truncated_normal_log_prob', ptr(value), ptr(m), ptr(s), ptr(p), stride, K, lop, los, hip, his,
         ptr(lp_out), ptr(acc), float(acc_scale), n, stream())
    return lp_out


# ---- samplers ---------------------------------------------------------------------------------------

def _out(n, device, want_lp):
    v = torch.empty(n, dtype=torch.float32, device=device)
    lp = torch.empty(n, dtype=torch.float32, device=device) if want_lp else None
    return v, lp


def _sample(family, params, n, seed, offset, first_index, with_log_prob, device):
    """n draws of a family (particle i from Philox index first_index + i), each parameter a scalar or [n]."""
    held, p, mask = _slots(params, n, device)
    v, lp = _out(n, device, with_log_prob)
    call('ppb_event_sample_d1', family, p[0], p[1], p[2], p[3], mask, ptr(v), ptr(lp), n, seed, offset, first_index,
         stream())
    return (v, lp) if with_log_prob else v


def normal_sample(mean, stddev, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Normal'], (mean, stddev), n, seed, offset, first_index, with_log_prob, device)


def uniform_sample(low, high, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Uniform'], (low, high), n, seed, offset, first_index, with_log_prob, device)


def poisson_sample(rate, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Poisson'], (rate,), n, seed, offset, first_index, with_log_prob, device)


def bernoulli_sample(probs, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Bernoulli'], (probs,), n, seed, offset, first_index, with_log_prob, device)


def exponential_sample(rate, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Exponential'], (rate,), n, seed, offset, first_index, with_log_prob, device)


def gamma_sample(concentration, rate, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Gamma'], (concentration, rate), n, seed, offset, first_index, with_log_prob, device)


def lognormal_sample(loc, scale, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['LogNormal'], (loc, scale), n, seed, offset, first_index, with_log_prob, device)


def weibull_sample(scale, concentration, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Weibull'], (scale, concentration), n, seed, offset, first_index, with_log_prob,
                   device)


def beta_sample(concentration1, concentration0, low, high, n, seed, offset, first_index=0, with_log_prob=False,
                device='cuda'):
    return _sample(EVENT_FAMILIES['Beta'], (concentration1, concentration0, low, high), n, seed, offset, first_index,
                   with_log_prob, device)


def binomial_sample(total_count, probs, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['Binomial'], (total_count, probs), n, seed, offset, first_index, with_log_prob,
                   device)


def von_mises_sample(loc, concentration, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    return _sample(EVENT_FAMILIES['VonMises'], (loc, concentration), n, seed, offset, first_index, with_log_prob,
                   device)


def categorical_sample(probs, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    p, stride, Cn = _rows(probs, n, device)
    v, lp = _out(n, device, with_log_prob)
    call('ppb_categorical_sample', ptr(p), stride, Cn, ptr(v), ptr(lp), n, seed, offset, first_index, stream())
    return (v, lp) if with_log_prob else v


def mixture_normal_sample(means, stddevs, probs, n, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    m, s, p, stride, K = _mixture_rows(means, stddevs, probs, n, device)
    v, lp = _out(n, device, with_log_prob)
    call('ppb_mixture_normal_sample', ptr(m), ptr(s), ptr(p), stride, K, ptr(v), ptr(lp), n, seed, offset,
         first_index, stream())
    return (v, lp) if with_log_prob else v


def mixture_truncated_normal_sample(means, stddevs, probs, low, high, n, seed, offset, first_index=0,
                                    with_log_prob=False, device='cuda'):
    m, s, p, stride, K = _mixture_rows(means, stddevs, probs, n, device)
    lo, lop, los = _param(low, n, device)
    hi, hip, his = _param(high, n, device)
    v, lp = _out(n, device, with_log_prob)
    call('ppb_mixture_truncated_normal_sample', ptr(m), ptr(s), ptr(p), stride, K, lop, los, hip, his, ptr(v),
         ptr(lp), n, seed, offset, first_index, stream())
    return (v, lp) if with_log_prob else v


# ---- event-shaped sites (C-ABI section 2b): D elements per particle ---------------------------------------------------

EVENT_MAX_D = 1 << 24          # element index: Philox counter bits 40 .. 63
EVENT_MAX_PARTICLES = 1 << 40  # particle index: Philox counter bits 0 .. 39


def _event_operand(x, n, D, device):
    """An operand of an event kernel -> (tensor kept alive, pointer, particle stride, element stride).

    x is a python scalar or 1-element tensor (shared scalar: (0, 0)), or a 2-D tensor: [n, 1] one per particle (1, 0),
    [1, D] or an [n, D] view with row stride 0 one shared event (0, 1), [n, D] one event per particle (D, 1)."""
    if not torch.is_tensor(x) or x.numel() == 1:
        t = _f32(x, device)
        return t, ptr(t), 0, 0
    t = x if (x.is_cuda and x.dtype == torch.float32) else x.to(device=device, dtype=torch.float32)
    if t.dim() != 2:
        raise ValueError('event operand must be a scalar or 2-D, got shape {}'.format(tuple(t.shape)))
    r, c = t.shape
    if c == 1 and r == n:
        t = t.reshape(n).contiguous()
        return t, ptr(t), 1, 0
    if c != D or r not in (1, n):
        raise ValueError('event operand of shape {} for n = {}, D = {}'.format(tuple(t.shape), n, D))
    if r == 1 or t.stride(0) == 0:
        row = t[0]
        if row.stride(0) != 1:
            row = row.contiguous()
        return row, ptr(row), 0, 1
    if t.stride(1) != 1 or t.stride(0) != D:
        t = t.contiguous()
    return t, ptr(t), D, 1


def _event_params(family, params, n, D, device):
    np_ = EVENT_NUM_PARAMS[family]
    if len(params) != np_:
        raise ValueError('family {} takes {} parameters, got {}'.format(family, np_, len(params)))
    held = [_event_operand(p, n, D, device) for p in params]
    args = []
    for k in range(4):
        args += [held[k][1], held[k][2], held[k][3]] if k < np_ else [None, 0, 0]
    return held, args


def event_log_prob(family, value, params, n, D, lp_out=None, acc=None, acc_scale=1.0, device='cuda'):
    """sum_j log p(value_ij) of an event site: acc[i] += acc_scale * row sum (fp64), and / or the element-wise
    log-densities lp_out [n, D] (allocated and returned when acc is None).  value / params are event operands (see
    _event_operand)."""
    n, D = int(n), int(D)
    v = _event_operand(value, n, D, device)
    held, args = _event_params(family, params, n, D, device)
    if lp_out is None and acc is None:
        lp_out = torch.empty(n, D, dtype=torch.float32, device=device)
    if lp_out is not None and (lp_out.dtype != torch.float32 or lp_out.numel() != n * D or not lp_out.is_contiguous()):
        raise ValueError('lp_out must be a contiguous float32 tensor of n * D elements')
    if acc is not None and (acc.dtype != torch.float64 or acc.numel() != n or not acc.is_contiguous()):
        raise ValueError('acc must be a contiguous float64 tensor of length n')
    call('ppb_event_log_prob', family, v[1], v[2], v[3], *args, n, D, ptr(lp_out), ptr(acc), float(acc_scale), stream())
    return lp_out


def event_sample(family, params, n, D, seed, offset, first_index=0, with_log_prob=False, device='cuda'):
    """[n, D] draws (element j of particle i from Philox index (first_index + i) | (j << 40)) and, with_log_prob, the
    event-summed log-density of each row [n]."""
    n, D = int(n), int(D)
    if not 1 <= D <= EVENT_MAX_D:
        raise ValueError('event size D = {} outside [1, 2^24]'.format(D))
    if first_index < 0 or first_index + n > EVENT_MAX_PARTICLES:
        raise ValueError('particle indices [{}, {}) outside [0, 2^40)'.format(first_index, first_index + n))
    held, args = _event_params(family, params, n, D, device)
    v = torch.empty(n, D, dtype=torch.float32, device=device)
    lp = torch.empty(n, dtype=torch.float32, device=device) if with_log_prob else None
    call('ppb_event_sample', family, *args, ptr(v), ptr(lp), n, D, seed, offset, first_index, stream())
    return (v, lp) if with_log_prob else v


# ---- importance weights -----------------------------------------------------------------------------

def weights_cast(acc):
    """fp64 accumulators -> (fp32 log weights, uint8 invalid mask)."""
    n = acc.numel()
    w = torch.empty(n, dtype=torch.float32, device=acc.device)
    bad = torch.empty(n, dtype=torch.uint8, device=acc.device)
    call('ppb_weights_cast', ptr(acc), ptr(w), ptr(bad), n, stream())
    return w, bad


def weights_partials(log_w):
    n = log_w.numel()
    nb = _lib.call('ppb_weights_num_partials', n)
    part = torch.empty(3 * nb, dtype=torch.float64, device=log_w.device)
    call('ppb_weights_partials', ptr(log_w), n, ptr(part), stream())
    return part


def weights_finalize(log_w, partials=None, want_logits=True):
    """-> (stats[4] = (logsumexp, ESS, max, sum exp(w-max)), normalised fp64 logits or None)."""
    log_w = log_w.contiguous()
    n = log_w.numel()
    if partials is None:
        partials = weights_partials(log_w)
    stats = torch.empty(4, dtype=torch.float64, device=log_w.device)
    logits = torch.empty(n, dtype=torch.float64, device=log_w.device) if want_logits else None
    call('ppb_weights_finalize', ptr(log_w), n, ptr(partials), partials.numel() // 3, ptr(stats), ptr(logits),
         stream())
    return stats, logits


# ---- Metropolis-Hastings chains (C-ABI section 7); `t` is a pyprob_b200.mcmc.Chains ---------------------------------

def mh_select(t, initial, seed, offset):
    call('ppb_mh_select', ptr(t.stamp), ptr(t.buf), ptr(t.cur_stamp), t.C, t.lda, t.ncols, ptr(t.choice), ptr(t.cand_n),
         ptr(t.cand_lpo), ptr(t.reuse), ptr(t.trans), int(initial), seed, offset, stream())


def mh_fetch(t, col, mask, n, first):
    old_v = torch.empty(n, dtype=torch.float32, device='cuda')
    old_lp = torch.empty(n, dtype=torch.float32, device='cuda')
    has = torch.empty(n, dtype=torch.uint8, device='cuda')
    call('ppb_mh_fetch', ptr(t.val), ptr(t.lp), ptr(t.stamp), ptr(t.buf), ptr(t.cur_stamp), t.C, t.lda, col, ptr(mask),
         n, first, ptr(old_v), ptr(old_lp), ptr(has), stream())
    return old_v, old_lp, has


def mh_site(t, kind, col, mask, n, first, fresh_v, fresh_lp, old_v, old_lp, has, rescored, p0, p1, seed, offset):
    """-> the value the program sees at this statement, [n] fp32"""
    out = torch.empty(n, dtype=torch.float32, device='cuda')
    a, ap, as_ = _param(p0 if p0 is not None else 0.0, n, 'cuda')
    b, bp, bs = _param(p1 if p1 is not None else 0.0, n, 'cuda')
    call('ppb_mh_site', kind, col, ptr(mask), n, first, ptr(fresh_v), ptr(fresh_lp), ptr(old_v), ptr(old_lp), ptr(has),
         ptr(rescored), ap, as_, bp, bs, ptr(t.val), ptr(t.lp), ptr(t.stamp), ptr(t.reused), ptr(t.buf), ptr(t.choice),
         t.step, t.C, t.lda, ptr(t.cand_n), ptr(t.reuse), ptr(t.trans), ptr(t.reused_count), ptr(out), seed, offset,
         stream())
    return out


def mh_accept(t, initial, slot, seed, offset):
    call('ppb_mh_accept', t.C, int(initial), t.step, ptr(t.buf), ptr(t.cur_stamp), ptr(t.cur_n), ptr(t.cur_lpo),
         ptr(t.cand_n), ptr(t.cand_lpo), ptr(t.reuse), ptr(t.trans), ptr(t.log_alpha), ptr(t.accepted),
         ptr(t.sites_all), ptr(t.cand_map), ptr(t.cur_map), t.map_words, ptr(t.out), slot, seed, offset, stream())


# ---- MCMC diagnostics (C-ABI section 8); x is a CUDA tensor [S, C, V], fp32 or fp64, any strides ---------------------

def _diag_args(x):
    if x.dim() != 3 or x.dtype not in (torch.float32, torch.float64):
        raise ValueError('diagnostics kernels take a [S, C, V] fp32 or fp64 tensor, got {} {}'.format(
            tuple(x.shape), x.dtype))
    dtype = 0 if x.dtype == torch.float32 else 1
    return (ptr(x), dtype) + tuple(x.shape) + tuple(x.stride())


def _host_i64(a):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.int64).reshape(-1))
    return a, a.ctypes.data_as(ctypes.c_void_p)


def diag_rhat(x, iters):
    """R-hat of every variable at every prefix length in iters (host ints >= 1) -> fp64 CUDA tensor [V, len(iters)]."""
    S, Cn, V = x.shape
    it, it_p = _host_i64(iters)
    nbytes = _lib.call('ppb_diag_rhat_workspace_bytes', S, Cn, V, it_p, len(it))
    if nbytes < 0:
        raise ValueError('ppb_diag_rhat: invalid arguments (S = {}, C = {}, V = {}, iters = {})'.format(S, Cn, V, it))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    out = torch.empty(V, len(it), dtype=torch.float64, device=x.device)
    call('ppb_diag_rhat', *_diag_args(x), it_p, len(it), ptr(out), ptr(ws), nbytes, stream())
    return out


def diag_autocorr(x, lags):
    """Autocorrelation of every chain of every variable at lags (host ints in [0, S]) -> fp64 CUDA tensor
    [V, C, len(lags)]."""
    S, Cn, V = x.shape
    lg, lg_p = _host_i64(lags)
    nbytes = _lib.call('ppb_diag_autocorr_workspace_bytes', _diag_args(x)[1], S, Cn, V, len(lg))
    if nbytes < 0:
        raise ValueError('ppb_diag_autocorr: invalid arguments (S = {}, C = {}, V = {})'.format(S, Cn, V))
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    out = torch.empty(V, Cn, len(lg), dtype=torch.float64, device=x.device)
    call('ppb_diag_autocorr', *_diag_args(x), lg_p, len(lg), ptr(out), ptr(ws), nbytes, stream())
    return out
