"""Data-parallel plumbing (torch.distributed): the ONE collective of the training step and the particle
sharding helpers.  The all-reduce helpers are pure torch and device-agnostic — the same code runs over NCCL on
the GPUs and over gloo in the CPU tests (tests/test_parallel_gloo.py).  On one NVLink node the training step uses
``PeerAdam`` instead: the gradient exchange and the optimiser fused into one kernel over peer memory.

Reference semantics (pyprob/nn/inference_network.py:296-333, :448, :529-530): every rank draws its own
minibatch, gradients are summed over ranks and divided by the world size, the loss is averaged, the learning
rate is scaled by sqrt(world).  The reference needs a presence map and one message per parameter tensor; with a
flat arena (absent gradients are zeros at fixed offsets) a single all-reduce carries everything.
"""
import ctypes as C
import math

import torch
import torch.distributed as dist


def world_info():
    if dist.is_available() and dist.is_initialized():
        return dist.get_world_size(), dist.get_rank()
    return 1, 0


def allreduce_grad_and_loss(grad_flat, loss):
    """Sum the flat gradient arena over ranks in place (loss scalar piggy-backed).

    Returns (mean loss as float, grad_scale) — grad_scale = 1/world is folded into the optimiser kernel
    (the grad_scale slot of the optimiser's hyper vector) instead of a separate divide pass."""
    world, _ = world_info()
    if world == 1:
        return float(loss), 1.0
    packed = torch.cat([grad_flat.reshape(-1), loss.detach().reshape(1).to(grad_flat.dtype)])
    dist.all_reduce(packed)
    grad_flat.copy_(packed[:-1].view_as(grad_flat))
    return float(packed[-1]) / world, 1.0 / world


def scaled_learning_rate(lr, world):
    return lr * math.sqrt(world)


def shard_range(n, rank, world):
    """Contiguous particle range [first, first+count) of rank `rank` (remainder spread over the low ranks)."""
    base, rem = divmod(n, world)
    count = base + (1 if rank < rem else 0)
    first = rank * base + min(rank, rem)
    return first, count


def gather_weight_partials(partials):
    """All-gather the per-block (max, sum exp, sum exp^2) triples of every rank -> one list that
    ppb_weights_finalize combines exactly (SURVEY 8e).  Ranks may hold different numbers of triples."""
    world, _ = world_info()
    if world == 1:
        return partials
    n_local = torch.tensor([partials.numel()], dtype=torch.int64, device=partials.device)
    sizes = [torch.zeros_like(n_local) for _ in range(world)]
    dist.all_gather(sizes, n_local)
    m = int(max(int(s) for s in sizes))
    padded = torch.zeros(m, dtype=partials.dtype, device=partials.device)
    padded[:partials.numel()] = partials
    bufs = [torch.zeros_like(padded) for _ in range(world)]
    dist.all_gather(bufs, padded)
    return torch.cat([b[:int(s)] for b, s in zip(bufs, sizes)])


class _RawDeviceMemory:
    """Adapter that lets torch.as_tensor wrap a raw device allocation without copying."""

    def __init__(self, address, nbytes):
        self.__cuda_array_interface__ = {'shape': (int(nbytes),), 'typestr': '|u1', 'data': (int(address), False),
                                         'version': 2}


class PeerAdam:
    """Data-parallel Adam fused with its collective over NVLink peer memory (``ppb_dp_adam_step``).

    Replaces ``allreduce_grad_and_loss`` + ``ppb_adam_step_dev`` when all ranks sit on one NVLink node: the gradient
    is reduce-scattered by peer loads, Adam runs on the owning rank's slice only, and the updated parameters
    are all-gathered by peer stores — one kernel, two NVLink crossings per element, no NCCL on the step.

    Every rank allocates one peer block (``ppb_dp_alloc``), the CUDA IPC handles are exchanged through
    torch.distributed, and each rank maps the others' blocks (``ppb_dp_open``).  ``params`` (float[n]) and
    ``grad`` (float[n + N_EXTRA], the tail carries piggy-backed scalars such as the loss) are tensor views of
    the local block: the network's arena must live in ``params`` and the backward pass must write ``grad``.
    """
    N_EXTRA = 8

    def __init__(self, n, device):
        from . import _lib
        self.world, self.rank = world_info()
        self.n = int(n)
        pad = lambda x: (x + 63) // 64 * 64
        self.param_off = 0
        self.grad_off = pad(self.n) * 4
        self.flag_off = self.grad_off + pad(self.n + self.N_EXTRA) * 4
        nbytes = self.flag_off + 512
        own = C.c_void_p()
        handle = C.create_string_buffer(64)
        _lib.call('ppb_dp_alloc', nbytes, C.byref(own), handle)
        handles = [handle.raw]
        if self.world > 1:
            handles = [None] * self.world
            dist.all_gather_object(handles, handle.raw)
        self._own = own.value
        self._blocks = (C.c_void_p * self.world)()
        self._mapped = []
        for r in range(self.world):
            if r == self.rank:
                self._blocks[r] = self._own
            else:
                q = C.c_void_p()
                _lib.call('ppb_dp_open', handles[r], C.byref(q))
                self._blocks[r] = q.value
                self._mapped.append(q.value)
        raw = torch.as_tensor(_RawDeviceMemory(self._own, nbytes), device=device)
        self._raw = raw
        self.params = raw[:self.n * 4].view(torch.float32)
        self.grad = raw[self.grad_off:self.grad_off + (self.n + self.N_EXTRA) * 4].view(torch.float32)
        self._flags = raw[self.flag_off:self.flag_off + 512].view(torch.int32)
        if self.world > 1:
            dist.barrier()   # every block is mapped (and zeroed) before anyone's first step

    def step(self, exp_avg, exp_avg_sq, hyper_dev, state_dev, stream):
        """hyper_dev: the Adam slots of the hyper vector, grad_scale = 1/world; state_dev: the Adam state block
        (both in include/pyprob_b200.h)."""
        from . import _lib
        _lib.call('ppb_dp_adam_step', self.world, self.rank, self._blocks, self.param_off, self.grad_off,
                  self.flag_off, _lib.ptr(exp_avg), _lib.ptr(exp_avg_sq), self.n, self.N_EXTRA, _lib.ptr(hyper_dev),
                  _lib.ptr(state_dev), stream)

    def rendezvous(self, stream):
        """Stream-ordered cross-rank rendezvous (ppb_dp_rendezvous): later work on `stream` starts together on all ranks."""
        from . import _lib
        _lib.call('ppb_dp_rendezvous', self.world, self.rank, self._blocks, self.flag_off, stream)

    def phase_totals_us(self, reset=False):
        """Mean durations (us) of the phases of ppb_dp_adam_step over the launches since the last reset: wait at barrier A
        (cross-rank skew of the backward passes), slice (peer loads + Adam + peer stores), wait at barrier B."""
        acc = [int(x) & 0xffffffff for x in self._flags[44:48].tolist()]
        n = max(acc[3], 1)
        out = {'launches': acc[3], 'barrier_a': acc[0] * 1e-3 / n, 'slice': acc[1] * 1e-3 / n,
               'barrier_b': acc[2] * 1e-3 / n}
        if reset:
            self._flags[44:48].zero_()
        return out

    def timed_out(self):
        """True if a cross-rank barrier gave up waiting (a rank died or fell out of step)."""
        return bool(int(self._flags[34]) != 0)

    def phase_trace_us(self):
        """Durations (us) of the last step's phases on this rank: barrier A, slice (reduce + Adam + peer
        stores + fence, block 0), barrier B (until the last block leaves)."""
        t = [int(x) & 0xffffffff for x in self._flags[40:44].tolist()]
        d = [((t[i + 1] - t[i]) & 0xffffffff) * 1e-3 for i in range(3)]
        return {'barrier_a': d[0], 'slice': d[1], 'barrier_b': d[2]}

    def close(self):
        from . import _lib
        torch.cuda.synchronize()
        if self.world > 1:
            dist.barrier()
        for q in self._mapped:
            _lib.call('ppb_dp_close', q)
        self._mapped = []
        self.params = self.grad = self._flags = self._raw = None
        if self._own:
            _lib.call('ppb_dp_free', self._own)
            self._own = None
