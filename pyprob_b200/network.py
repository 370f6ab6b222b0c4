"""InferenceNetworkLSTM and InferenceNetworkFeedForward — host-side mirrors of the reference network classes for the CUDA
hot path.

Same constructor keywords, attributes and method names as the reference (pyprob/nn/inference_network.py:24-78,
pyprob/nn/inference_network_lstm.py:13-27, pyprob/nn/inference_network_feedforward.py:13-19) so that
``Model.learn_inference_network`` / ``posterior_results`` drive it unchanged, but:

* all parameters live in ONE flat fp32 arena on the GPU (``_arena``), indexed by the reference's own
  state_dict key names (``parameter_index``), so reference checkpoints load verbatim;
* ``_loss`` encodes the minibatch into index tensors and calls the C-ABI forward/backward
  (include/pyprob_b200.h section 4) through one ``torch.autograd.Function``;
* the optimiser is the fused flat-arena Adam kernel (``ppb_adam_step``);
* there is no CPU execution path: every method raises without a CUDA device + the native library.
"""
import ctypes as C
import math
import os
import time
import warnings
from collections import OrderedDict

import numpy as np
import torch
import torch.nn as nn

from . import _lib, ops, parallel, util
from ._lib import call, ptr, stream
from .encoding import EncodedBatch
from .util import InferenceNetwork as InferenceNetworkType  # noqa: F401
from .util import LearningRateScheduler, ObserveEmbedding, Optimizer

_OPTIMIZER_KIND = {Optimizer.ADAM: 0, Optimizer.ADAM_LARC: 1, Optimizer.SGD: 2, Optimizer.SGD_LARC: 3}

FAMILY_NORMAL, FAMILY_UNIFORM, FAMILY_POISSON, FAMILY_CATEGORICAL, FAMILY_BERNOULLI = 0, 1, 2, 3, 4
_FAMILY_OF = {'Normal': FAMILY_NORMAL, 'Uniform': FAMILY_UNIFORM, 'Poisson': FAMILY_POISSON,
              'Categorical': FAMILY_CATEGORICAL, 'Bernoulli': FAMILY_BERNOULLI}
MAX_OBS, MAX_FF_LAYERS = 8, 4


# ---- ctypes mirrors of the ABI structs (sizes are cross-checked against ppb_sizeof) ---------------------
class LinearDesc(C.Structure):
    _fields_ = [('in_dim', C.c_int32), ('out_dim', C.c_int32), ('w_off', C.c_int64), ('b_off', C.c_int64)]


class FFDesc(C.Structure):
    _fields_ = [('num_layers', C.c_int32), ('in_dim', C.c_int32), ('out_dim', C.c_int32),
                ('layers', LinearDesc * MAX_FF_LAYERS)]


class NetDesc(C.Structure):
    _fields_ = [('lstm_dim', C.c_int32), ('obs_dim', C.c_int32), ('sample_dim', C.c_int32), ('addr_dim', C.c_int32),
                ('type_dim', C.c_int32), ('mixture_k', C.c_int32), ('num_obs', C.c_int32), ('obs_in_total', C.c_int32),
                ('obs_ff', FFDesc * MAX_OBS), ('obs_final', FFDesc),
                ('w_ih_off', C.c_int64), ('w_hh_off', C.c_int64), ('b_ih_off', C.c_int64), ('b_hh_off', C.c_int64),
                ('network_type', C.c_int32), ('reserved_', C.c_int32)]


NET_LSTM, NET_FEEDFORWARD = 0, 1   # ppb_net_desc.network_type


class AddrDesc(C.Structure):
    _fields_ = [('family', C.c_int32), ('num_categories', C.c_int32), ('head_hidden', C.c_int32),
                ('head_out', C.c_int32), ('smp_in', C.c_int32), ('type_id', C.c_int32),
                ('addr_emb_off', C.c_int64), ('smp_w_off', C.c_int64), ('smp_b_off', C.c_int64),
                ('w1_off', C.c_int64), ('b1_off', C.c_int64), ('w2_off', C.c_int64), ('b2_off', C.c_int64)]


class BatchStruct(C.Structure):  # opaque storage for ppb_batch (filled by ppb_batch_from_image)
    _fields_ = [('raw', C.c_uint8 * 256)]


def check_abi_struct_sizes():
    sizes = {0: C.sizeof(NetDesc), 1: C.sizeof(AddrDesc), 3: C.sizeof(FFDesc), 4: C.sizeof(LinearDesc)}
    for which, sz in sizes.items():
        native = _lib.call('ppb_sizeof', which)
        if native != sz:
            raise RuntimeError('ABI struct {} size mismatch: ctypes {} vs native {}'.format(which, sz, native))
    if _lib.call('ppb_sizeof', 2) > C.sizeof(BatchStruct):
        raise RuntimeError('ppb_batch is larger than its Python storage')


class _LossFunction(torch.autograd.Function):
    """loss = network._forward_native(batch); backward fills the flat gradient arena."""

    @staticmethod
    def forward(ctx, arena, net, enc):
        loss = net._forward_native(enc, want_grad=True)
        ctx.net, ctx.enc = net, enc
        return loss

    @staticmethod
    def backward(ctx, grad_out):
        net = ctx.net
        grad = torch.zeros_like(net._arena.data)
        net._backward_native(ctx.enc, grad, float(grad_out))
        return grad, None, None


class InferenceNetwork(nn.Module):
    """What does not depend on the network type (reference pyprob/nn/inference_network.py): the parameter arena, the
    observation layers, the loss call, the optimisers and the training loop, data-parallel training, checkpoints,
    workspaces and `_infer_init`.  Subclasses add the proposal layers of an address (`_add_address`), the native
    network description (`_fill_net_desc`, `_fill_addr_desc`), the infer step and `_segment_presence`."""

    def __init__(self, model=None, observe_embeddings={}, proposal_mixture_components=10, precision=0,
                 network_type=''):
        super().__init__()
        self._model = model
        self._network_type = network_type
        self._observe_embeddings = observe_embeddings
        self._observe_embedding_dim = None
        self._observe_names = []
        self._observe_in_dims = []
        self._proposal_mixture_components = proposal_mixture_components
        self._precision = precision
        self._layers_initialized = False
        self._layers_pre_generated = False
        # flat arena + index (reference state_dict names -> (offset, shape))
        self.parameter_index = OrderedDict()
        self._arena_used = 0
        self._arena_store = None          # capacity-sized device tensor
        self._arena = None                # nn.Parameter view of the used prefix
        self._addresses = OrderedDict()   # address -> info dict (insertion order = address id)
        self._types = OrderedDict()       # distribution name -> type id
        self._head_iterations = {}        # address -> _total_train_iterations of its proposal layer
        self._obs_ff = []                 # per observable: list of (in, out, w_name, b_name)
        self._final_ff = []
        # optimiser state
        self._optimizer_type = None
        self._optimizer_step = 0
        self._exp_avg = None
        self._exp_avg_sq = None
        self._peer = None                 # parallel.PeerAdam when training data-parallel over NVLink
        self._seg = None                  # device tables of the segment-aware optimiser step (LARC / SGD / skipping)
        self._skip_absent_gradients = False   # True: tensors absent from a minibatch are skipped like .grad None
        # Optimizer.ADAM hands over to the skipping step by itself when the flat kernel would differ from torch.optim
        # (_maybe_switch_to_segmented); PPB_FLAT_ADAM=1 keeps the flat kernel (absent gradient = zeros) throughout
        self._auto_skip_absent = os.environ.get('PPB_FLAT_ADAM') != '1'
        self._last_enc = None
        self._learning_rate_init = None
        self._learning_rate_end = None
        self._learning_rate_scheduler_type = None
        self._learning_rate = None
        self._momentum = None
        self._weight_decay = None
        self._adam_betas = (0.9, 0.999)
        self._adam_eps = 1e-8
        # bookkeeping the reference's diagnostics read (pyprob/diagnostics.py:336-372)
        self._total_train_seconds = 0
        self._total_train_traces = 0
        self._total_train_traces_end = None
        self._total_train_iterations = 0
        self._loss_init = None
        self._loss_min = float('inf')
        self._loss_max = None
        self._loss_previous = float('inf')
        self._history_train_loss = []
        self._history_train_loss_trace = []
        self._history_valid_loss = []
        self._history_valid_loss_trace = []
        self._history_num_params = []
        self._history_num_params_trace = []
        self._distributed_backend = None
        self._distributed_world_size = None
        self._modified = util.get_time_str()
        self._updates = 0
        self._on_cuda = True
        self._device = torch.device('cuda')
        # native handles (not pickled)
        self._handle = None
        self._tables_dirty = True
        self._workspace = None
        self._image_dev = None
        self._image_host = None
        self._loss_buf = None
        # inference state
        self._infer_observe = None
        self._infer_observe_embedding = None

    # ------------------------------------------------------------------------------------------------
    # arena management
    # ------------------------------------------------------------------------------------------------
    def _alloc(self, name, shape, init):
        """Append a parameter region (16-byte aligned) initialised from the CPU tensor `init`."""
        n = int(np.prod(shape))
        off = (self._arena_used + 3) // 4 * 4
        need = off + n
        dev = torch.device('cuda')
        if self._arena_store is None or need > self._arena_store.numel():
            cap = max(need * 2, 1 << 16)
            new = torch.zeros(cap, dtype=torch.float32, device=dev)
            if self._arena_store is not None:
                new[:self._arena_used] = self._arena_store[:self._arena_used]
            self._arena_store = new
        self._arena_store[off:off + n] = init.detach().reshape(-1).to(device=dev, dtype=torch.float32)
        self._arena_used = need
        self.parameter_index[name] = (off, tuple(shape))
        self._tables_dirty = True
        return off

    def _rebind(self):
        self._arena = nn.Parameter(self._arena_store[:self._arena_used])
        self._exp_avg = None
        self._exp_avg_sq = None

    def view(self, name):
        off, shape = self.parameter_index[name]
        return self._arena.data[off:off + int(np.prod(shape))].view(shape)

    def grad_view(self, name, grad=None):
        g = self._arena.grad if grad is None else grad
        off, shape = self.parameter_index[name]
        return g[off:off + int(np.prod(shape))].view(shape)

    def reference_state_dict(self):
        """Parameters under the reference's state_dict key names (clones)."""
        return OrderedDict((k, self.view(k).clone()) for k in self.parameter_index)

    def load_reference_state_dict(self, sd):
        for k in self.parameter_index:
            if k not in sd:
                raise KeyError('missing parameter {}'.format(k))
            self.view(k).copy_(sd[k].to(device='cuda', dtype=torch.float32))

    def _linear(self, prefix, in_dim, out_dim):
        ref = nn.Linear(in_dim, out_dim)  # reference init law (embedding_feedforward.py:24-30)
        self._alloc(prefix + '.weight', (out_dim, in_dim), ref.weight)
        self._alloc(prefix + '.bias', (out_dim,), ref.bias)

    def _ff(self, prefix, in_dim, out_dim, num_layers):
        """EmbeddingFeedForward layout (embedding_feedforward.py:8-33) -> list of (in, out, w_name, b_name)."""
        dims = []
        if num_layers == 1:
            dims.append((in_dim, out_dim))
        else:
            hidden = int((in_dim + out_dim) / 2)
            dims.append((in_dim, hidden))
            for _ in range(num_layers - 2):
                dims.append((hidden, hidden))
            dims.append((hidden, out_dim))
        if len(dims) > MAX_FF_LAYERS:
            raise NotImplementedError('feed-forward embeddings deeper than {} layers'.format(MAX_FF_LAYERS))
        out = []
        for i, (a, b) in enumerate(dims):
            p = '{}._layers.{}'.format(prefix, i)
            self._linear(p, a, b)
            out.append((a, b, p + '.weight', p + '.bias'))
        return out

    # ------------------------------------------------------------------------------------------------
    # layer construction (reference: inference_network.py:80-130, inference_network_lstm.py:29-80)
    # ------------------------------------------------------------------------------------------------
    def _init_layers_observe_embedding(self, observe_embeddings, example_trace):
        if len(observe_embeddings) == 0:
            raise ValueError('At least one observe embedding is needed to initialize inference network.')
        if isinstance(observe_embeddings, set):
            observe_embeddings = {o: {} for o in observe_embeddings}
        if len(observe_embeddings) > MAX_OBS:
            raise NotImplementedError('more than {} observables'.format(MAX_OBS))
        total = 0
        for name, value in observe_embeddings.items():
            variable = example_trace.named_variables[name]
            if 'reshape' in value:
                in_dim = int(np.prod(value['reshape']))
            else:
                in_dim = int(np.prod(example_trace.value_shape(variable)))
            out_dim = int(value.get('dim', 256))
            embedding = value.get('embedding', ObserveEmbedding.FEEDFORWARD)
            if embedding != ObserveEmbedding.FEEDFORWARD:
                raise NotImplementedError('pyprob_b200: only ObserveEmbedding.FEEDFORWARD is implemented '
                                          '(CNN embeddings are a "next" row, SURVEY.md 8f)')
            depth = int(value.get('depth', 2))
            self._obs_ff.append(self._ff('_layers_observe_embedding.{}'.format(name), in_dim, out_dim, depth))
            self._observe_names.append(name)
            self._observe_in_dims.append(in_dim)
            total += out_dim
        self._observe_embedding_dim = total
        self._final_ff = self._ff('_layers_observe_embedding_final', total, total, 2)

    def _init_layers(self):
        self._rebind()

    def _proposal_layers(self, address, family, num_categories, in_dim):
        """The proposal head of an address (proposal_*.py: EmbeddingFeedForward(in_dim -> out, 2 layers)) -> its info."""
        K = self._proposal_mixture_components
        # proposal_categorical_categorical.py: C logits; proposal_bernoulli_bernoulli.py: one logit; mixtures: 3K
        out = num_categories if family == FAMILY_CATEGORICAL else 1 if family == FAMILY_BERNOULLI else 3 * K
        hidden = int((in_dim + out) / 2)
        p = '_layers_proposal.{}._ff._layers'.format(address)
        self._linear(p + '.0', in_dim, hidden)
        self._linear(p + '.1', hidden, out)
        return dict(head_hidden=hidden, head_out=out)

    def _ensure_initialized(self, example_trace):
        if not self._layers_initialized:
            _lib.require_cuda()
            self._init_layers_observe_embedding(self._observe_embeddings, example_trace)
            self._init_layers()
            self._layers_initialized = True

    def _polymorph(self, batch):
        """Create layers for addresses not seen before; returns True if the network changed."""
        changed = False
        for address, dist_name, num_categories in batch.address_signature():
            if address not in self._addresses:
                self._add_address(address, dist_name, num_categories)
                changed = True
        if changed:
            self._rebind()
            num_params = sum(int(np.prod(s)) for _, s in self.parameter_index.values())
            print('Total addresses: {:,}, distribution types: {:,}, parameters: {:,}'.format(
                len(self._addresses), len(self._types), num_params))
            self._history_num_params.append(num_params)
            self._history_num_params_trace.append(self._total_train_traces)
        return changed

    @property
    def row_align(self):
        """Row layout the native path expects: 128-row segments on the tensor cores, compact rows on the SIMT path."""
        return 1 if self._precision == 2 else 128

    def num_parameters(self):
        return sum(int(np.prod(s)) for _, s in self.parameter_index.values())

    # ------------------------------------------------------------------------------------------------
    # native handle / tables
    # ------------------------------------------------------------------------------------------------
    def _ff_desc(self, layers):
        d = FFDesc()
        d.num_layers = len(layers)
        d.in_dim, d.out_dim = layers[0][0], layers[-1][1]
        for i, (a, b, wn, bn) in enumerate(layers):
            d.layers[i].in_dim, d.layers[i].out_dim = a, b
            d.layers[i].w_off, d.layers[i].b_off = self.parameter_index[wn][0], self.parameter_index[bn][0]
        return d

    def _sync_native(self):
        if self._handle is None:
            check_abi_struct_sizes()
            nd = NetDesc()
            nd.obs_dim, nd.mixture_k = self._observe_embedding_dim, self._proposal_mixture_components
            nd.num_obs, nd.obs_in_total = len(self._obs_ff), int(sum(self._observe_in_dims))
            for j, layers in enumerate(self._obs_ff):
                nd.obs_ff[j] = self._ff_desc(layers)
            nd.obs_final = self._ff_desc(self._final_ff)
            self._fill_net_desc(nd)
            h = C.c_void_p()
            call('ppb_net_create', C.byref(h), C.byref(nd))
            self._handle = h
            self._tables_dirty = True
        if self._tables_dirty and len(self._addresses) > 0:
            n = len(self._addresses)
            arr = (AddrDesc * n)()
            for address, info in self._addresses.items():
                a = arr[info['id']]
                a.family, a.num_categories = info['family'], info['num_categories']
                a.head_hidden, a.head_out, a.smp_in = info['head_hidden'], info['head_out'], info['smp_in']
                pi = self.parameter_index
                self._fill_addr_desc(a, address, info)
                a.w1_off = pi['_layers_proposal.{}._ff._layers.0.weight'.format(address)][0]
                a.b1_off = pi['_layers_proposal.{}._ff._layers.0.bias'.format(address)][0]
                a.w2_off = pi['_layers_proposal.{}._ff._layers.1.weight'.format(address)][0]
                a.b2_off = pi['_layers_proposal.{}._ff._layers.1.bias'.format(address)][0]
            toff = (C.c_int64 * len(self._types))()
            for name, tid in self._types.items():
                toff[tid] = self.parameter_index['_layers_distribution_type_embedding.{}'.format(name)][0]
            call('ppb_net_set_tables', self._handle, arr, n, toff if len(self._types) else None, len(self._types),
                 self._arena_used)
            self._tables_dirty = False

    def __getstate__(self):
        st = self.__dict__.copy()
        for k in ('_handle', '_workspace', '_image_dev', '_image_host', '_loss_buf', '_model',
                  '_infer_observe_embedding', '_peer', '_peer_hyper', '_peer_state', '_seg', '_last_enc'):
            st[k] = None
        if self._peer is not None:   # the arena lives in an NVLink peer block: pickle a private copy
            st['_arena_store'] = self._arena_store.clone()
            st['_arena'] = nn.Parameter(st['_arena_store'][:self._arena_used])
        st['_tables_dirty'] = True
        return st

    def __del__(self):
        try:
            if getattr(self, '_handle', None) is not None:
                _lib.call('ppb_net_destroy', self._handle)
        except Exception:
            pass

    # ------------------------------------------------------------------------------------------------
    # loss (reference: inference_network_lstm.py:136-220)
    # ------------------------------------------------------------------------------------------------
    def _stage_batch(self, enc):
        """Pack the batch image into pinned host memory, copy to the device, decode into a ppb_batch."""
        offs, total = enc.offsets()
        if self._image_host is None or self._image_host.numel() < total:
            self._image_host = torch.empty(max(total * 2, 1 << 16), dtype=torch.uint8).pin_memory()
            self._image_dev = torch.empty(self._image_host.numel(), dtype=torch.uint8, device='cuda')
        img = enc.pack(out=self._image_host.numpy())
        self._image_dev[:total].copy_(self._image_host[:total], non_blocking=True)
        bs = BatchStruct()
        call('ppb_batch_from_image', self._image_host.data_ptr(), self._image_dev.data_ptr(), total, C.byref(bs))
        return bs, total

    def _ensure_workspace(self, enc):
        need = _lib.call('ppb_ic_workspace_bytes', self._handle, enc.n_traces, enc.n_rows, enc.t_max, enc.n_steps,
                         enc.n_groups) + 512
        if self._workspace is None or self._workspace.numel() < need:
            self._workspace = torch.empty(int(need * 1.25), dtype=torch.uint8, device='cuda')
        if self._loss_buf is None:
            self._loss_buf = torch.zeros(4, dtype=torch.float32, device='cuda')
        return need

    def _forward_native(self, enc, want_grad, row_lp=None):
        self._sync_native()
        bs, _ = self._stage_batch(enc)
        need = self._ensure_workspace(enc)
        loss = torch.empty((), dtype=torch.float32, device='cuda')
        status = self._loss_buf[1:2].view(torch.int32)
        call('ppb_ic_loss_forward', self._handle, ptr(self._arena.data), C.byref(bs), ptr(self._workspace), need,
             self._precision, ptr(loss), ptr(status), ptr(row_lp), 1 if want_grad else 0, stream())
        enc._batch_struct = bs  # keep the decoded view for backward
        self._generation = getattr(self, '_generation', 0) + 1
        enc._generation = self._generation
        self._last_status = status
        return loss

    def _backward_native(self, enc, grad, grad_scale):
        if getattr(enc, '_generation', None) != getattr(self, '_generation', 0):
            raise RuntimeError('pyprob_b200: backward() must directly follow the _loss() that produced the loss — '
                               'the activation workspace and the staged batch are shared between calls')
        need = self._ensure_workspace(enc)
        call('ppb_ic_loss_backward', self._handle, ptr(self._arena.data), ptr(grad), C.byref(enc._batch_struct),
             ptr(self._workspace), need, self._precision, grad_scale, stream())

    def _loss(self, batch):
        """-> (success, loss) like the reference; loss is a 0-d CUDA tensor attached to the arena."""
        enc = batch.encode(self)
        if enc is None:
            return False, 0
        self._last_enc = enc
        for address, _, _ in batch.address_signature():
            self._head_iterations[address] += 1
        if torch.is_grad_enabled():
            loss = _LossFunction.apply(self._arena, self, enc)
        else:
            loss = self._forward_native(enc, want_grad=False)
        if int(self._last_status.item()) != 0:  # NaN / +inf in a proposal log_prob (:214-216)
            print('Nan or Inf present in proposal log_prob.')
            return False, 0
        return True, loss

    def row_log_probs(self, batch):
        """Per-row log q (time-major row order of the encoding) — used by parity tests."""
        enc = batch.encode(self)
        lp = torch.empty(enc.n_rows, dtype=torch.float32, device='cuda')
        with torch.no_grad():
            self._forward_native(enc, want_grad=False, row_lp=lp)
        return enc, lp

    # ------------------------------------------------------------------------------------------------
    # optimiser (reference: inference_network.py:343-379, :496)
    # ------------------------------------------------------------------------------------------------
    def _create_optimizer(self, state=None):
        if self._optimizer_type is None:
            return
        if self._optimizer_type not in _OPTIMIZER_KIND:
            raise NotImplementedError('pyprob_b200: unknown optimizer type {}'.format(self._optimizer_type))
        n = self._arena.numel()
        self._exp_avg = torch.zeros(n, dtype=torch.float32, device='cuda')
        self._exp_avg_sq = torch.zeros(n, dtype=torch.float32, device='cuda')
        self._optimizer_step = 0
        self._learning_rate = self._learning_rate_init
        self._seg = None
        self._present_sig = None
        if self._optimizer_type != Optimizer.ADAM or self._skip_absent_gradients:
            self._create_segment_state()
        if state is not None:
            self._exp_avg.copy_(state['exp_avg'])
            self._exp_avg_sq.copy_(state['exp_avg_sq'])
            self._optimizer_step = state['step']
            if self._seg is not None and state.get('segment_steps') is not None:
                self._seg['steps'].copy_(state['segment_steps'])

    def _create_segment_state(self):
        """Device tables of the segment-aware optimiser step (ppb_optimizer_step_segmented): one segment per parameter
        tensor of the reference.  Needed for LARC / SGD (per-tensor norms, per-tensor first-step flag) and for the
        reference's skipping of tensors whose gradient is absent from a minibatch (`_skip_absent_gradients`)."""
        names = self._segment_names()
        n = self._arena.numel()
        seg_of_block = np.full((n + 3) // 4, -1, dtype=np.int32)
        for k, name in enumerate(names):
            off, shape = self.parameter_index[name]
            seg_of_block[off // 4:(off + int(np.prod(shape)) + 3) // 4] = k
        S = len(names)
        scratch = _lib.call('ppb_optimizer_scratch_bytes', S)
        self._seg = {'names': names, 'index': {nm: k for k, nm in enumerate(names)},
                     'seg_of_block': torch.from_numpy(seg_of_block).cuda(),
                     'steps': torch.zeros(S, dtype=torch.int64, device='cuda'),
                     'present': torch.ones(S, dtype=torch.int32, device='cuda'),
                     'scratch': torch.empty(int(scratch), dtype=torch.uint8, device='cuda'),
                     'hyper': torch.zeros(10, dtype=torch.float32, device='cuda')}

    def _segment_names(self):
        return sorted(self.parameter_index, key=lambda k: self.parameter_index[k][0])

    def _segmented_optimizer_step(self, grad_scale):
        seg = self._seg
        b1, b2 = self._adam_betas
        seg['present'].copy_(torch.from_numpy(self._segment_presence(self._last_enc)))
        world, _ = parallel.world_info()
        if world > 1 and self._skip_absent_gradients:
            # a tensor is present if any rank saw it (the reference's presence map, inference_network.py:299-311)
            import torch.distributed as dist
            dist.all_reduce(seg['present'], op=dist.ReduceOp.MAX)
        seg['hyper'].copy_(torch.tensor([float(self._learning_rate), b1, b2, self._adam_eps,
                                         float(self._weight_decay or 0.0), float(grad_scale),
                                         float(self._momentum if self._momentum is not None else 0.9),
                                         0.002, 1e-8, 1.0 / 16000.0]))
        adam = self._optimizer_type in (Optimizer.ADAM, Optimizer.ADAM_LARC)
        call('ppb_optimizer_step_segmented', ptr(self._arena.data), ptr(self._arena.grad), ptr(self._exp_avg),
             ptr(self._exp_avg_sq) if adam else None, self._arena.numel(), ptr(seg['seg_of_block']), len(seg['names']),
             ptr(seg['present']), ptr(seg['steps']), ptr(seg['scratch']), seg['scratch'].numel(),
             _OPTIMIZER_KIND[self._optimizer_type], ptr(seg['hyper']), stream())

    @property
    def _optimizer(self):
        return None if self._exp_avg is None else self

    def _current_learning_rate(self):
        t = self._learning_rate_scheduler_type
        if t in (LearningRateScheduler.POLY1, LearningRateScheduler.POLY2):
            power = 1.0 if t == LearningRateScheduler.POLY1 else 2.0
            it, end = self._total_train_traces, self._total_train_traces_end
            return (self._learning_rate_init - self._learning_rate_end) * ((1 - it / end) ** power) + \
                self._learning_rate_end
        return self._learning_rate_init

    def _maybe_switch_to_segmented(self):
        """torch.optim skips parameter tensors whose gradient is absent from a minibatch (no moment decay, no step count,
        no weight decay) — the reference's behaviour on torch >= 2.0 (inference_network.py:343-355, zero_grad sets None).
        The flat Adam kernel treats an absent gradient as zeros, which is the same thing exactly as long as (a) the set of
        absent tensors never changes and (b) weight decay is zero.  The first time either fails, training continues on the
        segment-aware step (csrc/optim.cu) with the per-tensor step counts the history implies — no difference to the
        reference is ever applied."""
        if (self._seg is not None or self._optimizer_type != Optimizer.ADAM or self._peer is not None
                or self._last_enc is None or parallel.world_info()[0] > 1 or not self._auto_skip_absent):
            return
        present = self._segment_presence(self._last_enc, force=True)
        sig = present.tobytes()
        first = getattr(self, '_present_sig', None)
        if first is None:
            self._present_sig = sig
            if present.all() or not float(self._weight_decay or 0.0):
                return
        elif sig == first:
            return
        before = np.frombuffer(self._present_sig, dtype=np.int32)
        self._skip_absent_gradients = True
        self._create_segment_state()
        steps = torch.from_numpy(before.astype(np.int64) * int(self._optimizer_step))
        self._seg['steps'].copy_(steps)

    def optimizer_step(self, grad_scale=1.0):
        self._maybe_switch_to_segmented()
        self._optimizer_step += 1
        if self._seg is not None:
            self._segmented_optimizer_step(grad_scale)
            return
        b1, b2 = self._adam_betas
        call('ppb_adam_step', ptr(self._arena.data), ptr(self._arena.grad), ptr(self._exp_avg), ptr(self._exp_avg_sq),
             self._arena.numel(), float(self._learning_rate), b1, b2, self._adam_eps, float(self._weight_decay or 0.0),
             self._optimizer_step, float(grad_scale), stream())

    def _enable_peer_optimizer(self):
        """Move the arena into this rank's NVLink peer block and switch the optimiser step to the fused
        reduce-scatter + Adam + all-gather kernel (parallel.PeerAdam).  Arena offsets are unchanged."""
        n = self._arena.numel()
        peer = parallel.PeerAdam(n, self._arena.device)
        peer.params.copy_(self._arena.data)
        self._arena_store = peer.params
        self._arena = nn.Parameter(peer.params)
        self._peer = peer
        self._peer_hyper = torch.zeros(6, dtype=torch.float32, device=peer.params.device)
        self._peer_state = torch.zeros(4, dtype=torch.int32, device=peer.params.device)
        self._peer_state.view(torch.int64)[0] = int(self._optimizer_step)

    def _peer_optimizer_step(self, loss, world):
        peer, n = self._peer, self._arena.numel()
        peer.grad[:n].copy_(self._arena.grad)
        peer.grad[n:n + 1].copy_(loss.reshape(1))
        b1, b2 = self._adam_betas
        self._peer_hyper.copy_(torch.tensor([float(self._learning_rate), b1, b2, self._adam_eps,
                                             float(self._weight_decay or 0.0), 1.0 / world]))
        peer.step(self._exp_avg, self._exp_avg_sq, self._peer_hyper, self._peer_state, stream())
        self._optimizer_step += 1
        loss_value = float(peer.grad[n]) / world
        if peer.timed_out():
            raise RuntimeError('pyprob_b200: data-parallel optimiser step timed out waiting for a peer rank')
        return loss_value

    # ------------------------------------------------------------------------------------------------
    # training loop (reference: inference_network.py:381-599)
    # ------------------------------------------------------------------------------------------------
    def optimize(self, num_traces, dataset, dataset_valid=None, num_traces_end=1e9, batch_size=64, valid_every=None,
                 optimizer_type=Optimizer.ADAM, learning_rate_init=0.0001, learning_rate_end=1e-6,
                 learning_rate_scheduler_type=LearningRateScheduler.NONE, momentum=0.9, weight_decay=1e-5,
                 save_file_name_prefix=None, save_every_sec=600, distributed_backend=None,
                 distributed_params_sync_every_iter=10000, distributed_num_buckets=10,
                 dataloader_offline_num_workers=0, stop_with_bad_loss=False, log_file_name=None):
        import torch.distributed as dist
        self._ensure_initialized(dataset.example_trace())
        if distributed_backend is None:
            world, rank = 1, 0
        else:
            if not dist.is_initialized():
                dist.init_process_group(backend=distributed_backend)
            world, rank = dist.get_world_size(), dist.get_rank()
            self._distributed_backend, self._distributed_world_size = distributed_backend, world
        self.train()
        prev_seconds = self._total_train_seconds
        time_start = time.time()
        if self._optimizer_type is None:
            self._optimizer_type = optimizer_type
        if self._momentum is None:
            self._momentum = momentum
        if self._weight_decay is None:
            self._weight_decay = weight_decay
        if self._learning_rate_scheduler_type is None:
            self._learning_rate_scheduler_type = learning_rate_scheduler_type
        if self._learning_rate_init is None:
            self._learning_rate_init = learning_rate_init * math.sqrt(world)
        if self._learning_rate_end is None:
            self._learning_rate_end = learning_rate_end
        if self._total_train_traces_end is None:
            self._total_train_traces_end = num_traces_end
        trace, stop = 0, False
        last_save = time_start
        if hasattr(dataset, 'num_buckets'):      # offline data: bucketed rank-strided sampling (dataset.py:330-400)
            dataset.num_buckets = distributed_num_buckets
        if dataset_valid is not None:
            if hasattr(dataset_valid, 'num_buckets'):
                dataset_valid.num_buckets = distributed_num_buckets
            if not self._layers_pre_generated:   # reference inference_network.py:412-414
                for vbatch in dataset_valid.epoch_batches(batch_size):
                    self._polymorph(vbatch)
        if valid_every is None:
            valid_every = max(100, num_traces / 1000)
        last_validation_trace = -valid_every + 1
        valid_loss = 0
        log_file = None
        if rank == 0 and log_file_name is not None:
            log_file = open(log_file_name, mode='w', buffering=1)
            log_file.write('time, iteration, trace, loss, valid_loss, learning_rate, mean_trace_length_controlled, '
                           'sub_mini_batches, distributed_bucket_id, traces_per_second\n')
        time_last_batch = time_start
        while not stop:
            batch = dataset.next_batch(batch_size)
            time_batch = time.time()
            layers_changed = False if self._layers_pre_generated else self._polymorph(batch)
            if world > 1 and layers_changed:
                raise RuntimeError('pyprob_b200: new addresses appeared during data-parallel training; call '
                                   '_pre_generate_layers first so that every rank holds the same arena layout')
            if self._exp_avg is None or layers_changed:
                self._create_optimizer()
            if world > 1 and self._peer is None and self._seg is None and distributed_backend == 'nccl':
                self._enable_peer_optimizer()
            if world > 1 and self._total_train_iterations == 0:
                dist.broadcast(self._arena.data, 0)
            self._arena.grad = None
            success, loss = self._loss(batch)
            if not success:
                print('Cannot compute loss, skipping batch. Loss: {}'.format(loss))
                if stop_with_bad_loss:
                    return
                continue
            loss.backward()
            self._learning_rate = self._current_learning_rate()
            if self._peer is not None:
                # reduce-scatter + Adam + all-gather in one kernel over NVLink peer memory
                loss_value = self._peer_optimizer_step(loss.detach(), world)
            else:
                # one all-reduce over the flat gradient arena, loss scalar piggy-backed (SURVEY 8e)
                loss_value, grad_scale = parallel.allreduce_grad_and_loss(self._arena.grad, loss.detach())
                self.optimizer_step(grad_scale)
            if self._loss_init is None:
                self._loss_init = loss_value
                self._loss_max = loss_value
            self._loss_min = min(self._loss_min, loss_value)
            self._loss_max = max(self._loss_max, loss_value)
            self._loss_previous = loss_value
            self._total_train_iterations += 1
            trace += batch.size * world
            self._total_train_traces += batch.size * world
            self._total_train_seconds = prev_seconds + (time_batch - time_start)
            self._history_train_loss.append(loss_value)
            self._history_train_loss_trace.append(self._total_train_traces)
            traces_per_second = batch.size * world / max(time_batch - time_last_batch, 1e-9)
            time_last_batch = time_batch
            if dataset_valid is not None and trace - last_validation_trace > valid_every:
                valid_loss = self._validation_loss(dataset_valid, batch_size, world)
                self._history_valid_loss.append(valid_loss)
                self._history_valid_loss_trace.append(self._total_train_traces)
                last_validation_trace = trace - 1
            if save_file_name_prefix is not None and save_every_sec is not None:
                want_save = rank == 0 and time_batch - last_save > save_every_sec
                if world > 1 and self._peer is not None:
                    # the optimiser moments are sharded over the ranks: saving is a collective, rank 0's clock decides
                    flag = torch.tensor([1 if want_save else 0], dtype=torch.int32, device=self._arena.device)
                    dist.broadcast(flag, 0)
                    want_save = bool(int(flag))
                if want_save:
                    last_save = time_batch
                    moments = self._full_optimizer_moments()
                    if rank == 0:
                        self._save('{}_{}_traces_{}.network'.format(save_file_name_prefix, util.get_time_stamp(),
                                                                   self._total_train_traces), moments)
            if trace >= num_traces:
                stop = True
            if util._verbosity > 1 and (stop or self._total_train_iterations % 50 == 0):
                print('{} | {:9,} | loss {:+.2e} (init {:+.2e}, min {:+.2e}) | lr {:.2e} | {:,.1f} traces/s'.format(
                    util.days_hours_mins_secs_str(self._total_train_seconds), self._total_train_traces, loss_value,
                    self._loss_init, self._loss_min, self._learning_rate, traces_per_second))
            if log_file is not None:
                log_file.write('{}, {}, {}, {}, {}, {}, {}, {}, {}, {}\n'.format(
                    self._total_train_seconds, self._total_train_iterations, self._total_train_traces, loss_value,
                    valid_loss, self._learning_rate, batch.mean_length_controlled, batch.num_sub_batches,
                    getattr(dataset, 'current_bucket_id', None), traces_per_second))
        if log_file is not None:
            log_file.close()
        if save_file_name_prefix is not None:
            moments = self._full_optimizer_moments()   # collective under the fused data-parallel step
            if rank == 0:
                self._save('{}_{}_traces_{}.network'.format(save_file_name_prefix, util.get_time_stamp(),
                                                           self._total_train_traces), moments)

    def _validation_loss(self, dataset_valid, batch_size, world):
        """Mean minibatch loss over one pass of the validation set (reference inference_network.py:534-546): the
        sum of the per-minibatch losses of this rank's share, divided by (minibatches / world), averaged over
        ranks."""
        total, count = 0.0, 0
        with torch.no_grad():
            for vbatch in dataset_valid.epoch_batches(batch_size):
                success, v = self._loss(vbatch)
                if success:
                    total += float(v)
                count += 1
        denom = dataset_valid.num_batches(batch_size) / world if world > 1 else count
        value = total / max(denom, 1e-9)
        if world > 1:
            import torch.distributed as dist
            t = torch.tensor([value], dtype=torch.float32, device=self._arena.device)
            dist.all_reduce(t)
            value = float(t) / world
        return value

    def _pre_generate_layers(self, dataset, batch_size=64, save_file_name_prefix=None, num_batches=16):
        self._ensure_initialized(dataset.example_trace())
        self._layers_pre_generated = True
        if hasattr(dataset, 'address_signature'):
            # offline data: the files carry their address table, so one call sees what a full pass of the reference's
            # batch-by-batch _polymorph would discover (inference_network.py:270-288), in the same order
            changed = self._polymorph(dataset)
        else:
            changed = False
            for _ in range(num_batches):
                changed = self._polymorph(dataset.next_batch(batch_size)) or changed
        if changed and save_file_name_prefix is not None:
            self._save('{}_00000000_pre_generated.network'.format(save_file_name_prefix))

    # ------------------------------------------------------------------------------------------------
    # checkpoint (reference: inference_network.py:162-263)
    # ------------------------------------------------------------------------------------------------
    def _owned_slice(self, n, world, rank):
        """[lo, hi) of the flat arena whose optimiser state lives on `rank` under the fused data-parallel step
        (same split as k_dp_adam, csrc/dp.cu: ceil(n / 4 world) float4 blocks per rank)."""
        per = ((n + world * 4 - 1) // (world * 4)) * 4
        lo = min(n, rank * per)
        return lo, min(n, lo + per)

    def _full_optimizer_moments(self):
        """(exp_avg, exp_avg_sq) of the WHOLE arena.  With the fused data-parallel step every rank only ever updates the
        moments of the slice it owns; a checkpoint needs all of them, so the owned slices are summed over the ranks (each
        element is non-zero on exactly one rank).  COLLECTIVE when training data-parallel: every rank must call it."""
        if self._exp_avg is None:
            return None, None
        if self._peer is None:
            return self._exp_avg, self._exp_avg_sq
        import torch.distributed as dist
        world, rank = parallel.world_info()
        n = self._exp_avg.numel()
        lo, hi = self._owned_slice(n, world, rank)
        out = []
        for t in (self._exp_avg, self._exp_avg_sq):
            full = torch.zeros_like(t)
            full[lo:hi] = t[lo:hi]
            if world > 1:
                dist.all_reduce(full)
            out.append(full)
        return out[0], out[1]

    def _save(self, file_name, moments=None):
        """Write a checkpoint.  Data-parallel training over NVLink peer memory: call `_full_optimizer_moments()` on EVERY
        rank first and pass the result on the rank that writes (optimize() does this); a direct call on one rank falls
        back to that rank's local arrays."""
        self._modified = util.get_time_str()
        self._updates += 1
        m, v = moments if moments is not None else (
            self._full_optimizer_moments() if parallel.world_info()[0] == 1 else (self._exp_avg, self._exp_avg_sq))
        data = {'pyprob_b200_version': 1, 'torch_version': torch.__version__, 'inference_network': self,
                'optimizer_state': None if self._exp_avg is None else
                {'exp_avg': m.cpu(), 'exp_avg_sq': v.cpu(), 'step': self._optimizer_step,
                 'segment_steps': None if self._seg is None else self._seg['steps'].cpu()}}
        torch.save(data, file_name)

    @staticmethod
    def _load(file_name):
        data = torch.load(file_name, map_location='cuda', weights_only=False)
        ret = data['inference_network']
        ret._arena_store = ret._arena.data.clone()
        ret._arena = nn.Parameter(ret._arena_store[:ret._arena_used])
        ret._handle = None
        ret._tables_dirty = True
        for k, default in (('_peer', None), ('_seg', None), ('_skip_absent_gradients', False), ('_last_enc', None),
                           ('_auto_skip_absent', True), ('_present_sig', None)):
            ret.__dict__.setdefault(k, default)   # checkpoints written before these attributes existed
        if data['optimizer_state'] is not None:
            ret._create_optimizer(data['optimizer_state'])
        return ret

    def to(self, device=None, *args, **kwargs):
        if device is not None and 'cuda' not in str(device):
            raise RuntimeError('pyprob_b200 networks live on the GPU; there is no CPU path')
        return self

    # ------------------------------------------------------------------------------------------------
    # inference (reference: inference_network.py:141-148, inference_network_lstm.py:82-134)
    # ------------------------------------------------------------------------------------------------
    def _infer_workspace(self, n):
        need = _lib.call('ppb_ic_infer_workspace_bytes', self._handle, n)
        ws = getattr(self, '_infer_ws', None)
        if ws is None or ws.numel() < need:
            self._infer_ws = torch.empty(int(need), dtype=torch.uint8, device='cuda')
        return need

    def _infer_init(self, observe=None):
        """Embed the (single) observation once; `observe` maps names to values."""
        self._sync_native()
        self._infer_observe = observe
        vals = []
        for name, in_dim in zip(self._observe_names, self._observe_in_dims):
            v = torch.as_tensor(observe[name], dtype=torch.float32).reshape(-1)
            if v.numel() != in_dim:
                raise ValueError('observable {} has {} elements, expected {}'.format(name, v.numel(), in_dim))
            vals.append(v)
        obs = torch.cat(vals).view(1, -1).to('cuda')
        need = self._infer_workspace(1)
        emb = torch.empty(1, self._observe_embedding_dim, dtype=torch.float32, device='cuda')
        call('ppb_ic_embed_observe', self._handle, ptr(self._arena.data), ptr(obs), ptr(emb), 1, ptr(self._infer_ws),
             need, stream())
        self._infer_observe_embedding = emb
        self._infer_state = None

    def _address_by_id(self):
        """address id -> address string (ids are insertion order of `_addresses`)."""
        cache = getattr(self, '_by_id_cache', None)
        if cache is None or len(cache) != len(self._addresses):
            cache = {info['id']: a for a, info in self._addresses.items()}
            self._by_id_cache = cache
        return cache


class InferenceNetworkLSTM(InferenceNetwork):
    """pyprob/nn/inference_network_lstm.py: observation embedding, previous-sample / address / type embeddings -> LSTM ->
    the proposal head of each step's address."""

    def __init__(self, model=None, observe_embeddings={}, lstm_dim=512, lstm_depth=1, sample_embedding_dim=4,
                 address_embedding_dim=64, distribution_type_embedding_dim=8, proposal_mixture_components=10,
                 precision=0):
        if lstm_depth != 1:
            raise NotImplementedError('pyprob_b200: lstm_depth != 1 is not implemented (reference default is 1)')
        super().__init__(model=model, observe_embeddings=observe_embeddings,
                         proposal_mixture_components=proposal_mixture_components, precision=precision,
                         network_type='InferenceNetworkLSTM')
        self._lstm_dim, self._lstm_depth = lstm_dim, lstm_depth
        self._lstm_input_dim = None
        self._sample_embedding_dim = sample_embedding_dim
        self._address_embedding_dim = address_embedding_dim
        self._distribution_type_embedding_dim = distribution_type_embedding_dim

    def _init_layers(self):
        E = self._observe_embedding_dim
        self._lstm_input_dim = E + self._sample_embedding_dim + 2 * (self._address_embedding_dim +
                                                                     self._distribution_type_embedding_dim)
        ref = nn.LSTM(self._lstm_input_dim, self._lstm_dim, 1)
        self._alloc('_layers_lstm.weight_ih_l0', (4 * self._lstm_dim, self._lstm_input_dim), ref.weight_ih_l0)
        self._alloc('_layers_lstm.weight_hh_l0', (4 * self._lstm_dim, self._lstm_dim), ref.weight_hh_l0)
        self._alloc('_layers_lstm.bias_ih_l0', (4 * self._lstm_dim,), ref.bias_ih_l0)
        self._alloc('_layers_lstm.bias_hh_l0', (4 * self._lstm_dim,), ref.bias_hh_l0)
        self._rebind()

    def _add_address(self, address, dist_name, num_categories=0):
        """New address: address/type embeddings, sample-embedding layer, proposal head (:42-72)."""
        if dist_name not in _FAMILY_OF:
            raise RuntimeError('Distribution currently unsupported: {}'.format(dist_name))
        family = _FAMILY_OF[dist_name]
        self._alloc('_layers_address_embedding.{}'.format(address), (self._address_embedding_dim,),
                    torch.zeros(self._address_embedding_dim).normal_())
        if dist_name not in self._types:
            self._alloc('_layers_distribution_type_embedding.{}'.format(dist_name),
                        (self._distribution_type_embedding_dim,),
                        torch.zeros(self._distribution_type_embedding_dim).normal_())
            self._types[dist_name] = len(self._types)
        head = self._proposal_layers(address, family, num_categories, self._lstm_dim)
        smp_in = num_categories if family == FAMILY_CATEGORICAL else 1
        self._linear('_layers_sample_embedding.{}._layers.0'.format(address), smp_in, self._sample_embedding_dim)
        self._addresses[address] = dict(id=len(self._addresses), family=family, num_categories=num_categories,
                                        smp_in=smp_in, type=dist_name, **head)
        self._head_iterations[address] = 0

    def _segment_presence(self, enc, force=False):
        """int32[S]: 1 for every parameter tensor that took part in the forward pass of the encoded minibatch, i.e.
        whose .grad the reference's autograd would populate (all others stay None and are skipped by torch.optim):
        shared layers always; address / type embeddings and the proposal head of every address in the batch; the
        sample-embedding layer of every address that is some step's PREVIOUS address (inference_network_lstm.py:
        150-182)."""
        names = self._seg['names'] if self._seg is not None else self._segment_names()
        present = np.ones(len(names), dtype=np.int32)
        if (not self._skip_absent_gradients and not force) or enc is None:
            return present
        by_id = {info['id']: (a, info) for a, info in self._addresses.items()}
        cur = set(int(i) for i in np.unique(enc.arrays['step_addr']))
        prev = set(int(i) for i in np.unique(enc.arrays['step_prev_addr']) if i >= 0)
        types = set(by_id[i][1]['type'] for i in cur | prev)
        for k, name in enumerate(names):
            if name.startswith('_layers_address_embedding.'):
                a = name[len('_layers_address_embedding.'):]
                present[k] = int(self._addresses[a]['id'] in cur)
            elif name.startswith('_layers_distribution_type_embedding.'):
                present[k] = int(name[len('_layers_distribution_type_embedding.'):] in types)
            elif name.startswith('_layers_proposal.'):
                a = name[len('_layers_proposal.'):name.index('._ff._layers.')]
                present[k] = int(self._addresses[a]['id'] in cur)
            elif name.startswith('_layers_sample_embedding.'):
                a = name[len('_layers_sample_embedding.'):name.index('._layers.')]
                present[k] = int(self._addresses[a]['id'] in prev)
        return present

    def _infer_step_lanes(self, address, prev_address, prev_value, prior0, prior1, h, c):
        """One proposal step for the particles whose LSTM state rows are `h`, `c` ([m, H] contiguous, updated in place):
        all m particles sit at `address` and came from `prev_address` (None: first controlled site) with values
        `prev_value` [m].  Returns the proposal parameters [m, 3K] (means|stddevs|probs), [m, C] or [m, 1] (Bernoulli
        probs)."""
        info = self._addresses[address]
        m = h.size(0)
        width = info['head_out'] if info['family'] != FAMILY_CATEGORICAL else info['num_categories']
        params = torch.empty(m, width, dtype=torch.float32, device='cuda')
        need = self._infer_workspace(m)

        def par(x):
            if x is None:
                return None, 0, None
            t = ops._f32(x, 'cuda').reshape(-1)      # python scalars: cached device constants (no host->device copy)
            return t, (0 if t.numel() == 1 else 1), t
        p0, s0, k0 = par(prior0)
        p1, s1, k1 = par(prior1)
        pv = None if prev_value is None else prev_value.to(dtype=torch.float32).contiguous()
        call('ppb_ic_infer_step', self._handle, ptr(self._arena.data), ptr(self._infer_observe_embedding), 0,
             -1 if prev_address is None else self._addresses[prev_address]['id'], ptr(pv), info['id'],
             ptr(p0), s0, ptr(p1), s1, ptr(h), ptr(c), ptr(params), m, ptr(self._infer_ws), need, self._precision,
             stream())
        return params

    def _infer_step_batched(self, address, prev_address, prev_value, prior0, prior1, n):
        """Proposal parameters for n particles in lock-step at `address`.

        Returns a [n, 3K] (means|stddevs|probs), [n, C] or [n, 1] (Bernoulli probs) tensor, or None if the address is unknown
        (the caller then falls back to the prior, as the reference does with a warning)."""
        if address not in self._addresses or (prev_address is not None and prev_address not in self._addresses):
            warnings.warn('Address unknown by inference network: {}'.format(address))
            return None
        info = self._addresses[address]
        H = self._lstm_dim
        if prev_address is None or self._infer_state is None or self._infer_state[0].size(0) != n:
            self._infer_state = (torch.zeros(n, H, device='cuda'), torch.zeros(n, H, device='cuda'))
        h, c = self._infer_state
        width = info['head_out'] if info['family'] != FAMILY_CATEGORICAL else info['num_categories']
        params = torch.empty(n, width, dtype=torch.float32, device='cuda')
        need = self._infer_workspace(n)

        def par(x):
            if x is None:
                return None, 0, None
            t = torch.as_tensor(x, dtype=torch.float32, device='cuda').reshape(-1)
            return t, (0 if t.numel() == 1 else 1), t
        p0, s0, k0 = par(prior0)
        p1, s1, k1 = par(prior1)
        pv = None if prev_value is None else prev_value.to(dtype=torch.float32).contiguous()
        call('ppb_ic_infer_step', self._handle, ptr(self._arena.data), ptr(self._infer_observe_embedding), 0,
             -1 if prev_address is None else self._addresses[prev_address]['id'], ptr(pv), info['id'],
             ptr(p0), s0, ptr(p1), s1, ptr(h), ptr(c), ptr(params), n, ptr(self._infer_ws), need, self._precision,
             stream())
        return params

    def _fill_net_desc(self, nd):
        nd.network_type = NET_LSTM
        nd.lstm_dim, nd.sample_dim = self._lstm_dim, self._sample_embedding_dim
        nd.addr_dim, nd.type_dim = self._address_embedding_dim, self._distribution_type_embedding_dim
        nd.w_ih_off = self.parameter_index['_layers_lstm.weight_ih_l0'][0]
        nd.w_hh_off = self.parameter_index['_layers_lstm.weight_hh_l0'][0]
        nd.b_ih_off = self.parameter_index['_layers_lstm.bias_ih_l0'][0]
        nd.b_hh_off = self.parameter_index['_layers_lstm.bias_hh_l0'][0]

    def _fill_addr_desc(self, a, address, info):
        pi = self.parameter_index
        a.type_id = self._types[info['type']]
        a.addr_emb_off = pi['_layers_address_embedding.{}'.format(address)][0]
        a.smp_w_off = pi['_layers_sample_embedding.{}._layers.0.weight'.format(address)][0]
        a.smp_b_off = pi['_layers_sample_embedding.{}._layers.0.bias'.format(address)][0]


class InferenceNetworkFeedForward(InferenceNetwork):
    """pyprob/nn/inference_network_feedforward.py: every proposal head reads the observation embedding directly.  No LSTM
    and no address, type or sample embeddings; lstm_dim and lstm_depth are accepted and ignored, as in the reference."""

    def __init__(self, model=None, observe_embeddings={}, proposal_mixture_components=10, precision=0, lstm_dim=None,
                 lstm_depth=None):
        super().__init__(model=model, observe_embeddings=observe_embeddings,
                         proposal_mixture_components=proposal_mixture_components, precision=precision,
                         network_type='InferenceNetworkFeedForward')

    def _add_address(self, address, dist_name, num_categories=0):
        """New address: its proposal layer only (_polymorph, :21-51), Linear(E -> int((E + out) / 2)) -> out."""
        if dist_name not in _FAMILY_OF:
            raise RuntimeError('Distribution currently unsupported: {}'.format(dist_name))
        family = _FAMILY_OF[dist_name]
        head = self._proposal_layers(address, family, num_categories, self._observe_embedding_dim)
        self._addresses[address] = dict(id=len(self._addresses), family=family, num_categories=num_categories,
                                        smp_in=1 if family != FAMILY_CATEGORICAL else num_categories, type=dist_name,
                                        **head)
        self._head_iterations[address] = 0

    def _fill_net_desc(self, nd):
        nd.network_type = NET_FEEDFORWARD

    def _fill_addr_desc(self, a, address, info):
        pass

    def _segment_presence(self, enc, force=False):
        """int32[S]: the observation layers always take part; a proposal layer iff its address is in the minibatch."""
        names = self._seg['names'] if self._seg is not None else self._segment_names()
        present = np.ones(len(names), dtype=np.int32)
        if (not self._skip_absent_gradients and not force) or enc is None:
            return present
        cur = set(int(i) for i in np.unique(enc.arrays['step_addr']))
        for k, name in enumerate(names):
            if name.startswith('_layers_proposal.'):
                a = name[len('_layers_proposal.'):name.index('._ff._layers.')]
                present[k] = int(self._addresses[a]['id'] in cur)
        return present

    def _infer_step_lanes(self, address, prior0, prior1, m):
        """Proposal parameters at `address` for m particles (_infer_step, :53-66): the head runs once on the shared
        observation embedding; only the priors differ per particle.  [m, 3K] (means|stddevs|probs), [m, C] or [m, 1]."""
        info = self._addresses[address]
        width = info['head_out'] if info['family'] != FAMILY_CATEGORICAL else info['num_categories']
        params = torch.empty(m, width, dtype=torch.float32, device='cuda')
        need = self._infer_workspace(m)

        def par(x):
            if x is None:
                return None, 0
            t = ops._f32(x, 'cuda').reshape(-1)      # python scalars: cached device constants (no host->device copy)
            return t, (0 if t.numel() == 1 else 1)
        p0, s0 = par(prior0)
        p1, s1 = par(prior1)
        call('ppb_ic_infer_step', self._handle, ptr(self._arena.data), ptr(self._infer_observe_embedding), 0, -1, None,
             info['id'], ptr(p0), s0, ptr(p1), s1, None, None, ptr(params), m, ptr(self._infer_ws), need,
             self._precision, stream())
        return params

    def _infer_step_batched(self, address, prev_address, prev_value, prior0, prior1, n):
        """As InferenceNetworkLSTM._infer_step_batched; the previous site plays no part.  None if the address is unknown
        (the caller then falls back to the prior)."""
        if address not in self._addresses:
            warnings.warn('Address unknown by inference network: {}'.format(address))
            return None
        return self._infer_step_lanes(address, prior0, prior1, n)
