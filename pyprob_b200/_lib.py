"""ctypes binding of the C-ABI in include/pyprob_b200.h.

The shared library is built in-tree by ``__graft_entry__.build()`` (nvcc, sm_90a).  There is no CPU
fallback: if the library is missing, or an entry point fails, the call raises.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libpyprob_b200.so')

_lib = None

c_f = C.c_void_p  # device pointers travel as integers
c_i32 = C.c_int32
c_i64 = C.c_int64
c_u64 = C.c_uint64
c_dbl = C.c_double
c_flt = C.c_float
c_int = C.c_int

# name -> argtypes (restype is int unless listed in _RESTYPES)
_SIGNATURES = {
    'ppb_version': [],
    'ppb_device_arch': [],
    'ppb_launch_count': [],
    'ppb_prof_enable': [c_int],
    'ppb_prof_read': [C.c_void_p, C.c_void_p, C.c_void_p],
    'ppb_categorical_log_prob': [c_f, c_f, c_i64, c_int, c_f, c_f, c_dbl, c_i64, c_f],
    'ppb_mixture_normal_log_prob': [c_f, c_f, c_f, c_f, c_i64, c_int, c_f, c_f, c_dbl, c_i64, c_f],
    'ppb_mixture_truncated_normal_log_prob': [c_f, c_f, c_f, c_f, c_i64, c_int, c_f, c_int, c_f, c_int, c_f, c_f,
                                              c_dbl, c_i64, c_f],
    'ppb_categorical_sample': [c_f, c_i64, c_int, c_f, c_f, c_i64, c_u64, c_u64, c_i64, c_f],
    'ppb_mixture_normal_sample': [c_f, c_f, c_f, c_i64, c_int, c_f, c_f, c_i64, c_u64, c_u64, c_i64, c_f],
    'ppb_mixture_truncated_normal_sample': [c_f, c_f, c_f, c_i64, c_int, c_f, c_int, c_f, c_int, c_f, c_f, c_i64,
                                            c_u64, c_u64, c_i64, c_f],
    'ppb_event_log_prob': [c_int, c_f, c_i64, c_i64, c_f, c_i64, c_i64, c_f, c_i64, c_i64, c_f, c_i64, c_i64, c_f,
                           c_i64, c_i64, c_i64, c_i64, c_f, c_f, c_dbl, c_f],
    'ppb_event_sample': [c_int, c_f, c_i64, c_i64, c_f, c_i64, c_i64, c_f, c_i64, c_i64, c_f, c_i64, c_i64, c_f, c_f,
                         c_i64, c_i64, c_u64, c_u64, c_i64, c_f],
    'ppb_event_log_prob_d1': [c_int, c_f, c_f, c_f, c_f, c_f, c_int, c_f, c_f, c_dbl, c_i64, c_f],
    'ppb_event_sample_d1': [c_int, c_f, c_f, c_f, c_f, c_int, c_f, c_f, c_i64, c_u64, c_u64, c_i64, c_f],
    'ppb_weights_cast': [c_f, c_f, c_f, c_i64, c_f],
    'ppb_weights_num_partials': [c_i64],
    'ppb_weights_partials': [c_f, c_i64, c_f, c_f],
    'ppb_weights_finalize': [c_f, c_i64, c_f, c_int, c_f, c_f, c_f],
    'ppb_net_create': [C.c_void_p, C.c_void_p],
    'ppb_net_set_tables': [C.c_void_p, C.c_void_p, c_i32, C.c_void_p, c_i32, c_i64],
    'ppb_net_destroy': [C.c_void_p],
    'ppb_ic_workspace_bytes': [C.c_void_p, c_i32, c_i32, c_i32, c_i32, c_i32],
    'ppb_batch_from_image': [C.c_void_p, c_f, c_i64, C.c_void_p],
    'ppb_sizeof': [c_int],
    'ppb_ic_loss_forward': [C.c_void_p, c_f, C.c_void_p, c_f, c_i64, c_int, c_f, c_f, c_f, c_int, c_f],
    'ppb_ic_loss_backward': [C.c_void_p, c_f, c_f, C.c_void_p, c_f, c_i64, c_int, c_flt, c_f],
    'ppb_adam_step_dev': [c_f, c_f, c_f, c_f, c_i64, c_f, c_f, c_f],
    'ppb_optimizer_scratch_bytes': [c_i32],
    'ppb_optimizer_step_segmented': [c_f, c_f, c_f, c_f, c_i64, c_f, c_i32, c_f, c_f, c_f, c_i64, c_int, c_f, c_f],
    'ppb_dp_alloc': [c_i64, C.c_void_p, C.c_void_p],
    'ppb_dp_open': [C.c_void_p, C.c_void_p],
    'ppb_dp_close': [c_f],
    'ppb_dp_free': [c_f],
    'ppb_dp_rendezvous': [c_int, c_int, C.c_void_p, c_i64, c_f],
    'ppb_dp_adam_step': [c_int, c_int, C.c_void_p, c_i64, c_i64, c_i64, c_f, c_f, c_i64, c_i64, c_f, c_f, c_f],
    'ppb_ic_infer_step': [C.c_void_p, c_f, c_f, c_int, c_i32, c_f, c_i32, c_f, c_int, c_f, c_int, c_f, c_f, c_f,
                          c_i64, c_f, c_i64, c_int, c_f],
    'ppb_ic_embed_observe': [C.c_void_p, c_f, c_f, c_f, c_i64, c_f, c_i64, c_f],
    'ppb_ic_infer_workspace_bytes': [C.c_void_p, c_i64],
    'ppb_net_refresh_weights': [C.c_void_p, c_f, c_f],
    'ppb_net_forget_uploads': [C.c_void_p],
    'ppb_ic_train_step_host': [C.c_void_p, c_f, c_f, c_f, c_f, c_i64, C.c_void_p, c_i64, c_f, c_f, c_i64, c_int,
                               c_flt, c_flt, c_flt, c_flt, c_flt, c_i64, C.c_void_p, C.c_void_p, c_f],
    'ppb_packed_floats': [c_i64, c_i64],
    'ppb_pack_tf32': [c_f, c_i64, c_i64, c_i64, c_f, c_f, c_f],
    'ppb_pack_tf32_mn': [c_f, c_i64, c_i64, c_i64, c_f, c_f, c_f],
    'ppb_debug_trace': [c_f],
    'ppb_gemm_packed_tn': [c_f, c_f, c_f, c_f, c_f, c_i64, c_i64, c_i64, c_i64, c_int, c_f],
    'ppb_gemm_packed': [c_f, c_f, c_f, c_f, c_f, c_i64, c_i64, c_i64, c_i64, c_f, c_int, c_int, c_f],
    'ppb_gemm_packed_cluster': [c_f, c_f, c_f, c_f, c_f, c_i64, c_i64, c_i64, c_i64, c_f, c_int, c_int, c_int, c_f],
    'ppb_tc_run_problems': [C.c_void_p, c_int, c_int, c_int, c_int, c_int, c_f],
    'ppb_mh_select': [c_f, c_f, c_f, c_i64, c_i64, c_int, c_f, c_f, c_f, c_f, c_f, c_int, c_u64, c_u64, c_f],
    'ppb_mh_fetch': [c_f, c_f, c_f, c_f, c_f, c_i64, c_i64, c_int, c_f, c_i64, c_i64, c_f, c_f, c_f, c_f],
    'ppb_mh_site': [c_int, c_int, c_f, c_i64, c_i64, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_int, c_f, c_int, c_f, c_f,
                    c_f, c_f, c_f, c_f, c_i32, c_i64, c_i64, c_f, c_f, c_f, c_f, c_f, c_u64, c_u64, c_f],
    'ppb_mh_accept': [c_i64, c_int, c_i32, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_int, c_f,
                      c_i64, c_u64, c_u64, c_f],
    'ppb_diag_rhat_workspace_bytes': [c_i64, c_i64, c_i64, C.c_void_p, c_int],
    'ppb_diag_rhat': [c_f, c_int, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, C.c_void_p, c_int, c_f, c_f, c_i64, c_f],
    'ppb_diag_autocorr_workspace_bytes': [c_int, c_i64, c_i64, c_i64, c_int],
    'ppb_diag_autocorr': [c_f, c_int, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, C.c_void_p, c_int, c_f, c_f, c_i64,
                          c_f],
}
_RESTYPES = {
    'ppb_diag_rhat_workspace_bytes': c_i64,
    'ppb_diag_autocorr_workspace_bytes': c_i64,
    'ppb_ic_workspace_bytes': c_i64,
    'ppb_ic_infer_workspace_bytes': c_i64,
    'ppb_packed_floats': c_i64,
    'ppb_sizeof': c_i64,
    'ppb_launch_count': c_i64,
    'ppb_optimizer_scratch_bytes': c_i64,
}
# entry points whose integer return value is data, not a status
_VALUE_RETURNS = {'ppb_optimizer_scratch_bytes', 'ppb_version', 'ppb_device_arch', 'ppb_weights_num_partials', 'ppb_ic_workspace_bytes',
                  'ppb_ic_infer_workspace_bytes', 'ppb_packed_floats', 'ppb_sizeof', 'ppb_launch_count',
                  'ppb_diag_rhat_workspace_bytes', 'ppb_diag_autocorr_workspace_bytes'}

EXPORTED_SYMBOLS = sorted(list(_SIGNATURES.keys()) + ['ppb_last_error'])


def load():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError('pyprob_b200: native library not found at {} — run `python -c "import __graft_entry__ as g; '
                           'g.build()"` (nvcc, sm_90a). There is no CPU fallback.'.format(LIB_PATH))
    lib = C.CDLL(LIB_PATH)
    for name, argtypes in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            raise RuntimeError('pyprob_b200: {} does not export {} — stale build? rebuild with '
                               '__graft_entry__.build(force=True)'.format(LIB_PATH, name))
        fn.argtypes = argtypes
        fn.restype = _RESTYPES.get(name, c_int)
    lib.ppb_last_error.argtypes = []
    lib.ppb_last_error.restype = C.c_char_p
    _lib = lib
    return lib


def last_error():
    return load().ppb_last_error().decode('utf-8', 'replace')


def call(name, *args):
    """Call an entry point; raise RuntimeError with ppb_last_error() on a non-zero status."""
    lib = load()
    ret = getattr(lib, name)(*args)
    if name in _VALUE_RETURNS:
        return ret
    if ret != 0:
        raise RuntimeError('{} failed with status {}: {}'.format(name, ret, last_error()))
    return 0


def ptr(t):
    """Device pointer of a CUDA tensor (None -> NULL)."""
    if t is None:
        return None
    if not t.is_cuda:
        raise RuntimeError('pyprob_b200 kernels need CUDA tensors (no CPU fallback); got device {}'.format(t.device))
    return t.data_ptr()


def stream():
    return torch.cuda.current_stream().cuda_stream


def require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError('pyprob_b200 needs a CUDA device (sm_90a: H100); there is no CPU fallback')
