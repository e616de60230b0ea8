"""ctypes binding of libpromp_b200.so (the C ABI declared in include/promp_b200.h).

PyTorch tensors are used only as device buffers: every call passes raw `data_ptr()` addresses and
the current CUDA stream handle.  There is NO CPU fallback: if the library is missing or no CUDA
device is present, the product path raises.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_uint64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('PROMP_B200_LIB', os.path.join(_HERE, 'libpromp_b200.so'))   # override: kernel experiments

# enums (mirror include/promp_b200.h)
ENV_POINT_CORNER, ENV_POINT, ENV_CHEETAH_DIR, ENV_POINT_WALLS, ENV_POINT_MOMENTUM = 0, 1, 2, 3, 4
ENV_WALKER, ENV_SWIMMER = 5, 6
EARLY_TERM_ENVS = (ENV_POINT, ENV_WALKER)        # env kinds whose paths end on `done` (variable-length paths)
INFO_ENVS = (ENV_CHEETAH_DIR, ENV_SWIMMER)       # env kinds whose kernels write env_infos channels
# env modules (promp_env_module_load): kernel slots and dims
ENV_MODULE_SLOTS, ENV_MODULE_NDIMS, ENV_SLOT_STEP, ENV_SLOT_OBSERVE, ENV_SLOT_ROLLOUT = 34, 6, 0, 1, 2
ENV_SLOT_ROLLOUT_DEEP = 18
REWARD_SPARSE, REWARD_DENSE, REWARD_DENSE_SQUARED = 0, 1, 2
OBJ_RATIO, OBJ_LOGLIK, OBJ_CLIP, OBJ_NONE, OBJ_EXPLORE = 0, 1, 2, 3, 4
BASELINE_ZERO, BASELINE_LINEAR_FEATURE, BASELINE_LINEAR_TIME, BASELINE_GIVEN = 0, 1, 2, 3
# the policy / rollout `hidden` argument: width | activation flag (no flag = tanh) | output flag (no flag = identity)
HIDDEN_WIDTH_MASK, ACT_RELU, OUT_TANH = 0xFF, 0x100, 0x1000
# ... | the number of hidden layers in a 3-bit field (no bits = two hidden layers)
HIDDEN_DEPTH_SHIFT, HIDDEN_DEPTH_MASK = 14, 0x1C000


def hidden_depth(layers):
    """The depth bits of the `hidden` argument for `layers` hidden layers (PROMP_HIDDEN_DEPTH; 0 for two layers)."""
    return 0 if layers == 2 else layers << HIDDEN_DEPTH_SHIFT

_P = c_void_p


class PolicyStage(ctypes.Structure):
    """promp_policy_stage of include/promp_b200.h (one stage of promp_policy_chain)."""
    _fields_ = [('kind', c_int32), ('N', c_int32), ('n_valid', _P), ('params', _P), ('param_stride', c_int64),
                ('obs', _P), ('act', _P), ('adv', _P), ('old_mean', _P), ('old_log_std', _P),
                ('ls_per_sample', c_int32), ('obj_kind', c_int32), ('obj_scale', c_float), ('clip_eps', c_float),
                ('kl_coeff', c_float), ('clip_log_std', c_int32), ('grad', _P), ('out_params', _P), ('sgd_lr', c_float),
                ('inner_lr', c_float), ('vec', _P), ('out', _P), ('stats', _P), ('kl_coeff_dev', _P),
                ('step_size', _P)]


_SIGNATURES = {
    'promp_last_error': (c_char_p, []),
    'promp_version': (c_int, []),
    'promp_num_params': (c_int, [c_int, c_int, c_int]),
    'promp_env_state_dim': (c_int, [c_int]),
    'promp_env_task_dim': (c_int, [c_int]),
    'promp_rollout': (c_int, [c_int, c_int, c_float, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, c_uint64,
                              c_uint64, _P, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'promp_rollout_early_term': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, c_uint64, c_uint64,
                                         _P, c_int, c_float, _P, _P, _P, _P, _P, _P, _P]),
    'promp_rollout_ex': (c_int, [c_int, c_int, c_float, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, c_uint64,
                                 c_uint64, _P, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int]),
    'promp_rollout_early_term_ex': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, c_uint64,
                                            c_uint64, _P, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, c_int]),
    'promp_paths_workspace_bytes': (c_int64, [c_int, c_int, c_int]),
    'promp_paths_finalize': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int64, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                     _P, _P, _P, _P, _P, _P, _P, _P, c_int64, _P]),
    'promp_paths_histogram': (c_int, [c_int, c_int, c_int, _P, _P, _P]),
    'promp_paths_finalize_ex': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int64, _P, _P, _P, _P, _P, _P, _P, _P,
                                        _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64, _P]),
    'promp_counter_add': (c_int, [_P, c_uint64, _P]),
    'promp_set_tasks': (c_int, [c_int, c_int, c_int, _P, _P, _P, _P]),
    'promp_env_step': (c_int, [c_int, c_int, c_float, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'promp_env_observe': (c_int, [c_int, c_int, _P, _P, _P]),
    'promp_process_workspace_bytes': (c_int64, [c_int, c_int, c_int, c_int]),
    'promp_process_samples': (c_int, [c_int, c_int, c_int, c_int, _P, _P, c_double, c_double, c_double, c_int, c_int,
                                      c_int, _P, _P, _P, _P, _P, c_int64, _P]),
    'promp_process_workspace_bytes_ragged': (c_int64, [c_int, c_int, c_int, c_int]),
    'promp_process_samples_ragged': (c_int, [c_int, c_int, c_int, c_int, _P, _P, _P, _P, c_double, c_double, c_double, c_int,
                                             c_int, c_int, _P, _P, _P, _P, _P, c_int64, _P]),
    'promp_process_samples_given': (c_int, [c_int, c_int, c_int, c_int, _P, _P, _P, c_double, c_double, c_int, c_int, _P, _P,
                                            _P, _P, c_int64, _P]),
    'promp_process_samples_ragged_given': (c_int, [c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, c_double, c_double, c_int,
                                                   c_int, _P, _P, _P, _P, c_int64, _P]),
    'promp_process_launch_info': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, _P]),
    'promp_adj_avg_rewards': (c_int, [c_int64, _P, c_double, c_double, _P, _P]),
    'promp_emaml_coeff': (c_int, [c_int, _P, _P, c_int, _P, _P]),
    'promp_emaml_totals': (c_int, [c_int, _P, _P, c_int, _P, _P]),
    'promp_emaml_finish': (c_int, [c_int, _P, _P, c_int, _P, _P, _P]),
    'promp_baseline_fit_workspace_bytes': (c_int64, [c_int, c_int, c_int]),
    'promp_baseline_fit': (c_int, [c_int, c_int, c_int, _P, _P, _P, c_double, _P, _P, _P, c_int64, _P]),
    'promp_baseline_predict': (c_int, [c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    'promp_baseline_fit_ex': (c_int, [c_int, c_int, c_int, c_int, _P, _P, _P, c_double, _P, _P, _P, c_int64, _P]),
    'promp_baseline_predict_ex': (c_int, [c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    'promp_policy_workspace_bytes': (c_int64, [c_int, c_int, c_int, c_int, c_int]),
    'promp_policy_grad': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, _P, _P, c_int, c_int,
                                  c_float, c_float, c_float, c_int, c_float, _P, _P, c_float, _P, _P, c_int64, _P]),
    'promp_policy_hvp': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, _P, _P, c_int, c_int,
                                 c_float, c_float, c_int, c_float, _P, _P, _P, _P, c_int64, _P]),
    'promp_policy_grad_ragged': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, c_int64, _P, _P, _P, _P, _P, c_int, c_int,
                                         c_float, c_float, c_float, c_int, c_float, _P, _P, c_float, _P, _P, c_int64, _P]),
    'promp_policy_grad_ex': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, c_int64, _P, _P, _P, _P, _P, c_int, c_int,
                                     c_float, c_float, c_float, c_int, c_float, _P, _P, c_float, _P, _P, _P, _P, _P, _P, c_int64, _P]),
    'promp_policy_hvp_ragged': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, c_int64, _P, _P, _P, _P, _P, c_int, c_int,
                                        c_float, c_float, c_int, c_float, _P, _P, _P, _P, c_int64, _P]),
    'promp_policy_chain_workspace_bytes': (c_int64, [c_int, c_int, c_int, c_int, c_int, _P]),
    'promp_policy_chain_num_launches': (c_int, [c_int, c_int, c_int, c_int, c_int, _P]),
    'promp_policy_chain_plan_info': (c_int, [c_int, c_int, _P, _P]),
    'promp_policy_chain': (c_int, [c_int, c_int, c_int, c_int, c_float, c_int, _P, _P, _P, _P, c_int64, _P]),
    'promp_meta_loss_terms': (c_int, [c_int, c_int, _P, c_float, _P, c_int, _P, _P]),
    'promp_phase_log_terms': (c_int, [c_int, c_int, c_double, _P, _P, _P, _P]),
    'promp_promp_log_terms': (c_int, [c_int, _P, _P, _P]),
    'promp_adapt_kl_coeff': (c_int, [c_int, _P, c_double, c_int, _P, _P, _P]),
    'promp_reduce_tasks': (c_int, [c_int, c_int, _P, c_float, _P, _P]),
    'promp_reduce_tasks2': (c_int, [c_int, c_int, _P, _P, c_float, _P, _P]),
    'promp_adam_tf1': (c_int, [c_int, _P, _P, _P, _P, _P, c_float, c_float, c_float, c_float, _P]),
    'promp_vec_axpy': (c_int, [c_int, c_float, _P, _P, _P, _P]),
    'promp_cg_init': (c_int, [c_int, _P, _P, _P, _P, _P, _P]),
    'promp_cg_step': (c_int, [c_int, _P, _P, c_float, c_float, _P, _P, _P, _P, c_float, _P]),
    'promp_trpo_step': (c_int, [c_int, _P, _P, c_float, c_float, _P, c_float, _P, _P, _P]),
    'promp_trpo_select': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, c_float, _P, _P, _P, _P, _P, _P]),
    'promp_policy_forward': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P]),
    'promp_policy_layout': (c_int, [c_int, c_int, c_int, _P]),
    'promp_policy_workspace_bytes_padded': (c_int64, [c_int, c_int, c_int, c_int, c_int]),
    'promp_policy_forward_padded': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P]),
    'promp_policy_grad_ex_padded': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, c_int64, _P, _P, _P, _P, _P, c_int, c_int,
                                            c_float, c_float, c_float, c_int, c_float, _P, _P, c_float, _P, _P, _P, _P, _P, _P,
                                            c_int64, _P]),
    'promp_policy_hvp_ragged_padded': (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P, c_int64, _P, _P, _P, _P, _P, c_int,
                                               c_int, c_float, c_float, c_int, c_float, _P, _P, _P, _P, c_int64, _P]),
    'promp_policy_chain_workspace_bytes_padded': (c_int64, [c_int, c_int, c_int, c_int, c_int, _P]),
    'promp_policy_chain_num_launches_padded': (c_int, [c_int, c_int, c_int, c_int, c_int, _P]),
    'promp_policy_chain_padded': (c_int, [c_int, c_int, c_int, c_int, c_float, c_int, _P, _P, _P, _P, c_int64, _P]),
    'promp_set_option': (c_int, [c_char_p, c_int]),
    'promp_comm_buffer_bytes': (c_int64, [c_int, c_int]),
    'promp_comm_alloc': (c_int, [c_int64, _P]),
    'promp_comm_free': (c_int, [_P]),
    'promp_ipc_get_handle': (c_int, [_P, _P]),
    'promp_ipc_open_handle': (c_int, [_P, _P]),
    'promp_ipc_close_handle': (c_int, [_P]),
    'promp_meta_update': (c_int, [c_int, c_int, _P, c_float, _P, _P, _P, _P, _P, c_float, c_float, c_float, c_float, c_int, c_int,
                                  c_int, _P, _P, _P, _P, _P]),
    'promp_reduce_tasks_sgd': (c_int, [c_int, c_int, _P, c_int, _P, _P, c_float, _P, _P]),
    'promp_meta_update_sgd': (c_int, [c_int, c_int, _P, c_int, _P, _P, _P, c_float, _P, _P, _P, _P, _P, _P, _P, _P, c_float,
                                      c_float, c_float, c_float, c_int, c_int, c_int, _P, _P, _P, _P, _P]),
    'promp_meta_loss_terms_p2p': (c_int, [c_int, c_int, _P, c_float, _P, c_int, _P, c_int, c_int, c_int, _P, _P, _P, _P]),
    'promp_allreduce_p2p': (c_int, [c_int, c_int, c_int, c_int, _P, _P, c_float, _P, _P, _P, _P, _P]),
    'promp_env_module_load': (c_int, [_P, c_int64, _P, c_int, _P, _P]),
    'promp_env_module_unload': (c_int, [_P]),
    'promp_rollout_module': (c_int, [_P, c_int, c_float, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, c_uint64,
                                     c_uint64, _P, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int]),
    'promp_rollout_early_term_module': (c_int, [_P, c_int, c_int, c_int, c_int, c_int, c_int, _P, c_int64, _P, _P, _P, c_uint64,
                                                c_uint64, _P, c_int, c_float, _P, _P, _P, _P, _P, _P, _P, c_int]),
    'promp_env_step_module': (c_int, [_P, c_int, c_float, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    'promp_env_observe_module': (c_int, [_P, c_int, _P, _P, _P]),
    'promp_cuda_build_version': (c_int, []),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib = None


class PrompLibraryError(RuntimeError):
    pass


def load():
    """Load the shared library (once).  Raises ImportError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                "promp_b200: %s is missing. Build it with `python -m promp_b200._build` (needs nvcc; "
                "sm_90a). There is no CPU fallback." % LIB_PATH)
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)        # AttributeError here = header / library out of sync
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error():
    return load().promp_last_error().decode('utf-8', 'replace')


def check(status, what):
    if status != 0:
        raise PrompLibraryError("%s failed (status %d): %s" % (what, status, last_error()))


def ptr(t):
    """Device pointer of a torch tensor (or None -> NULL).  Tensors must be contiguous CUDA tensors."""
    if t is None:
        return None
    if not t.is_cuda:
        raise PrompLibraryError("promp_b200 kernels need CUDA tensors (got a %s tensor); there is no CPU fallback"
                                % t.device)
    if not t.is_contiguous():
        raise PrompLibraryError("promp_b200 kernels need contiguous tensors")
    return t.data_ptr()


def ptr_array(tensors):
    """Host array of device pointers (the lam / g arguments of promp_meta_update_sgd / promp_reduce_tasks_sgd)."""
    return (c_void_p * max(len(tensors), 1))(*[ptr(t) for t in tensors])


def stream():
    """Raw cudaStream_t of torch's current stream on the current device (the fast private accessor when available:
    torch.cuda.current_stream() costs ~15 us per call, which at ~35 launches per meta-iteration is 0.5 ms of host time)."""
    import torch
    raw = getattr(torch._C, '_cuda_getCurrentRawStream', None)
    if raw is not None:
        return raw(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise PrompLibraryError("promp_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    load()


def set_option(name, value):
    check(load().promp_set_option(name.encode(), int(value)), 'promp_set_option')


def call(name, *args):
    check(getattr(load(), name)(*args), name)


def policy_layout(obs_dim, act_dim, hidden):
    """(obs_cap, act_cap, hidden, P) of the zero-padded parameter layout of the *_padded policy entry points
    (promp_policy_layout)."""
    out = (c_int32 * 4)()
    check(load().promp_policy_layout(int(obs_dim), int(act_dim), int(hidden), ctypes.cast(out, c_void_p)), 'promp_policy_layout')
    return tuple(int(v) for v in out)
