"""ctypes binding of libscalerl_b200.so (the C ABI declared in include/scalerl_b200.h).

The product path has NO CPU fallback: if the shared library is missing this module raises at import
of the first op (build it with ``python -m scalerl_b200.build`` or ``__graft_entry__.build()``).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libscalerl_b200.so')

_lib = None


class SrlDpPeers(C.Structure):
    """mirror of srl_dp_peers_t: peer-mapped gradient buffers and control blocks of a data-parallel group (<= 8 ranks)"""
    _fields_ = [('grads', C.c_void_p * 8), ('exchange', C.c_void_p * 8), ('ctl', C.c_void_p * 8), ('rank', C.c_int32), ('world', C.c_int32),
                ('grads_multicast', C.c_void_p)]


class SrlConfig(C.Structure):
    """mirror of srl_config_t"""
    _fields_ = [('T', C.c_int32), ('B', C.c_int32), ('A', C.c_int32), ('optimizer', C.c_int32),
                ('reward_clip_abs_one', C.c_int32), ('precision', C.c_int32),
                ('discounting', C.c_float), ('baseline_cost', C.c_float), ('entropy_cost', C.c_float),
                ('clip_rho_threshold', C.c_float), ('clip_pg_rho_threshold', C.c_float),
                ('max_grad_norm', C.c_float), ('learning_rate', C.c_float), ('alpha', C.c_float), ('epsilon', C.c_float),
                ('adam_beta1', C.c_float), ('adam_beta2', C.c_float), ('adam_eps', C.c_float), ('use_lstm', C.c_int32)]


_P, _I, _F, _L = C.c_void_p, C.c_int, C.c_float, C.c_int64

# name -> argtypes; every function returns int except where noted
_SIGS = {
    'srl_vtrace_from_importance_weights': [_P, _P, _P, _P, _P, _I, _I, _F, _F, _P, _P, _I, _P],
    'srl_vtrace_from_logits': [_P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _F, _P, _P, _P, _P, _P, _P],
    'srl_impala_loss_and_head_grads': [_P, _P, _P, _P, _P, _P, _I, _I, _I, _F, _I, _F, _F, _F, _F, _P, _P, _P, _P, _P, _P, _P],
    'srl_policy_rows_forward': [_P, _P, _L, _I, _P, _P, _P],
    'srl_policy_rows_backward': [_P, _P, _P, _P, _L, _I, _P, _P],
    'srl_reduce_sum': [_P, _L, _I, _F, _P, _P],
    'srl_sample_actions': [_P, _P, _L, _I, _P, _P],
    'srl_learner_create': [C.POINTER(SrlConfig), _P, _P, _P, _P, C.POINTER(_P)],
    'srl_learner_destroy': [_P],
    'srl_learner_set_config': [_P, C.POINTER(SrlConfig)],
    'srl_learner_pack_weights': [_P, _P],
    'srl_debug_kernel_timeline': [_P],
    'srl_learner_forward': [_P, _P, _P, _P, _I, _P, _P, _P],
    'srl_learner_forward_backward': [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    'srl_learner_forward_backward_begin': [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    'srl_learner_backward_finish': [_P, _P, _P],
    'srl_learner_forward_lstm': [_P] * 12,
    'srl_learner_forward_backward_lstm': [_P] * 12,
    'srl_learner_forward_lstm_step': [_P] * 12,
    'srl_learner_apply_gradients': [_P, _P, _P],
    'srl_learner_apply_gradients_dp': [_P, _P, _P, _P],
    'srl_learner_debug_buffer': [_P, C.c_char_p, C.POINTER(_P), C.POINTER(_L)],
    'srl_lstm_create': [_I, _I, _I, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P)],
    'srl_lstm_destroy': [_P],
    'srl_lstm_forward': [_P, _P, _P, _P, _P, _P, _P, _P, _P],
    'srl_lstm_backward': [_P, _P, _P, _P, _P],
    'srl_per_create': [_L, C.c_double, C.POINTER(_P)],
    'srl_per_destroy': [_P],
    'srl_per_add': [_P, _L, _P],
    'srl_per_update_priorities': [_P, _P, _P, _L, _P],
    'srl_per_sample': [_P, _P, _I, C.c_double, _P, _P, _P, _P],
    'srl_per_debug_trees': [_P, _P, _P, _P, _P],
    'srl_unpack_slots': [_P, _L, C.POINTER(_L), _I, _I, _I, _P, _P, _P, _P, _P, _P, _P],
    'srl_grad_norm_clip_coef': [_P, _L, _F, _P, _P, _P],
    'srl_rmsprop_step': [_P, _P, _P, _L, _P, _F, _F, _F, _P],
    'srl_adam_step': [_P, _P, _P, _P, _L, _P, _F, _F, _F, _F, _I, _P],
    'srl_learner_set_option': [_P, C.c_char_p, _I],
    'srl_learner_snapshot_params': [_P, _P, _P, _P],
    'srl_learner_set_step': [_P, _L, _P],
    'srl_learner_set_lr_schedule': [_P, _I, _F, C.c_double, C.c_double],
    'srl_learner_set_momentum': [_P, _F, _P],
    'srl_memcpy_d2d': [_P, _P, _L, _P],
    'srl_host_register': [_P, _L],
    'srl_host_unregister': [_P],
    'srl_learner_set_profiling': [_P, _I],
    'srl_profile_slot_count': [],
    'srl_learner_profile_collect': [_P, _P],
    'srl_version': [],
}
# libscalerl_b200_testhooks.so (include/scalerl_b200_testhooks.h): unit-test entry points, loaded by tests only
_HOOK_SIGS = {
    'srl_test_shifted_operand': [_P, _P, _P, _I, _I, _I, _P],
    'srl_test_poison_smem': [_P],
    'srl_test_pdl': [_P, _P, _I, C.c_uint, _P],
}
HOOK_EXPORTS = sorted(list(_HOOK_SIGS) + ['srl_test_last_error'])
HOOKS_PATH = os.path.join(_HERE, 'libscalerl_b200_testhooks.so')
_hooks = None


def hooks():
    """the test-hook library (tests only; the product path never loads it)"""
    global _hooks
    if _hooks is None:
        if not os.path.exists(HOOKS_PATH):
            raise RuntimeError(f'{HOOKS_PATH} is missing: build it with python -m scalerl_b200.build')
        H = C.CDLL(HOOKS_PATH)
        for name, args in _HOOK_SIGS.items():
            fn = getattr(H, name)
            fn.argtypes = args
            fn.restype = C.c_int
        H.srl_test_last_error.restype = C.c_char_p
        H.srl_test_last_error.argtypes = []
        _hooks = H
    return _hooks


def check_hook(rc, what=''):
    if rc != 0:
        msg = hooks().srl_test_last_error().decode()
        raise (ValueError if rc == -1 else RuntimeError)(f'{what}: rc={rc}: {msg}')


EXPORTS = sorted(list(_SIGS) + ['srl_last_error', 'srl_param_layout', 'srl_param_layout_ex', 'srl_learner_workspace_bytes', 'srl_profile_slot_name', 'srl_lstm_last_error', 'srl_per_last_error', 'srl_per_size', 'srl_per_capacity', 'srl_per_invalid_updates', 'srl_learner_get_step'])


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(f'{LIB_PATH} is missing: the CUDA library must be built (python -m scalerl_b200.build); '
                               'scalerl_b200 has no CPU fallback')
        L = C.CDLL(LIB_PATH)
        for name, args in _SIGS.items():
            fn = getattr(L, name)
            fn.argtypes = args
            fn.restype = C.c_int
        L.srl_last_error.restype = C.c_char_p
        L.srl_last_error.argtypes = []
        L.srl_param_layout.restype = C.c_int64
        L.srl_param_layout.argtypes = [_I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_param_layout_ex.restype = C.c_int64
        L.srl_param_layout_ex.argtypes = [_I, _I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_per_last_error.restype = C.c_char_p
        L.srl_per_last_error.argtypes = []
        for nm in ('srl_per_size', 'srl_per_capacity'):
            getattr(L, nm).restype = C.c_int64
            getattr(L, nm).argtypes = [_P]
        L.srl_learner_get_step.restype = C.c_int64
        L.srl_learner_get_step.argtypes = [_P, _P]
        L.srl_per_invalid_updates.restype = C.c_int64
        L.srl_per_invalid_updates.argtypes = [_P, _P]
        L.srl_lstm_last_error.restype = C.c_char_p
        L.srl_lstm_last_error.argtypes = []
        L.srl_profile_slot_name.restype = C.c_char_p
        L.srl_profile_slot_name.argtypes = [_I]
        L.srl_learner_workspace_bytes.restype = C.c_int64
        L.srl_learner_workspace_bytes.argtypes = [_P]
        _lib = L
    return _lib


def check(rc, what=''):
    if rc != 0:
        msg = lib().srl_last_error().decode()
        if rc == -1:
            raise ValueError(f'{what}: {msg}')
        raise RuntimeError(f'{what}: rc={rc}: {msg}')


def param_layout(A, use_lstm=False):
    """(total floats, offsets, counts) of the flat parameter buffer; 12 AtariNet tensors (+ 8 nn.LSTM tensors with use_lstm)"""
    off = (_L * 20)()
    cnt = (_L * 20)()
    total = lib().srl_param_layout_ex(int(A), 1 if use_lstm else 0, off, cnt)
    n = 20 if use_lstm else 12
    return int(total), [int(x) for x in off][:n], [int(x) for x in cnt][:n]
