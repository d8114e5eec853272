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
    'srl_encoder_create': [_I, C.POINTER(_P)],
    'srl_encoder_destroy': [_P],
    'srl_encoder_sizes': [_I, _I, C.POINTER(_L), C.POINTER(_L)],
    'srl_encoder_forward': [_P, _P, _P, _P, _I, _I, C.POINTER(_P), _P, _P, _P, _P],
    'srl_encoder_backward': [_P, _P, _I, _I, _P, _P, C.POINTER(_P), _P],
    'srl_lstm_create': [_I, _I, _I, C.POINTER(_P), C.POINTER(_P), C.POINTER(_P)],
    'srl_lstm_destroy': [_P],
    'srl_lstm_forward': [_P, _P, _P, _P, _P, _P, _P, _P, _P],
    'srl_lstm_backward': [_P, _P, _P, _P, _P],
    'srl_lstm_core_sizes': [_I, _I, _I, C.POINTER(_L), C.POINTER(_L)],
    'srl_lstm_core_forward': [_P, _P, _P, _P, _I, _I, _I, C.POINTER(_P), _P, _P, _P, _P, _P, _P],
    'srl_lstm_core_backward': [_P, _P, _P, _I, _I, _I, _P, _P, C.POINTER(_P), _P, _P, _P, _P],
    'srl_lstm_core_debug_buffer': [_I, _I, _I, _P, _P, C.c_char_p, _I, C.POINTER(_P), C.POINTER(_L)],
    'srl_lstm_debug_buffer': [_P, C.c_char_p, _I, C.POINTER(_P), C.POINTER(_L)],
    'srl_per_create': [_L, C.c_double, C.POINTER(_P)],
    'srl_per_destroy': [_P],
    'srl_per_add': [_P, _L, _P],
    'srl_per_update_priorities': [_P, _P, _P, _L, _P],
    'srl_per_sample': [_P, _P, _I, C.c_double, _P, _P, _P, _P],
    'srl_per_debug_trees': [_P, _P, _P, _P, _P],
    'srl_replay_create': [_L, _I, _I, C.c_double, C.c_double, C.POINTER(_P)],
    'srl_replay_destroy': [_P],
    'srl_replay_add': [_P] * 7,
    'srl_replay_sample': [_P, _P, _I] + [_P] * 9,
    'srl_replay_gather': [_P, _P, _L] + [_P] * 6,
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
    'srl_apex_learner_create': [C.c_void_p, _P, _P, _P, _P, _P, C.POINTER(_P)],
    'srl_apex_learner_destroy': [_P],
    'srl_apex_learner_step': [_P] * 11,
    'srl_apex_learner_update_target': [_P, _F, _P],
    'srl_apex_learner_set_step': [_P, _L, _P],
    'srl_apex_learner_q_values': [_P, _P, _I, _P, _P],
    'srl_apex_learner_debug_buffer': [_P, C.c_char_p, C.POINTER(_P), C.POINTER(_L)],
    'srl_apex_actor_create': [_I, _I, _I, C.c_uint64, _P, C.POINTER(_P)],
    'srl_apex_actor_create_ex': [_I, _I, _I, _I, C.c_uint64, _P, C.POINTER(_P)],
    'srl_apex_actor_create_cat': [_I, _I, _I, _I, _F, _F, C.c_uint64, _P, C.POINTER(_P)],
    'srl_apex_actor_create_noisy': [_I, _I, _I, _I, _I, _F, _F, _I, C.c_uint64, _P, C.POINTER(_P)],
    'srl_apex_actor_create_quantile': [_I, _I, _I, _I, _I, _F, _F, _I, _F, _I, C.c_uint64, _P, C.POINTER(_P)],
    'srl_apex_actor_create_dist_dueling': [_I, _I, _I, _I, _I, _F, _F, _I, _F, _I, _I, C.c_uint64, _P, C.POINTER(_P)],
    'srl_apex_actor_debug_buffer': [_P, C.c_char_p, C.POINTER(_P), C.POINTER(_L)],
    'srl_apex_actor_destroy': [_P],
    'srl_apex_actor_act': [_P] * 5,
    'srl_apex_actor_q_values': [_P, _P, _I, _P, _P],
    'srl_replay_add_prioritized': [_P] * 7 + [_F, _P],
    'srl_frame_replay_create': [_L, _I, _I, C.c_double, C.c_double, _L, C.POINTER(_P)],
    'srl_frame_replay_destroy': [_P],
    'srl_frame_replay_add': [_P] * 7,
    'srl_frame_replay_add_prioritized': [_P] * 7 + [_F, _P],
    'srl_frame_replay_sample': [_P, _P, _I] + [_P] * 9,
    'srl_frame_replay_gather': [_P, _P, _L] + [_P] * 6,
    'srl_r2d2_learner_create': [C.c_void_p, _P, _P, _P, _P, _P, C.POINTER(_P)],
    'srl_r2d2_learner_destroy': [_P],
    'srl_r2d2_learner_step': [_P] * 12,
    'srl_r2d2_learner_q_values': [_P, _P, _P, _P, _P, _I, _I, _P, _P, _P, _P, _P, _P],
    'srl_r2d2_learner_update_target': [_P, _F, _P],
    'srl_r2d2_learner_set_step': [_P, _L, _P],
    'srl_r2d2_learner_debug_buffer': [_P, C.c_char_p, C.POINTER(_P), C.POINTER(_L)],
}
# libscalerl_b200_testhooks.so (include/scalerl_b200_testhooks.h): unit-test entry points, loaded by tests only
_HOOK_SIGS = {
    'srl_test_shifted_operand': [_P, _P, _P, _I, _I, _I, _P],
    'srl_test_poison_smem': [_P],
    'srl_test_pdl': [_P, _P, _I, C.c_uint, _P],
    'srl_test_clip_optim': [_I, _P, _P, _P, _P, _L, _F, _P, _P, _F, _F, _F, _F, _I, _P, _I, _F, C.c_double, C.c_double, _P, _F, _P, _P, _P],
    'srl_test_encoder_row': [_I, _I, C.c_char_p, _P, _P, C.POINTER(_P), C.POINTER(_P), C.POINTER(_L)],
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


EXPORTS = sorted(list(_SIGS) + ['srl_last_error', 'srl_param_layout', 'srl_param_layout_ex', 'srl_learner_workspace_bytes', 'srl_profile_slot_name', 'srl_lstm_last_error', 'srl_per_last_error', 'srl_per_size', 'srl_per_capacity', 'srl_per_invalid_updates', 'srl_learner_get_step', 'srl_apex_param_layout', 'srl_apex_param_layout_ex', 'srl_apex_param_layout_cat', 'srl_apex_param_layout_noisy', 'srl_apex_param_layout_quantile', 'srl_apex_param_layout_dist_dueling', 'srl_replay_size', 'srl_replay_per', 'srl_frame_replay_size', 'srl_frame_replay_per', 'srl_frame_replay_frames_allocated', 'srl_frame_replay_retired', 'srl_r2d2_param_layout'])


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
        L.srl_replay_size.restype = C.c_int64
        L.srl_replay_size.argtypes = [_P]
        L.srl_replay_per.restype = _P
        L.srl_replay_per.argtypes = [_P]
        L.srl_frame_replay_size.restype = C.c_int64
        L.srl_frame_replay_size.argtypes = [_P]
        L.srl_frame_replay_per.restype = _P
        L.srl_frame_replay_per.argtypes = [_P]
        for nm in ('srl_frame_replay_frames_allocated', 'srl_frame_replay_retired'):
            getattr(L, nm).restype = C.c_int64
            getattr(L, nm).argtypes = [_P, _P]
        L.srl_learner_get_step.restype = C.c_int64
        L.srl_learner_get_step.argtypes = [_P, _P]
        L.srl_per_invalid_updates.restype = C.c_int64
        L.srl_per_invalid_updates.argtypes = [_P, _P]
        L.srl_lstm_last_error.restype = C.c_char_p
        L.srl_lstm_last_error.argtypes = []
        L.srl_profile_slot_name.restype = C.c_char_p
        L.srl_profile_slot_name.argtypes = [_I]
        L.srl_apex_param_layout.restype = C.c_int64
        L.srl_apex_param_layout.argtypes = [_I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_apex_param_layout_ex.restype = C.c_int64
        L.srl_apex_param_layout_ex.argtypes = [_I, _I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_apex_param_layout_cat.restype = C.c_int64
        L.srl_apex_param_layout_cat.argtypes = [_I, _I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_apex_param_layout_noisy.restype = C.c_int64
        L.srl_apex_param_layout_noisy.argtypes = [_I, _I, _I, _I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_apex_param_layout_quantile.restype = C.c_int64
        L.srl_apex_param_layout_quantile.argtypes = [_I, _I, _I, _I, _I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_apex_param_layout_dist_dueling.restype = C.c_int64
        L.srl_apex_param_layout_dist_dueling.argtypes = [_I, _I, _I, _I, _I, _I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_r2d2_param_layout.restype = C.c_int64
        L.srl_r2d2_param_layout.argtypes = [_I, _I, C.POINTER(_L), C.POINTER(_L)]
        L.srl_learner_workspace_bytes.restype = C.c_int64
        L.srl_learner_workspace_bytes.argtypes = [_P]
        _lib = L
    return _lib


def check(rc, what='', last_error=None):
    """raises on a non-zero return code: ValueError for a bad argument (SRL_EINVAL), RuntimeError otherwise, with the library's
    message (``last_error``: its getter, the product library's srl_last_error by default)"""
    if rc != 0:
        msg = (last_error or lib().srl_last_error)().decode()
        if rc == -1:
            raise ValueError(f'{what}: {msg}')
        raise RuntimeError(f'{what}: rc={rc}: {msg}')


def check_hook(rc, what=''):
    """check() for the test-hook library"""
    check(rc, what, hooks().srl_test_last_error)


class SrlApexConfig(C.Structure):
    """mirror of srl_apex_config_t"""
    _fields_ = [('B', C.c_int32), ('A', C.c_int32), ('precision', C.c_int32), ('double_dqn', C.c_int32),
                ('gamma', C.c_float), ('max_grad_norm', C.c_float), ('learning_rate', C.c_float), ('adam_beta1', C.c_float),
                ('adam_beta2', C.c_float), ('adam_eps', C.c_float), ('priority_eps', C.c_float), ('dueling', C.c_int32),
                ('num_atoms', C.c_int32), ('v_min', C.c_float), ('v_max', C.c_float), ('noisy', C.c_int32), ('noise_seed', C.c_uint64),
                ('num_quantiles', C.c_int32), ('kappa', C.c_float), ('dist_dueling', C.c_int32)]


def apex_param_layout(A, dueling=False, num_atoms=0, noisy=False, num_quantiles=0, dist_dueling=False):
    """(total floats, offsets, counts) of the Ape-X Q network's flat buffer in state_dict order (srl_apex_param_layout_dist_dueling):
    10 tensors, or 12 with the dueling head; num_atoms > 0: the categorical head's 10 (q.weight [A num_atoms, 512], q.bias
    [A num_atoms]); num_quantiles > 0: the quantile head's 10 (q.weight [A num_quantiles, 512], q.bias [A num_quantiles]);
    dist_dueling: either head's 12 as value [W, 512] and advantage [A W, 512] (W = num_atoms or num_quantiles); noisy: 14, or 18 with
    value and advantage"""
    off = (_L * 18)()
    cnt = (_L * 18)()
    total = lib().srl_apex_param_layout_dist_dueling(int(A), 1 if dueling else 0, int(num_atoms), int(num_quantiles), 1 if dist_dueling else 0,
                                                     1 if noisy else 0, off, cnt)
    if total < 0:
        check(-1, 'srl_apex_param_layout_dist_dueling')
    n = 6 + (3 if dueling or dist_dueling else 2) * (4 if noisy else 2)
    return int(total), [int(x) for x in off][:n], [int(x) for x in cnt][:n]


def apex_actor_create(A, num_envs, precision, seed, params, head) -> C.c_void_p:
    """srl_apex_actor_create_dist_dueling for ``head`` (dueling, num_atoms, v_min, v_max, num_quantiles, kappa, dist_dueling, noisy)
    on the device buffer at ``params``"""
    h = C.c_void_p()
    check(lib().srl_apex_actor_create_dist_dueling(A, num_envs, precision, int(head.dueling), head.num_atoms, head.v_min, head.v_max,
                                                   head.num_quantiles, head.kappa, int(head.dist_dueling), int(head.noisy), seed, params,
                                                   C.byref(h)),
          'srl_apex_actor_create_dist_dueling')
    return h


class SrlR2d2Config(C.Structure):
    """mirror of srl_r2d2_config_t"""
    _fields_ = [('B', C.c_int32), ('A', C.c_int32), ('burn_in', C.c_int32), ('T', C.c_int32), ('n_step', C.c_int32), ('gamma', C.c_float),
                ('dueling', C.c_int32), ('value_rescaling', C.c_int32), ('rescale_eps', C.c_float), ('priority_eta', C.c_float),
                ('priority_eps', C.c_float), ('max_grad_norm', C.c_float), ('learning_rate', C.c_float), ('adam_beta1', C.c_float),
                ('adam_beta2', C.c_float), ('adam_eps', C.c_float)]


def r2d2_param_layout(A, dueling=False):
    """(total floats, offsets, counts) of the R2D2 Q network's flat buffer in state_dict order (srl_r2d2_param_layout): 18 tensors, or
    20 with the dueling head"""
    off = (_L * 20)()
    cnt = (_L * 20)()
    total = lib().srl_r2d2_param_layout(int(A), 1 if dueling else 0, off, cnt)
    if total < 0:
        check(-1, 'srl_r2d2_param_layout')
    n = 20 if dueling else 18
    return int(total), [int(x) for x in off][:n], [int(x) for x in cnt][:n]


def param_layout(A, use_lstm=False):
    """(total floats, offsets, counts) of the flat parameter buffer; 12 AtariNet tensors (+ 8 nn.LSTM tensors with use_lstm)"""
    off = (_L * 20)()
    cnt = (_L * 20)()
    total = lib().srl_param_layout_ex(int(A), 1 if use_lstm else 0, off, cnt)
    n = 20 if use_lstm else 12
    return int(total), [int(x) for x in off][:n], [int(x) for x in cnt][:n]
