"""The LSTM actor step without a GPU: its kernels fit the register file (ptxas log of the build) and its entry point rejects bad
pointers before it touches the context or a device."""
import ctypes
import os

import pytest

from scalerl_b200 import _lib, build as B

STEP_KERNELS = ('lstm_step_kernel', 'lstm_step_pack_kernel', 'lstm_step_prep_kernel')


@pytest.fixture(scope='module')
def report():
    path = os.path.join(B.HERE, 'build', 'ptxas.log')
    if not os.path.exists(path):
        B.build(force=True)
    return B.ptxas_report(path)


def test_step_kernels_do_not_spill(report):
    kernels = {k: v for k, v in report['lstm.cu'].items() if any(n in k for n in STEP_KERNELS)}
    # the step GEMM in its four cluster sizes (K split 1, 2, 3, 6), the operand kernel and the pack kernel
    assert len([k for k in kernels if 'lstm_step_kernel' in k]) == 4 and len(kernels) == 6, sorted(kernels)
    spills = {k: (v['spill_stores'], v['spill_loads']) for k, v in kernels.items() if v['spill_stores'] or v['spill_loads']}
    assert not spills, f'spilling LSTM step kernels (bytes stored, loaded): {spills}'
    assert not any(v['serialized'] for v in kernels.values())


def _call(L, ptrs, **over):
    a = dict(zip(('obs', 'reward', 'done', 'action', 'h_in', 'c_in', 'logits', 'baseline', 'h_out', 'c_out'), ptrs))
    a.update(over)
    return _lib.lib().srl_learner_forward_lstm_step(L, a['obs'], a['reward'], a['done'], a['action'], a['h_in'], a['c_in'], a['logits'],
                                                    a['baseline'], a['h_out'], a['c_out'], None)


def test_step_argument_errors_without_gpu():
    """NULL or aliased pointers give SRL_EINVAL before the context is read (the addresses below are never dereferenced)"""
    B.build()
    ptrs = [0x10000 * (i + 1) for i in range(10)]
    lib = _lib.lib()
    for k in ('obs', 'done', 'h_in', 'c_out'):
        assert _call(None, ptrs, **{k: None}) == -1
        assert b'NULL pointer' in lib.srl_last_error()
    h_in, c_in, h_out, c_out = ptrs[4], ptrs[5], ptrs[8], ptrs[9]
    for over in ({'h_out': h_in}, {'h_out': c_in}, {'c_out': h_in}, {'c_out': c_in}, {'c_out': h_out}):
        dummy = ctypes.c_void_p(0x1234)          # not a context: the alias check must come first
        assert _call(dummy, ptrs, **over) == -1
        assert b'must not alias' in lib.srl_last_error()
    assert _call(None, ptrs) == -1
    assert b'learner is NULL' in lib.srl_last_error()
    assert 'srl_learner_forward_lstm_step' in _lib.EXPORTS
