"""CPU: the C-ABI library builds, loads and exports every symbol include/scalerl_b200.h declares (no compute)."""
import ctypes
import os
import re

import pytest

from scalerl_b200 import _lib, build as srl_build

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return ctypes.CDLL(_lib.LIB_PATH)


def _declared():
    src = open(os.path.join(ROOT, 'include', 'scalerl_b200.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    return sorted(set(re.findall(r'\b(srl_[a-z0-9_]+)\s*\(', src)))


def test_header_symbols_exported(lib):
    names = _declared()
    assert len(names) >= 20
    for n in names:
        assert hasattr(lib, n), f'{n} declared in include/scalerl_b200.h but not exported'
    assert sorted(_lib.EXPORTS) == names, 'ctypes binding table and header disagree'


def test_testhooks_library_is_separate():
    """unit-test entry points live in libscalerl_b200_testhooks.so, declared in their own header; the product library
    exports none of them"""
    src = open(os.path.join(ROOT, 'include', 'scalerl_b200_testhooks.h')).read()
    src = re.sub(r'/\*.*?\*/', '', src, flags=re.S)
    names = sorted(set(re.findall(r'\b(srl_[a-z0-9_]+)\s*\(', src)))
    srl_build.build()
    H = ctypes.CDLL(_lib.HOOKS_PATH)
    P = ctypes.CDLL(_lib.LIB_PATH)
    assert names == sorted(_lib.HOOK_EXPORTS)
    for n in names:
        assert hasattr(H, n), n
        assert not hasattr(P, n), f'{n} must not ship in the product library'


def test_action_count_limit():
    """A = 32 would need a 33rd warp lane for the baseline: rejected at creation (ADVICE r1)"""
    L = _lib.lib()
    cfg = _lib.SrlConfig()
    cfg.T, cfg.B, cfg.A = 20, 32, 32
    h = ctypes.c_void_p()
    assert L.srl_learner_create(ctypes.byref(cfg), None, None, None, None, ctypes.byref(h)) == -1
    assert b'[1,31]' in L.srl_last_error()


def test_param_layout_matches_atarinet():
    total, off, cnt = _lib.param_layout(6)
    assert sum(cnt) == 1687768        # AtariNet((4,84,84), 6) parameter count (SURVEY.md §8)
    assert all(o % 4 == 0 for o in off) and total >= sum(cnt)
    total4, _, cnt4 = _lib.param_layout(4)
    assert sum(cnt4) == 1686718


def test_config_struct_size():
    assert ctypes.sizeof(_lib.SrlConfig) == 19 * 4


def test_dp_peers_struct_and_argument_checks():
    """srl_dp_peers_t: 3 x 8 pointers + rank + world + the NVLS multicast pointer; bad descriptors are rejected before any CUDA call"""
    assert ctypes.sizeof(_lib.SrlDpPeers) == 3 * 8 * 8 + 8 + 8
    L = _lib.lib()
    assert L.srl_learner_apply_gradients_dp(None, None, None, None) == -1
    assert b'NULL' in L.srl_last_error()


def test_bench_roofline_tables_are_consistent():
    """bench.py's algorithmic flops / bytes tables: same kernels, intensities in the range DESIGN.md quotes"""
    import importlib.util
    spec = importlib.util.spec_from_file_location('bench_mod', os.path.join(ROOT, 'bench.py'))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    assert set(b.SLOT_FLOPS) == set(b.SLOT_BYTES)
    NF, NB = 21 * 32, 20 * 32
    ai = {}
    for slot, (layer, which) in b.SLOT_FLOPS.items():
        n = NF if which == 'fwd' else NB
        ai[slot] = 2.0 * b.MACS[layer] * n / (b.SLOT_BYTES[slot][0] * n + b.SLOT_BYTES[slot][1])
    assert 75 < ai['conv1_wgrad'] < 85 and 75 < ai['conv1_fwd'] < 85 and 140 < ai['conv2_fwd'] < 155 and 205 < ai['conv3_fwd'] < 225
    assert all(v < 600 for v in ai.values())


def test_argument_errors_without_gpu(lib):
    L = _lib.lib()
    # NULL pointers / bad shapes are rejected before any CUDA call
    assert L.srl_vtrace_from_importance_weights(None, None, None, None, None, 4, 4, 1.0, 1.0, None, None, 0, None) == -1
    assert b'NULL' in L.srl_last_error()
    assert L.srl_vtrace_from_importance_weights(None, None, None, None, None, 0, 4, 1.0, 1.0, None, None, 0, None) == 0  # empty
    cfg = _lib.SrlConfig()
    cfg.T, cfg.B, cfg.A = 20, 32, 99
    h = ctypes.c_void_p()
    assert L.srl_learner_create(ctypes.byref(cfg), None, None, None, None, ctypes.byref(h)) == -1
    assert b'A=99' in L.srl_last_error()


def test_one_error_message_per_library(lib):
    """the replay sampler reports through srl_last_error (srl_per_last_error returns the same message); the test-hook library keeps
    a message of its own"""
    L, H = _lib.lib(), _lib.hooks()
    h = ctypes.c_void_p()
    assert H.srl_test_shifted_operand(None, None, None, 0, 0, 0, None) == -1
    assert L.srl_vtrace_from_importance_weights(None, None, None, None, None, 4, 4, 1.0, 1.0, None, None, 0, None) == -1
    assert L.srl_per_create(1, 0.6, ctypes.byref(h)) == -1
    msg = L.srl_last_error()
    assert msg.startswith(b'per_create: ') and b'memory_size' in msg
    assert L.srl_per_last_error() == msg
    assert H.srl_test_last_error().startswith(b'test_shifted_operand: ')


def test_timeline_entry_is_inert_in_the_product_build(lib):
    """srl_debug_kernel_timeline only works in a diagnostics build (SRL_DEFINES=SRL_KSTAMP): the shipped library refuses, without touching CUDA"""
    L = _lib.lib()
    assert L.srl_debug_kernel_timeline(None) != 0
    assert b'SRL_KSTAMP' in L.srl_last_error()


def test_product_path_has_no_oracle_import():
    """the shipped package must never import the oracle or fall back to CPU"""
    pkg = os.path.join(ROOT, 'scalerl_b200')
    for dp, _, fs in os.walk(pkg):
        for f in fs:
            if f.endswith('.py'):
                s = open(os.path.join(dp, f)).read()
                assert 'import oracle' not in s and 'from oracle' not in s, f
