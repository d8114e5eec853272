"""CPU: the replay memory's oracle against the reference-pinned fixture, and the argument checks that need no GPU."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from oracle import replay_oracle as O
from scalerl_b200 import _lib, build as srl_build
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
from tests.conftest import GOLDEN


def test_oracle_reproduces_reference_fixture():
    """the oracle's ring (fold, env order, wrap-around) equals the reference's PrioritizedReplayBuffer mapped to tree leaves"""
    z = np.load(os.path.join(GOLDEN, 'replay_cases.npz'))
    for ci, case in enumerate(O.CASES):
        M, E, n, dr, steps, seed, size, ptr = z[f'c{ci}_meta']
        assert (int(M), int(E), int(n), float(dr), int(steps), int(seed)) == case
        table, tree_ptr = O.run_case(*case)
        assert tree_ptr == int(ptr) and len(table['action']) == int(size)
        for k, v in table.items():
            assert np.array_equal(v, z[f'c{ci}_{k}']), (case, k)


def test_fold_rounds_like_numpy_float32():
    """r0 + r1 * fp32(g) + r2 * fp32(g^2) with each operation rounded in fp32, stopping after the first done"""
    w = [((0, 0), 0, np.float32(1.1), 'a', 0), ((1, 0), 0, np.float32(-0.7), 'b', 0), ((2, 0), 0, np.float32(0.3), 'c', 1)]
    s, a, r, ns, d = O.fold(w, 0.99)
    g1, g2 = np.float32(0.99), np.float32(0.99 ** 2)
    assert r == np.float32(np.float32(np.float32(1.1) + np.float32(np.float32(-0.7) * g1)) + np.float32(np.float32(0.3) * g2))
    assert (s, ns, d) == ((0, 0), 'c', 1)
    w[0] = ((0, 0), 0, np.float32(1.1), 'a', 1)                   # done at the oldest step: nothing folds
    assert O.fold(w, 0.99)[2:] == (np.float32(1.1), 'a', 1)


@pytest.mark.parametrize('kw', [dict(memory_size=1, num_envs=1), dict(memory_size=2.5, num_envs=1), dict(memory_size=8, num_envs=0),
                                dict(memory_size=8, num_envs=9), dict(memory_size=8, num_envs=2, n_step=0),
                                dict(memory_size=8, num_envs=2, n_step=33), dict(memory_size=8, num_envs=2, gamma=float('nan')),
                                dict(memory_size=8, num_envs=2, alpha=float('inf'))])
def test_constructor_arguments_raise_without_gpu(kw):
    with pytest.raises(ValueError):
        GpuPrioritizedReplayBuffer(**kw)


def _unbuilt(num_envs):
    """a memory object with only its host attributes (the shape and dtype checks run before any device work)"""
    m = GpuPrioritizedReplayBuffer.__new__(GpuPrioritizedReplayBuffer)
    m.num_envs, m.device, m._h = num_envs, torch.device('cuda', 0), None
    return m


@pytest.mark.parametrize('field,value', [('state', np.zeros((3, 4, 84, 84), np.uint8)), ('state', np.zeros((2, 4, 84, 84), np.float32)),
                                         ('next_state', np.zeros((2, 84, 84), np.uint8)), ('action', np.zeros(2, np.float32)),
                                         ('action', np.zeros((2, 1), np.int64)), ('reward', np.zeros(2, np.int64)),
                                         ('done', np.zeros(2, np.float32)), ('done', np.zeros(3, np.uint8))])
def test_save_to_memory_shapes_and_dtypes_raise(field, value):
    args = dict(state=np.zeros((2, 4, 84, 84), np.uint8), action=np.zeros(2, np.int64), reward=np.zeros(2, np.float32),
                next_state=np.zeros((2, 4, 84, 84), np.uint8), done=np.zeros(2, bool))
    args[field] = value
    with pytest.raises(ValueError, match=field):
        _unbuilt(2).save_to_memory(**args, is_vectorised=True)


def test_single_env_form_needs_one_env():
    with pytest.raises(ValueError, match='num_envs == 1'):
        _unbuilt(2).save_to_memory(np.zeros((4, 84, 84), np.uint8), 0, 0.0, np.zeros((4, 84, 84), np.uint8), False)


def test_c_abi_rejects_bad_arguments_before_cuda():
    srl_build.build()
    L = _lib.lib()
    h = C.c_void_p()
    for args in ((1, 1, 1, 0.99, 0.6), (8, 9, 1, 0.99, 0.6), (8, 2, 33, 0.99, 0.6), (8, 2, 1, float('nan'), 0.6)):
        assert L.srl_replay_create(*args, C.byref(h)) == -1
        assert L.srl_last_error().startswith(b'replay_create: ')
    assert L.srl_replay_add(None, None, None, None, None, None, None) == -1
    assert L.srl_replay_sample(None, None, 4, None, None, None, None, None, None, None, None, None) == -1
    assert L.srl_replay_gather(None, None, 4, None, None, None, None, None, None) == -1
    assert L.srl_replay_size(None) == 0 and L.srl_replay_per(None) is None
