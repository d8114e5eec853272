"""CPU: the frame replay memory's oracle (oracle/frame_replay_oracle.py) against ReplayOracle, its frame counts and retirement, and the
argument checks of GpuFrameReplayBuffer and srl_frame_replay_* that need no GPU."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import frame_replay_oracle as FO
from oracle import replay_oracle as O
from scalerl_b200 import _lib, build as srl_build
from scalerl_b200.data.replay_memory import GpuFrameReplayBuffer


def _run(M, E, n, steps, seed, done=None, frame_capacity=None, done_rate=0.05):
    """the same Atari-like adds into ReplayOracle (stacks) and FrameReplayOracle (frames)"""
    rng = np.random.RandomState(seed + 1)
    action = rng.randint(0, 18, size=(steps, E)).astype(np.int64)
    reward = rng.randn(steps, E).astype(np.float32)
    si, ni, done, K = FO.atari_stream(E, steps, seed, done=done, done_rate=done_rate)
    frames = FO.stream_frames(E, K, seed)
    ro, fo = O.ReplayOracle(M, E, n, O.GAMMA), FO.FrameReplayOracle(M, E, n, O.GAMMA, frame_capacity)
    for t in range(steps):
        s, ns = FO.stream_stacks(frames, si[t]), FO.stream_stacks(frames, ni[t])
        ro.add(list(s), action[t], reward[t], list(ns), done[t])
        fo.add(s, action[t], reward[t], ns, done[t])
    return ro, fo, si


def _same_slot(ro, fo, slot):
    s, a, r, ns, d = fo.gather(slot)
    rs, ra, rr, rns, rd = ro.slots[slot]
    return np.array_equal(s, rs) and np.array_equal(ns, rns) and a == ra and np.float32(r).view(np.uint32) == np.float32(rr).view(np.uint32) and d == rd


def test_oracle_gathers_equal_replay_oracle_on_every_case():
    for M, E, n, dr, steps, seed in O.CASES:
        _, _, done = O.case_inputs(E, steps, dr, seed)
        ro, fo, _ = _run(M, E, n, steps, seed, done=done)
        assert fo.size == ro.size and fo.tree_ptr == ro.tree_ptr and fo.retired == 0
        for slot in range(ro.size):
            assert _same_slot(ro, fo, slot), (M, E, n, dr, slot)


def test_frame_counts_on_an_atari_like_stream():
    """one frame per env step, one more per episode start (the reset frame repeated 4 times is stored once), life losses included"""
    M, E, n, steps = 1024, 4, 3, 200
    ro, fo, si = _run(M, E, n, steps, seed=5, done_rate=0.08)
    starts = int(np.all(si == si[..., :1], axis=-1).sum())
    assert starts > E                                        # resets happened after the first episode
    assert fo.head == FO.expected_new_frames(si) == E * steps + starts
    assert all(_same_slot(ro, fo, slot) for slot in range(ro.size))


def test_frame_counts_without_sharing():
    """stacks that share nothing cost 8 frames a step"""
    E, steps = 2, 6
    rng = np.random.RandomState(0)
    fo = FO.FrameReplayOracle(64, E, 1)
    for _ in range(steps):
        fo.add(rng.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8), np.zeros(E, np.int64), np.zeros(E, np.float32),
               rng.randint(0, 256, (E, 4, 84, 84)).astype(np.uint8), np.zeros(E, np.uint8))
    assert fo.head == 8 * E * steps


@pytest.mark.parametrize('n', [1, 3])
def test_retirement_on_a_small_pool(n):
    """at the minimum frame_capacity the pool wraps: slots whose frames are overwritten retire, every other stored slot still
    gathers ReplayOracle's bytes, and a slot the fold writes again is live"""
    M, E, steps = 128, 2, 120
    F = 8 * E * (n + 1)
    ro, fo, _ = _run(M, E, n, steps, seed=9, frame_capacity=F, done_rate=0.2)
    assert fo.retired > 0 and fo.retired_slots
    live_from = fo.head - F
    for slot in range(ro.size):
        if slot in fo.retired_slots:
            assert fo.oldest[slot] < live_from
        else:
            assert fo.oldest[slot] >= live_from and _same_slot(ro, fo, slot), slot
    newest = [(fo.tree_ptr - 1 - k) % M for k in range(E)]
    assert not set(newest) & fo.retired_slots


@pytest.mark.parametrize('kw', [dict(memory_size=1, num_envs=1), dict(memory_size=8, num_envs=9), dict(memory_size=8, num_envs=2, n_step=33),
                                dict(memory_size=8, num_envs=2, gamma=float('nan')), dict(memory_size=8, num_envs=2, frame_capacity=31),
                                dict(memory_size=8, num_envs=2, n_step=2, frame_capacity=47), dict(memory_size=8, num_envs=1, frame_capacity=16.0),
                                dict(memory_size=8, num_envs=1, frame_capacity=(1 << 32) + 1)])
def test_constructor_arguments_raise_without_gpu(kw):
    with pytest.raises(ValueError):
        GpuFrameReplayBuffer(**kw)


def test_default_frame_capacity():
    m = GpuFrameReplayBuffer.__new__(GpuFrameReplayBuffer)
    m.memory_size, m.num_envs, m.n_step, m._frame_capacity_arg = 100_000, 64, 3, None
    m._check_extra()
    assert m.frame_capacity == 100_000 + 12_500 + 8 * 64 * 7 == FO.default_frame_capacity(100_000, 64, 3)


def test_save_to_memory_checks_fields_before_device_work():
    m = GpuFrameReplayBuffer.__new__(GpuFrameReplayBuffer)
    m.num_envs, m.device, m._h = 2, torch.device('cuda', 0), None
    with pytest.raises(ValueError, match='next_state'):
        m.save_to_memory(np.zeros((2, 4, 84, 84), np.uint8), np.zeros(2, np.int64), np.zeros(2, np.float32), np.zeros((2, 84, 84), np.uint8),
                         np.zeros(2, bool), is_vectorised=True)


def test_c_abi_rejects_bad_arguments_before_cuda():
    srl_build.build()
    L = _lib.lib()
    h = C.c_void_p()
    for args in ((1, 1, 1, 0.99, 0.6, 16), (8, 9, 1, 0.99, 0.6, 144), (8, 2, 33, 0.99, 0.6, 1000), (8, 2, 1, float('nan'), 0.6, 32),
                 (8, 2, 1, 0.99, 0.6, 31), (8, 2, 3, 0.99, 0.6, 63), (8, 1, 1, 0.99, 0.6, (1 << 32) + 1)):
        assert L.srl_frame_replay_create(*args, C.byref(h)) == -1
        assert L.srl_last_error().startswith(b'frame_replay_create: ')
    assert L.srl_frame_replay_create(8, 1, 1, 0.99, 0.6, 16, None) == -1
    assert L.srl_frame_replay_add(None, None, None, None, None, None, None) == -1
    assert L.srl_frame_replay_add_prioritized(None, None, None, None, None, None, None, 0.01, None) == -1
    assert L.srl_frame_replay_sample(None, None, 4, None, None, None, None, None, None, None, None, None) == -1
    assert L.srl_frame_replay_gather(None, None, 4, None, None, None, None, None, None) == -1
    assert L.srl_frame_replay_size(None) == 0 and L.srl_frame_replay_per(None) is None
    assert L.srl_frame_replay_frames_allocated(None, None) == -1 and L.srl_frame_replay_retired(None, None) == -1
