"""Ape-X actor without a GPU: the epsilon schedule's closed form, the host-side argument errors of B200ApexActor and of the prioritized
add, the C argument errors, and the initial-priority oracle on hand-computed cases."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import apex_oracle as O
from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.apex import AtariQNet, B200ApexActor, apex_epsilons
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
from tests.apex_cases import frames, unbuilt


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


@pytest.mark.parametrize('N', [1, 8, 256])
def test_apex_epsilons_closed_form(N):
    e = apex_epsilons(N)
    assert e.shape == (N,) and e.dtype == np.float64
    want = [0.4] if N == 1 else [0.4 ** (1 + 7.0 * i / (N - 1)) for i in range(N)]
    assert np.allclose(e, want, rtol=1e-15, atol=0)
    assert e[0] == 0.4 and (N == 1 or e[-1] == pytest.approx(0.4 ** 8, rel=1e-15))
    assert np.all(np.diff(e) < 0)
    assert apex_epsilons(3, eps=0.5, alpha=2.0).tolist() == pytest.approx([0.5, 0.25, 0.125], rel=1e-15)


@pytest.mark.parametrize('kw,match', [(dict(num_envs=0), 'num_envs'), (dict(num_envs=65537), 'num_envs'), (dict(num_envs=2.0), 'num_envs'),
                                      (dict(num_actions=0), 'num_actions'), (dict(num_actions=32), 'num_actions'),
                                      (dict(seed=-1), 'seed'), (dict(precision='fp16'), 'precision'),
                                      (dict(priority_eps=0.0), 'priority_eps'), (dict(priority_eps=-1e-6), 'priority_eps'),
                                      (dict(priority_eps=float('nan')), 'priority_eps'), (dict(epsilons=[0.1, 0.2]), 'epsilons'),
                                      (dict(epsilons=[0.1, 0.2, 1.5, 0.0]), 'epsilons'), (dict(epsilons=[0.1, float('nan'), 0.2, 0.0]), 'epsilons')])
def test_constructor_errors_without_gpu(kw, match):
    args = dict(num_envs=4, num_actions=6)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        B200ApexActor(**args)


def _unbuilt_actor(num_envs=4, num_actions=6):
    """an actor with only its host attributes: the checks before any device work"""
    return unbuilt(B200ApexActor, num_envs=num_envs, num_actions=num_actions, device=torch.device('cuda', 0), _h=None, priority_eps=1e-6)


@pytest.mark.parametrize('eps', [[0.1] * 3, [0.1] * 5, [0.1, 0.1, -0.1, 0.1], [0.1, 2.0, 0.1, 0.1]])
def test_set_epsilons_errors(eps):
    with pytest.raises(ValueError, match='epsilons'):
        _unbuilt_actor().set_epsilons(eps)


@pytest.mark.parametrize('obs', [np.zeros((3, 4, 84, 84), np.uint8), np.zeros((4, 4, 84, 84), np.float32), np.zeros((4, 84, 84), np.uint8),
                                 np.zeros((4, 3, 84, 84), np.uint8)])
def test_act_obs_errors(obs):
    with pytest.raises(ValueError, match='obs'):
        _unbuilt_actor().act(obs)


def test_sync_from_needs_a_learner():
    with pytest.raises(ValueError, match='B200ApexLearner'):
        _unbuilt_actor().sync_from(object())


def _unbuilt_memory(num_envs):
    return unbuilt(GpuPrioritizedReplayBuffer, num_envs=num_envs, device=torch.device('cuda', 0), _h=None)


@pytest.mark.parametrize('actor,match', [(object(), 'B200ApexActor'), (_unbuilt_actor(num_envs=3), 'num_envs'), ('dev', 'cuda:1')])
def test_prioritized_save_to_memory_errors(actor, match):
    if actor == 'dev':
        actor = _unbuilt_actor(num_envs=2)
        actor.device = torch.device('cuda', 1)
    args = (np.zeros((2, 4, 84, 84), np.uint8), np.zeros(2, np.int64), np.zeros(2, np.float32), np.zeros((2, 4, 84, 84), np.uint8),
            np.zeros(2, bool))
    with pytest.raises(ValueError, match=match):
        _unbuilt_memory(2).save_to_memory(*args, is_vectorised=True, priorities_from=actor)


def test_c_argument_errors(lib):
    """each bad argument is one message and a non-zero return before any CUDA call"""
    h = C.c_void_p()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    for args, msg in (((6, 4, 0, 0, None), b'NULL'), ((0, 4, 0, 0, p), b'A=0'), ((32, 4, 0, 0, p), b'A=32'),
                      ((6, 0, 0, 0, p), b'num_envs=0'), ((6, 65537, 0, 0, p), b'num_envs=65537'), ((6, 4, 2, 0, p), b'precision=2')):
        assert lib.srl_apex_actor_create(*args, C.byref(h)) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_actor_create: ') and msg in m and b'\n' not in m, m
    assert lib.srl_apex_actor_act(None, None, None, None, None) == -1 and b'NULL' in lib.srl_last_error()
    assert lib.srl_apex_actor_q_values(None, None, 1, None, None) == -1 and b'NULL' in lib.srl_last_error()
    assert lib.srl_apex_actor_destroy(None) == 0
    assert lib.srl_replay_add_prioritized(None, None, None, None, None, None, None, 1e-6, None) == -1
    assert lib.srl_last_error().startswith(b'replay_add_prioritized: NULL')
    # priority_eps is checked before either handle is read: any non-NULL pointers do
    for eps in (0.0, -1e-6, float('nan'), float('inf')):
        assert lib.srl_replay_add_prioritized(p, p, p, p, p, p, p, eps, None) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'replay_add_prioritized: priority_eps=') and b'> 0' in m, m


def _sd(A, seed=0):
    torch.manual_seed(seed)
    return AtariQNet(A).state_dict()


def test_initial_priorities_hand_computed():
    A, N = 5, 6
    sd = _sd(A)
    s, ns = frames(N, 1), frames(N, 2)
    a = torch.tensor([0, 1, 2, 3, 4, 2])
    R = torch.tensor([0.5, -1.0, 2.0, 0.0, 0.25, 3.0])
    q = O.RefQNet(A, sd)(s).detach()
    qa = q[torch.arange(N), a]
    # all done: y = R, whatever gamma and s'
    p = O.initial_priorities(sd, s, a, R, ns, torch.ones(N, dtype=torch.bool), 0.97, 1e-6)
    assert p.dtype == torch.float64 and torch.equal(p, (qa - R).abs().double() + 1e-6)
    # gamma = 0: y = R
    p0 = O.initial_priorities(sd, s, a, R, ns, torch.zeros(N, dtype=torch.bool), 0.0, 0.0)
    assert torch.equal(p0, (qa - R).abs().double())
    # a Q head with a unique argmax at s': q.bias[3] dominates, so max_a Q(s') = Q(s')[3] and y = R + gamma_n Q(s')[3] where not done
    sd2 = {k: v.clone() for k, v in sd.items()}
    sd2['q.bias'][3] += 100.0
    qn = O.RefQNet(A, sd2)(ns).detach()
    assert bool((qn.argmax(1) == 3).all()) and bool((qn[:, 3:4] > qn[:, [0, 1, 2, 4]]).all())
    d = torch.tensor([0, 1, 0, 0, 1, 0], dtype=torch.bool)
    q2 = O.RefQNet(A, sd2)(s).detach()[torch.arange(N), a]
    y = R + (1 - d.float()) * 0.5 * qn[:, 3]
    p2 = O.initial_priorities(sd2, s, a, R, ns, d, 0.5, 1e-3)
    assert torch.equal(p2, (q2 - y).abs().double() + 1e-3)
    assert torch.equal(p2[d], (q2 - R).abs().double()[d] + 1e-3)
