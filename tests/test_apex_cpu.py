"""Ape-X learner without a GPU: hyper-parameter and argument errors, the oracle's closed forms, and the flat parameter layout."""
import ctypes
import math

import pytest
import torch
from torch import nn

from oracle import apex_oracle as O
from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.apex import APEX_PARAM_NAMES, ApexHParams, AtariQNet, apex_param_shapes


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


@pytest.mark.parametrize('field,value', [('batch_size', 0), ('batch_size', 65537), ('num_actions', 0), ('num_actions', 32),
                                         ('gamma', -0.1), ('gamma', math.nan), ('learning_rate', 0.0), ('max_grad_norm', 0.0),
                                         ('target_update_frequency', 0), ('soft_update_tau', 1.5), ('precision', 'fp16'),
                                         ('priority_eps', -1e-6), ('adam_beta1', 1.0), ('adam_eps', -1.0)])
def test_hparam_errors(field, value):
    with pytest.raises(ValueError):
        ApexHParams(**{field: value}).validate()


def test_hparam_defaults_are_the_reference_learners():
    hp = ApexHParams()
    assert (hp.gamma, hp.learning_rate, hp.max_grad_norm, hp.double_dqn, hp.target_update_frequency, hp.soft_update_tau) == \
        (0.99, 1e-3, None, False, 100, 1.0)
    assert hp.to_c().max_grad_norm == math.inf      # no clip: coefficient exactly 1 in the same kernel


def test_c_argument_errors(lib):
    h = ctypes.c_void_p()
    cfg = ApexHParams(num_actions=6).to_c()
    assert lib.srl_apex_learner_create(ctypes.addressof(cfg), None, None, None, None, None, ctypes.byref(h)) == -1
    assert b'NULL' in lib.srl_last_error()
    cfg.A = 40
    assert lib.srl_apex_learner_create(ctypes.addressof(cfg), None, None, None, None, None, ctypes.byref(h)) == -1
    assert b'A=40' in lib.srl_last_error()
    cfg.A, cfg.max_grad_norm = 6, -1.0
    assert lib.srl_apex_learner_create(ctypes.addressof(cfg), None, None, None, None, None, ctypes.byref(h)) == -1
    assert b'max_grad_norm' in lib.srl_last_error()
    assert lib.srl_apex_learner_step(None, *([None] * 10)) == -1
    assert lib.srl_apex_learner_update_target(None, 1.0, None) == -1
    assert lib.srl_apex_learner_q_values(None, None, 1, None, None) == -1


@pytest.mark.parametrize('A', [1, 6, 18, 31])
def test_atari_qnet_matches_the_flat_layout(lib, A):
    total, off, cnt = _lib.apex_param_layout(A)
    net = AtariQNet(A)
    names = [n for n, _ in net.named_parameters()]
    assert tuple(names) == APEX_PARAM_NAMES
    shapes = apex_param_shapes(A)
    for i, (n, p) in enumerate(net.named_parameters()):
        assert tuple(p.shape) == shapes[n] and cnt[i] == p.numel(), n
        assert off[i] % 4 == 0
    assert max(off) == off[APEX_PARAM_NAMES.index('fc.weight')]      # fc.weight last
    assert total == off[6] + cnt[6]
    spans = sorted((off[i], off[i] + cnt[i]) for i in range(10))
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))


def test_atari_qnet_is_the_oracle_network():
    torch.manual_seed(3)
    net = AtariQNet(5)
    ref = O.RefQNet(5, net.state_dict())
    obs = torch.randint(0, 256, (3, 4, 84, 84), dtype=torch.uint8)
    assert torch.equal(net(obs), ref(obs))


def _batch(B, A, seed=0, done_p=0.3):
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g), torch.randint(0, A, (B,), generator=g),
            torch.randn(B, generator=g), torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g),
            torch.rand(B, generator=g) < done_p)


def _sds(A):
    torch.manual_seed(0)
    on, tg = AtariQNet(A), AtariQNet(A)
    return on.state_dict(), tg.state_dict()


def test_oracle_closed_forms():
    A, B = 4, 6
    on, tg = _sds(A)
    obs, a, r, nobs, d = _batch(B, A)
    # gamma = 0: y = r
    out = O.learn_step(on, tg, obs, a, r, nobs, d, gamma=0.0)
    assert torch.equal(out['y'], r)
    # done = 1: y = r whatever gamma
    out = O.learn_step(on, tg, obs, a, r, nobs, torch.ones(B, dtype=torch.bool), gamma=0.99)
    assert torch.equal(out['y'], r)
    # plain max over the target network vs. the target's value of the online argmax
    d0 = torch.zeros(B, dtype=torch.bool)
    qt = O.RefQNet(A, tg)(nobs).detach()
    qo = O.RefQNet(A, on)(nobs).detach()
    plain = O.learn_step(on, tg, obs, a, r, nobs, d0, gamma=0.5)
    dbl = O.learn_step(on, tg, obs, a, r, nobs, d0, gamma=0.5, double_dqn=True)
    assert torch.equal(plain['y'], r + 0.5 * qt.max(1)[0])
    assert torch.equal(dbl['y'], r + 0.5 * qt.gather(1, qo.argmax(1, keepdim=True)).squeeze(1))
    # w = 1 is nn.MSELoss (dqn_agent.py:81,171), and the priorities are |q - y|
    q = O.RefQNet(A, on)(obs).gather(1, a.unsqueeze(1)).squeeze(1).detach()
    assert plain['loss'] == pytest.approx(float(nn.MSELoss()(plain['y'], q)), rel=1e-6)
    assert torch.equal(plain['td'], (plain['q'] - plain['y']).abs())
    w = torch.rand(B)
    wl = O.learn_step(on, tg, obs, a, r, nobs, d0, weights=w, gamma=0.5)
    assert wl['loss'] == pytest.approx(float((w * (q - plain['y']) ** 2).mean()), rel=1e-6)


def test_oracle_soft_update_tau_one_copies():
    src, tgt = [torch.randn(5)], [torch.randn(5)]
    O.soft_target_update(src, tgt, 1.0)
    assert torch.equal(src[0], tgt[0])
