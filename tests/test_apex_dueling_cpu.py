"""The dueling head of the Ape-X learner and actors without a GPU: the dueling_dqn switch and its checks, AtariQNet(A, dueling=True)
against the formula written out, the 12-tensor flat layout, the C argument errors of the dueling entry points, and the oracle's
closed forms (the advantage gradients sum to zero over actions; both targets value s' with the dueling Q)."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from oracle import apex_oracle as O
from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.apex import (APEX_DUELING_PARAM_NAMES, APEX_PARAM_NAMES, ApexHParams, AtariQNet, B200ApexActor,
                                          B200ApexLearner, apex_param_shapes, default_q_state_dict)
from tests.apex_cases import frames, unbuilt

DUELING = O.Head('dueling')


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


def test_dueling_dqn_default_and_validation():
    hp = ApexHParams()
    assert hp.dueling_dqn is False and hp.to_c().dueling == 0
    assert ApexHParams(dueling_dqn=True).to_c().dueling == 1
    for bad in (1, 0, 'yes', None, 1.0):
        with pytest.raises(ValueError, match='dueling_dqn'):
            ApexHParams(dueling_dqn=bad).validate()
    with pytest.raises(ValueError, match='dueling_dqn'):
        B200ApexActor(4, 6, dueling_dqn=1)


@pytest.mark.parametrize('A', [1, 6, 18])
def test_dueling_net_names_and_shapes(A):
    net = AtariQNet(A, dueling=True)
    names = [n for n, _ in net.named_parameters()]
    assert tuple(names) == APEX_DUELING_PARAM_NAMES and tuple(net.state_dict()) == APEX_DUELING_PARAM_NAMES
    assert {n: tuple(p.shape) for n, p in net.named_parameters()} == dict(apex_param_shapes(A, dueling=True))
    assert dict(apex_param_shapes(A, dueling=True))['value.weight'] == (1, 512)
    assert dict(apex_param_shapes(A, dueling=True))['advantage.weight'] == (A, 512)
    # the plain network and its names are unchanged
    assert tuple(AtariQNet(A).state_dict()) == APEX_PARAM_NAMES and tuple(apex_param_shapes(A)) == APEX_PARAM_NAMES
    sd = default_q_state_dict(A, 3, dueling=True)
    assert tuple(sd) == APEX_DUELING_PARAM_NAMES
    assert torch.equal(sd['advantage.weight'], default_q_state_dict(A, 3, dueling=True)['advantage.weight'])


@pytest.mark.parametrize('A', [1, 6])
def test_dueling_forward_is_the_formula(A):
    torch.manual_seed(5)
    net = AtariQNet(A, dueling=True)
    obs = torch.randint(0, 256, (7, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        x = obs.double() / 255.0
        p = {n: t.double() for n, t in net.state_dict().items()}
        x = F.relu(F.conv2d(x, p['conv1.weight'], p['conv1.bias'], stride=4))
        x = F.relu(F.conv2d(x, p['conv2.weight'], p['conv2.bias'], stride=2))
        x = F.relu(F.conv2d(x, p['conv3.weight'], p['conv3.bias'], stride=1))
        h = F.relu(x.reshape(7, -1) @ p['fc.weight'].T + p['fc.bias'])
        v = h @ p['value.weight'].T + p['value.bias']                              # [7, 1]
        adv = h @ p['advantage.weight'].T + p['advantage.bias']                    # [7, A]
        want = v + adv - adv.sum(1, keepdim=True) / A
        got = net(obs).double()
    assert got.shape == (7, A)
    assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()), float((got - want).abs().max())
    if A == 1:                                  # one action: Q = V
        assert torch.allclose(got, v, rtol=1e-6, atol=1e-6)
    # the oracle's network computes the same Q from the same state dict
    ref = O.RefQNet(A, net.state_dict(), DUELING)
    assert torch.equal(ref(obs), net(obs))


@pytest.mark.parametrize('A', [1, 6, 18, 31])
def test_dueling_flat_layout(A, lib):
    total, off, cnt = _lib.apex_param_layout(A, dueling=True)
    shapes = apex_param_shapes(A, dueling=True)
    assert len(off) == len(cnt) == 12
    for (n, shp), c in zip(shapes.items(), cnt):
        assert c == int(torch.Size(shp).numel()), n
    assert all(o % 4 == 0 for o in off)
    spans = sorted(zip(off, cnt))
    for (o0, c0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + c0 <= o1                                               # disjoint, each tensor once
    assert len(set(off)) == 12 and spans[-1][0] == off[APEX_DUELING_PARAM_NAMES.index('fc.weight')]    # fc.weight last
    assert total == spans[-1][0] + spans[-1][1]
    iv, ia = APEX_DUELING_PARAM_NAMES.index('value.weight'), APEX_DUELING_PARAM_NAMES.index('advantage.weight')
    assert off[ia] == off[iv] + 512                                        # one [(A + 1), 512] head block
    ib, iab = APEX_DUELING_PARAM_NAMES.index('value.bias'), APEX_DUELING_PARAM_NAMES.index('advantage.bias')
    assert off[iab] == off[ib] + 4
    # dueling = 0 through the new entry point is the plain layout
    p_off, p_cnt = (C.c_int64 * 10)(), (C.c_int64 * 10)()
    p_total = lib.srl_apex_param_layout(A, p_off, p_cnt)
    assert _lib.apex_param_layout(A) == (p_total, list(p_off), list(p_cnt))


def test_dueling_c_argument_errors(lib):
    off, cnt = (C.c_int64 * 12)(), (C.c_int64 * 12)()
    for (A, d), msg in (((6, 2), b'dueling=2'), ((6, -1), b'dueling=-1'), ((0, 1), b'A=0'), ((32, 1), b'A=32')):
        assert lib.srl_apex_param_layout_ex(A, d, off, cnt) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_param_layout: ') and msg in m, m
    with pytest.raises(ValueError, match='dueling=2'):
        _lib.check(-1 if lib.srl_apex_param_layout_ex(6, 2, off, cnt) < 0 else 0, 'layout')
    h = C.c_void_p()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    for args, msg in (((6, 4, 0, 0, 0, None), b'NULL'), ((0, 4, 0, 1, 0, p), b'A=0'), ((6, 4, 0, 2, 0, p), b'dueling=2'),
                      ((6, 4, 0, -1, 0, p), b'dueling=-1'), ((6, 4, 2, 1, 0, p), b'precision=2')):
        assert lib.srl_apex_actor_create_ex(*args, C.byref(h)) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_actor_create: ') and msg in m and b'\n' not in m, m
    # the learner's config check runs before any CUDA call
    cfg = ApexHParams(dueling_dqn=True).to_c()
    cfg.dueling = 2
    assert lib.srl_apex_learner_create(C.addressof(cfg), p, p, p, p, p, C.byref(h)) == -1
    assert b'dueling=2' in lib.srl_last_error()


@pytest.mark.parametrize('learner_dueling', [False, True])
def test_sync_from_needs_the_same_head(learner_dueling):
    L = unbuilt(B200ApexLearner, hp=ApexHParams(num_actions=6, dueling_dqn=learner_dueling), device=torch.device('cuda', 0))
    X = unbuilt(B200ApexActor, num_envs=4, num_actions=6, dueling_dqn=not learner_dueling, device=torch.device('cuda', 0), _h=None)
    with pytest.raises(ValueError, match='dueling_dqn'):
        X.sync_from(L)


def _case(A, B, seed=0):
    on, tg = default_q_state_dict(A, seed, dueling=True), default_q_state_dict(A, seed + 1, dueling=True)
    g = torch.Generator().manual_seed(seed + 2)
    return on, tg, (frames(B, seed + 3), torch.randint(0, A, (B,), generator=g), torch.randn(B, generator=g), frames(B, seed + 4),
                    torch.rand(B, generator=g) < 0.3), torch.rand(B, generator=g) + 0.1


@pytest.mark.parametrize('A', [1, 6])
def test_oracle_advantage_gradients_sum_to_zero(A):
    on, tg, batch, w = _case(A, 8)
    out = O.learn_step(on, tg, *batch, weights=w, double_dqn=True, head=DUELING)
    gW, gb = out['grads']['advantage.weight'], out['grads']['advantage.bias']
    assert tuple(out['grads']) == APEX_DUELING_PARAM_NAMES
    if A == 1:                                  # Adv - mean(Adv) is 0 for one action: no gradient reaches the advantage stream
        assert not bool(gW.any()) and not bool(gb.any())
    else:
        scale = float(gW.abs().max())
        assert scale > 0 and float(gW.sum(0).abs().max()) <= 1e-5 * scale * A
        assert abs(float(gb.sum())) <= 1e-5 * float(gb.abs().max()) * A
    # the value stream carries dL/dq: its bias gradient is sum_n dq_n = 2/B sum_n w_n (q_n - y_n)
    dq = 2.0 * w * (out['q'] - out['y']) / 8
    assert float(out['grads']['value.bias'][0]) == pytest.approx(float(dq.sum()), rel=1e-4, abs=1e-7)


@pytest.mark.parametrize('double', [False, True])
def test_oracle_targets_use_the_dueling_q(double):
    A, B, gamma = 5, 6, 0.9
    on, tg, (obs, a, r, nobs, d), w = _case(A, B, seed=10)
    tg['advantage.bias'][1] += 1.0              # the target network prefers action 1, the online network does not

    def q_rows(sd, x):                          # the formula, on the oracle's own features
        net = O.RefQNet(A, sd, DUELING)
        with torch.no_grad():
            h = net.features(x)
            v = h @ sd['value.weight'].T + sd['value.bias']
            adv = h @ sd['advantage.weight'].T + sd['advantage.bias']
            return v + adv - adv.mean(1, keepdim=True)

    qn_t, qn_o = q_rows(tg, nobs), q_rows(on, nobs)
    astar = (qn_o if double else qn_t).argmax(1)
    want_y = r + (1 - d.float()) * gamma * qn_t.gather(1, astar[:, None]).squeeze(1)
    want_q = q_rows(on, obs).gather(1, a[:, None]).squeeze(1)
    out = O.learn_step(on, tg, obs, a, r, nobs, d, weights=w, gamma=gamma, double_dqn=double, head=DUELING)
    torch.testing.assert_close(out['y'], want_y, rtol=1e-6, atol=1e-6)
    torch.testing.assert_close(out['q'], want_q, rtol=1e-6, atol=1e-6)
    # the two rules pick different actions somewhere, so the test tells them apart
    assert not torch.equal(qn_o.argmax(1), qn_t.argmax(1))


def test_initial_priorities_on_the_dueling_net():
    A, N = 4, 5
    sd = default_q_state_dict(A, 2, dueling=True)
    s, ns = frames(N, 1), frames(N, 2)
    a = torch.tensor([0, 1, 2, 3, 1])
    R = torch.tensor([0.5, -1.0, 2.0, 0.0, 0.25])
    d = torch.tensor([0, 1, 0, 0, 1], dtype=torch.bool)
    net = O.RefQNet(A, sd, DUELING)
    with torch.no_grad():
        q = net(s)[torch.arange(N), a]
        y = R + (1 - d.float()) * 0.5 * net(ns).max(1)[0]
    p = O.initial_priorities(sd, s, a, R, ns, d, 0.5, 1e-3, head=DUELING)
    assert torch.equal(p, (q - y).abs().double() + 1e-3)
