"""The categorical (C51) head of the Ape-X learner and actors without a GPU: the categorical_dqn switch and its checks,
AtariQNet(A, categorical=True) against the formula written out, the flat layout with q.weight [A K, 512], the C argument errors of the
categorical entry points, and the oracle's closed forms (the projection preserves mass, puts a reward on an atom there and splits one
between atoms linearly, clamps to the end atoms; the torch projection equals an fp64 loop; the written logit gradient equals autograd's;
KL >= 0 with KL = 0 at p = m)."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import apex_oracle as O
from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.apex import (APEX_PARAM_NAMES, ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner, apex_param_shapes,
                                          categorical_support, default_q_state_dict)
from tests.apex_cases import frames, unbuilt


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


def test_categorical_dqn_defaults_and_validation():
    hp = ApexHParams()
    assert hp.categorical_dqn is False and (hp.v_min, hp.v_max, hp.num_atoms) == (0.0, 200.0, 51)      # DQNArguments' defaults
    c = hp.to_c()
    assert c.num_atoms == 0 and hp.atoms() == 0
    c = ApexHParams(categorical_dqn=True, v_min=-10.0, v_max=10.0, num_atoms=64).to_c()
    assert (c.num_atoms, c.v_min, c.v_max, c.dueling) == (64, -10.0, 10.0, 0)
    for bad in (1, 0, 'yes', None):
        with pytest.raises(ValueError, match='categorical_dqn'):
            ApexHParams(categorical_dqn=bad).validate()
    for K in (1, 65, 0, 2.0, True):
        with pytest.raises(ValueError, match='num_atoms'):
            ApexHParams(categorical_dqn=True, num_atoms=K).validate()
    for lo, hi in ((1.0, 1.0), (2.0, -2.0), (math.nan, 1.0), (0.0, math.inf), (-1e39, 0.0)):
        with pytest.raises(ValueError, match='v_min'):
            ApexHParams(categorical_dqn=True, v_min=lo, v_max=hi).validate()
    with pytest.raises(ValueError, match='dueling'):
        ApexHParams(categorical_dqn=True, dueling_dqn=True).validate()
    with pytest.raises(ValueError, match='dueling'):
        AtariQNet(6, dueling=True, categorical=True)
    for kw, msg in ((dict(categorical_dqn=1), 'categorical_dqn'), (dict(categorical_dqn=True, num_atoms=65), 'num_atoms'),
                    (dict(categorical_dqn=True, v_min=3.0, v_max=3.0), 'v_min'), (dict(categorical_dqn=True, dueling_dqn=True), 'dueling')):
        with pytest.raises(ValueError, match=msg):
            B200ApexActor(4, 6, **kw)


@pytest.mark.parametrize('A,K', [(1, 2), (6, 51), (18, 51), (31, 64)])
def test_categorical_net_names_and_shapes(A, K):
    net = AtariQNet(A, categorical=True, num_atoms=K, v_min=-10.0, v_max=10.0)
    assert tuple(n for n, _ in net.named_parameters()) == APEX_PARAM_NAMES and tuple(net.state_dict()) == APEX_PARAM_NAMES
    assert {n: tuple(p.shape) for n, p in net.named_parameters()} == dict(apex_param_shapes(A, num_atoms=K))
    assert dict(apex_param_shapes(A, num_atoms=K))['q.weight'] == (A * K, 512) and dict(apex_param_shapes(A, num_atoms=K))['q.bias'] == (A * K,)
    assert tuple(apex_param_shapes(A)['q.weight']) == (A, 512)                 # the plain head is unchanged
    z = net.support
    assert z.dtype == torch.float32 and z.shape == (K,) and float(z[0]) == -10.0
    assert abs(float(z[-1]) - 10.0) <= 1e-5
    sd = default_q_state_dict(A, 3, num_atoms=K)
    assert tuple(sd) == APEX_PARAM_NAMES and tuple(sd['q.weight'].shape) == (A * K, 512)
    assert torch.equal(sd['q.weight'], default_q_state_dict(A, 3, num_atoms=K)['q.weight'])
    # the encoder's initial weights are the plain network's (the head is drawn last)
    assert torch.equal(sd['fc.weight'], default_q_state_dict(A, 3)['fc.weight'])
    AtariQNet(A).load_state_dict({k: v for k, v in default_q_state_dict(A, 3).items()})
    with pytest.raises(ValueError, match='categorical'):
        AtariQNet(A).dist(torch.zeros(1, 4, 84, 84, dtype=torch.uint8))


@pytest.mark.parametrize('A,K,lo,hi', [(1, 2, 0.0, 200.0), (6, 51, -10.0, 10.0)])
def test_categorical_forward_is_the_formula(A, K, lo, hi):
    torch.manual_seed(5)
    net = AtariQNet(A, categorical=True, num_atoms=K, v_min=lo, v_max=hi)
    obs = torch.randint(0, 256, (7, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        x = obs.double() / 255.0
        p = {n: t.double() for n, t in net.state_dict().items()}
        x = F.relu(F.conv2d(x, p['conv1.weight'], p['conv1.bias'], stride=4))
        x = F.relu(F.conv2d(x, p['conv2.weight'], p['conv2.bias'], stride=2))
        x = F.relu(F.conv2d(x, p['conv3.weight'], p['conv3.bias'], stride=1))
        h = F.relu(x.reshape(7, -1) @ p['fc.weight'].T + p['fc.bias'])
        logits = (h @ p['q.weight'].T + p['q.bias']).view(7, A, K)            # row a K + k: atom k of action a
        e = (logits - logits.max(2, keepdim=True)[0]).exp()
        want_p = e / e.sum(2, keepdim=True)
        z = lo + torch.arange(K, dtype=torch.float64) * ((hi - lo) / (K - 1))
        want_q = (want_p * z).sum(2)
        got_p, got_q = net.dist(obs).double(), net(obs).double()
    assert got_p.shape == (7, A, K) and got_q.shape == (7, A)
    assert float((got_p - want_p).abs().max()) <= 1e-6
    assert float((got_q - want_q).abs().max()) <= 1e-5 * max(abs(lo), abs(hi))
    assert torch.equal(categorical_support(K, lo, hi), O.support(K, lo, hi)[0])
    # the oracle's network computes the same logits from the same state dict
    assert torch.equal(O.RefQNet(A, net.state_dict(), O.Head('categorical', num_atoms=K, v_min=lo, v_max=hi))(obs), net.q(net._features(obs)).view(7, A, K))


@pytest.mark.parametrize('K', [2, 51, 64])
@pytest.mark.parametrize('A', [1, 6, 18, 31])
def test_categorical_flat_layout(A, K, lib):
    total, off, cnt = _lib.apex_param_layout(A, num_atoms=K)
    shapes = apex_param_shapes(A, num_atoms=K)
    assert len(off) == len(cnt) == 10
    for (n, shp), c in zip(shapes.items(), cnt):
        assert c == int(torch.Size(shp).numel()), n
    assert all(o % 4 == 0 for o in off)
    spans = sorted(zip(off, cnt))
    for (o0, c0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + c0 <= o1
    iq, ifc = APEX_PARAM_NAMES.index('q.weight'), APEX_PARAM_NAMES.index('fc.weight')
    assert spans[-1][0] == off[ifc] and off[iq] < off[ifc] and total == off[ifc] + cnt[ifc]     # q.weight before fc.weight, fc last
    # num_atoms = 0 is the plain layout
    o10, c10 = (C.c_int64 * 10)(), (C.c_int64 * 10)()
    assert lib.srl_apex_param_layout_cat(A, 0, o10, c10) == _lib.apex_param_layout(A)[0] and list(o10) == _lib.apex_param_layout(A)[1]


def test_categorical_c_argument_errors(lib):
    off, cnt = (C.c_int64 * 10)(), (C.c_int64 * 10)()
    for (A, K), msg in (((6, 1), b'num_atoms=1'), ((6, 65), b'num_atoms=65'), ((6, -1), b'num_atoms=-1'), ((32, 51), b'A=32')):
        assert lib.srl_apex_param_layout_cat(A, K, off, cnt) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_param_layout: ') and msg in m, m
    h = C.c_void_p()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    nan, inf = float('nan'), float('inf')
    for args, msg in (((6, 4, 0, 51, 0.0, 1.0, 0, None), b'NULL'), ((6, 4, 0, 1, 0.0, 1.0, 0, p), b'num_atoms=1'),
                      ((6, 4, 0, 65, 0.0, 1.0, 0, p), b'num_atoms=65'), ((6, 4, 0, 51, 1.0, 1.0, 0, p), b'v_min=1'),
                      ((6, 4, 0, 51, 2.0, -2.0, 0, p), b'v_min=2'), ((6, 4, 0, 51, nan, 1.0, 0, p), b'v_min=nan'),
                      ((6, 4, 0, 51, 0.0, inf, 0, p), b'v_max=inf'), ((6, 4, 2, 51, 0.0, 1.0, 0, p), b'precision=2')):
        assert lib.srl_apex_actor_create_cat(*args, C.byref(h)) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_actor_create: ') and msg in m and b'\n' not in m, m
    # the learner's config check runs before any CUDA call
    for kw, msg in ((dict(num_atoms=65), b'num_atoms=65'), (dict(num_atoms=1), b'num_atoms=1'), (dict(v_min=20.0), b'v_min=20'),
                    (dict(v_max=nan), b'v_max=nan'), (dict(dueling=1), b'dueling=1')):
        cfg = ApexHParams(categorical_dqn=True, v_min=-10.0, v_max=10.0).to_c()
        for k, v in kw.items():
            setattr(cfg, k, v)
        assert lib.srl_apex_learner_create(C.addressof(cfg), p, p, p, p, p, C.byref(h)) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_learner: ') and msg in m, m
    # a zeroed head setting is the scalar head: the support is not read
    cfg = ApexHParams().to_c()
    assert (cfg.num_atoms, cfg.v_min, cfg.v_max) == (0, 0.0, 200.0)
    cfg.v_min = cfg.v_max = nan
    assert lib.srl_apex_learner_create(C.addressof(cfg), None, p, p, p, p, C.byref(h)) == -1
    assert b'NULL' in lib.srl_last_error()


@pytest.mark.parametrize('learner,msg', [(dict(categorical_dqn=False), 'categorical_dqn'), (dict(num_atoms=64), 'num_atoms'),
                                         (dict(v_min=-10.0), 'v_min'), (dict(v_max=10.0), 'v_max')])
def test_sync_from_needs_the_same_head(learner, msg):
    hp = dict(num_actions=6, categorical_dqn=True, v_min=0.0, v_max=200.0, num_atoms=51)
    hp.update(learner)
    L = unbuilt(B200ApexLearner, hp=ApexHParams(**hp), device=torch.device('cuda', 0))
    X = unbuilt(B200ApexActor, num_envs=4, num_actions=6, dueling_dqn=False, categorical_dqn=True, num_atoms=51, v_min=0.0, v_max=200.0,
                 device=torch.device('cuda', 0), _h=None)
    with pytest.raises(ValueError, match=msg):
        X.sync_from(L)


# ---------------------------------------------------------------------------------------------------------------- the oracle
def _dist(N, K, seed):
    g = torch.Generator().manual_seed(seed)
    return F.softmax(3 * torch.randn(N, K, generator=g), dim=1)


@pytest.mark.parametrize('K,lo,hi,gamma', [(2, 0.0, 200.0, 0.99), (51, -10.0, 10.0, 0.97), (64, 0.0, 200.0, 0.99 ** 3)])
def test_projection_preserves_mass_and_equals_the_fp64_loop(K, lo, hi, gamma):
    N = 64
    p = _dist(N, K, K)
    g = torch.Generator().manual_seed(1)
    r = 4 * torch.randn(N, generator=g) * (hi - lo) / 20
    d = torch.rand(N, generator=g) < 0.3
    z, dz = O.support(K, lo, hi)
    m = O.project(p, r, d, gamma, z, dz, lo, hi)
    assert bool((m >= 0).all())
    torch.testing.assert_close(m.sum(1), torch.ones(N), rtol=0, atol=2e-6)
    m64 = O.project_fp64_loop(p.double().numpy(), r.double().numpy(), d.numpy(), float(np.float32(gamma)), lo, hi)
    assert np.allclose(m64.sum(1), 1.0, atol=1e-12)
    # b_j <= K - 1 carries fp32 rounding of a few ulp of 64 (about 4e-6 each), which moves that much mass between neighbours
    assert float(np.abs(m.double().numpy() - m64).max()) <= 1e-5


@pytest.mark.parametrize('K,lo,hi', [(51, -10.0, 10.0), (11, 0.0, 200.0)])
def test_projection_closed_forms(K, lo, hi):
    z, dz = O.support(K, lo, hi)
    p = _dist(5, K, 3)
    # done (or gamma = 0): Tz = r for every j; a reward on atom i puts all the mass there
    i = K // 3
    m = O.project(p, torch.full((5,), float(z[i])), torch.ones(5, dtype=torch.bool), 0.99, z, dz, lo, hi)
    want = torch.zeros(5, K)
    want[:, i] = 1.0
    torch.testing.assert_close(m, want, rtol=0, atol=2e-6)
    torch.testing.assert_close(O.project(p, torch.full((5,), float(z[i])), torch.zeros(5, dtype=torch.bool), 0.0, z, dz, lo, hi), want,
                               rtol=0, atol=2e-6)
    # a reward a quarter of the way from atom i to atom i + 1 splits 3 : 1
    r = float(z[i]) + 0.25 * float(dz)
    m = O.project(p, torch.full((5,), r), torch.ones(5, dtype=torch.bool), 0.99, z, dz, lo, hi)
    torch.testing.assert_close(m[:, i], torch.full((5,), 0.75), rtol=0, atol=2e-5)
    torch.testing.assert_close(m[:, i + 1], torch.full((5,), 0.25), rtol=0, atol=2e-5)
    assert float(m.sum(1).sub(1).abs().max()) <= 2e-6
    # Tz beyond the support clamps to the end atoms
    big = 10 * (hi - lo)
    for r, k in ((big, K - 1), (-big, 0)):
        m = O.project(p, torch.full((5,), r), torch.zeros(5, dtype=torch.bool), 0.5, z, dz, lo, hi)
        want = torch.zeros(5, K)
        want[:, k] = 1.0
        torch.testing.assert_close(m, want, rtol=0, atol=2e-6)


def test_kl_is_nonnegative_and_zero_at_m_equals_p():
    p = _dist(32, 51, 9)
    logp = p.log()
    assert float(O.kl(p, logp).abs().max()) <= 1e-6
    m = _dist(32, 51, 10)
    m[:, :5] = 0                                   # 0 log 0 = 0
    m = m / m.sum(1, keepdim=True)
    k = O.kl(m, F.log_softmax(torch.randn(32, 51, generator=torch.Generator().manual_seed(2)), dim=1))
    assert bool(torch.isfinite(k).all()) and float(k.min()) >= 0.0


@pytest.mark.parametrize('double', [False, True])
def test_written_logit_gradient_is_autogradss(double):
    A, K, B, lo, hi = 4, 11, 6, -10.0, 10.0
    on, tg = default_q_state_dict(A, 0, num_atoms=K), default_q_state_dict(A, 1, num_atoms=K)
    g = torch.Generator().manual_seed(2)
    a, r, d, w = torch.randint(0, A, (B,), generator=g), 3 * torch.randn(B, generator=g), torch.rand(B, generator=g) < 0.3, torch.rand(B, generator=g) + 0.1
    obs = frames(B, 3)
    out = O.learn_step(on, tg, obs, a, r, frames(B, 4), d, weights=w, gamma=0.9, double_dqn=double,
                       head=O.Head('categorical', num_atoms=K, v_min=lo, v_max=hi))
    with torch.no_grad():
        logits = O.RefQNet(A, on, O.Head('categorical', num_atoms=K, v_min=lo, v_max=hi))(obs)
        p = F.softmax(logits, dim=2)[torch.arange(B), a]
    want = torch.zeros(B, A * K)
    dl = (w / B)[:, None] * (p * out['m'].sum(1, keepdim=True) - out['m'])       # (w / B) (p_k sum m - m_k) on the taken action
    for n in range(B):
        want[n, a[n] * K:(a[n] + 1) * K] = dl[n]
    torch.testing.assert_close(out['dlogits'], want, rtol=1e-5, atol=1e-8)
    assert float(out['loss']) == pytest.approx(float((w * out['ce']).mean()), rel=1e-6)
    # the q.bias gradient is the sum of the logit gradients over transitions
    torch.testing.assert_close(out['grads']['q.bias'], out['dlogits'].sum(0), rtol=1e-5, atol=1e-8)
    assert bool((out['kl'] >= 0).all()) and bool(torch.isfinite(out['kl']).all())


def test_initial_priorities_are_the_learners_kl():
    A, K, N, lo, hi = 4, 21, 5, 0.0, 200.0
    sd = default_q_state_dict(A, 2, num_atoms=K)
    head = O.Head('categorical', num_atoms=K, v_min=lo, v_max=hi)
    s, ns = frames(N, 1), frames(N, 2)
    a = torch.tensor([0, 1, 2, 3, 1])
    Rw = torch.tensor([0.5, -1.0, 2.0, 0.0, 0.25])
    d = torch.tensor([0, 1, 0, 0, 1], dtype=torch.bool)
    p = O.initial_priorities(sd, s, a, Rw, ns, d, 0.5, 1e-3, head=head)
    out = O.learn_step(sd, sd, s, a, Rw, ns, d, gamma=0.5, head=head)
    assert torch.equal(p, out['kl'].clamp(min=0).double() + 1e-3)
