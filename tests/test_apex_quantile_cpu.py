"""The quantile (QR-DQN) head of the Ape-X learner and actors without a GPU: the quantile_dqn switch and its checks, the refused
combinations in Python and C, AtariQNet(A, quantile=True) against the formula written out, the flat layout of
srl_apex_param_layout_quantile against apex_param_shapes with and without noise, the C argument errors of the quantile entry points,
sync_from on a head mismatch, and the oracle's closed forms (the written dtheta equals fp64 autograd of the loss; loss >= 0, 0 when
every quantile equals every target; rho inside |u| <= kappa; a done transition's target is r whatever s' holds), and no spills in the
new kernels."""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import apex_oracle as O
from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.apex import (APEX_NOISY_PARAM_NAMES, APEX_PARAM_NAMES, ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner,
                                          apex_param_shapes, default_q_state_dict, quantile_taus)
from scalerl_b200.algorithms.apex.learner import QHead
from tests.apex_cases import frames, unbuilt


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


def test_quantile_dqn_defaults_and_validation():
    hp = ApexHParams()
    assert hp.quantile_dqn is False and (hp.num_quantiles, hp.quantile_kappa) == (200, 1.0)
    c = hp.to_c()
    assert c.num_quantiles == 0 and hp.quantiles() == 0
    c = ApexHParams(quantile_dqn=True, num_quantiles=51, quantile_kappa=0.5).to_c()
    assert (c.num_quantiles, c.kappa, c.num_atoms, c.dueling) == (51, 0.5, 0, 0)
    assert ApexHParams(quantile_dqn=True).head == QHead(num_quantiles=200, kappa=1.0)
    assert ApexHParams(quantile_dqn=True, noisy_dqn=True).head == QHead(noisy=True, num_quantiles=200, kappa=1.0)
    # the existing heads are unchanged, as are their descriptions
    assert ApexHParams().head == QHead() and str(QHead()) == 'dueling_dqn=False, categorical_dqn=False, noisy_dqn=False'
    assert 'quantile' not in str(ApexHParams(categorical_dqn=True).head)
    for bad in (1, 0, 'yes', None):
        with pytest.raises(ValueError, match='quantile_dqn'):
            ApexHParams(quantile_dqn=bad).validate()
    for N in (1, 257, 0, 2.0, True, -3):
        with pytest.raises(ValueError, match='num_quantiles'):
            ApexHParams(quantile_dqn=True, num_quantiles=N).validate()
    for k in (0.0, -1.0, math.nan, math.inf, 1e39, True, '1'):
        with pytest.raises(ValueError, match='quantile_kappa'):
            ApexHParams(quantile_dqn=True, quantile_kappa=k).validate()
    with pytest.raises(ValueError, match='dueling'):
        ApexHParams(quantile_dqn=True, dueling_dqn=True).validate()
    with pytest.raises(ValueError, match='categorical'):
        ApexHParams(quantile_dqn=True, categorical_dqn=True).validate()
    for kw in (dict(dueling=True), dict(categorical=True)):
        with pytest.raises(ValueError, match='quantile'):
            AtariQNet(6, quantile=True, **kw)
    for kw, msg in ((dict(quantile_dqn=1), 'quantile_dqn'), (dict(quantile_dqn=True, num_quantiles=257), 'num_quantiles'),
                    (dict(quantile_dqn=True, quantile_kappa=0.0), 'quantile_kappa'), (dict(quantile_dqn=True, dueling_dqn=True), 'dueling'),
                    (dict(quantile_dqn=True, categorical_dqn=True), 'categorical')):
        with pytest.raises(ValueError, match=msg):
            B200ApexActor(4, 6, **kw)


@pytest.mark.parametrize('noisy', [False, True])
@pytest.mark.parametrize('A,N', [(1, 2), (6, 200), (18, 51), (31, 256)])
def test_quantile_net_names_shapes_and_flat_layout(A, N, noisy, lib):
    names = APEX_NOISY_PARAM_NAMES if noisy else APEX_PARAM_NAMES
    net = AtariQNet(A, quantile=True, num_quantiles=N, noisy=noisy)
    shapes = apex_param_shapes(A, noisy=noisy, num_quantiles=N)
    assert tuple(n for n, _ in net.named_parameters()) == names and tuple(net.state_dict()) == names
    assert {n: tuple(p.shape) for n, p in net.named_parameters()} == dict(shapes)
    w = 'q.weight_mu' if noisy else 'q.weight'
    assert shapes[w] == (A * N, 512)
    assert torch.equal(net.taus, quantile_taus(N)) and torch.equal(net.taus, O.taus(N))
    sd = default_q_state_dict(A, 3, noisy=noisy, num_quantiles=N)
    assert tuple(sd) == names and tuple(sd[w].shape) == (A * N, 512)
    # the encoder's initial weights are the plain network's (the head is drawn last)
    assert torch.equal(sd['fc.weight_mu' if noisy else 'fc.weight'], default_q_state_dict(A, 3, noisy=noisy)['fc.weight_mu' if noisy else 'fc.weight'])
    # the flat layout of the quantile entry point: every tensor's count, 4-float segments, no overlap, the head's rows before fc.weight
    total, off, cnt = _lib.apex_param_layout(A, noisy=noisy, num_quantiles=N)
    assert len(off) == len(cnt) == len(names)
    for (n, shp), c in zip(shapes.items(), cnt):
        assert c == int(torch.Size(shp).numel()), n
    assert all(o % 4 == 0 for o in off)
    spans = sorted(zip(off, cnt))
    for (o0, c0), (o1, _) in zip(spans, spans[1:]):
        assert o0 + c0 <= o1
    # the categorical layout of as many rows is the same buffer: the layout depends on the head's rows alone
    if N <= 64:
        assert _lib.apex_param_layout(A, noisy=noisy, num_atoms=N) == (total, off, cnt)
    # num_quantiles = 0 is srl_apex_param_layout_noisy's
    o18, c18 = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    q18, d18 = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    assert lib.srl_apex_param_layout_quantile(A, 0, 0, 0, int(noisy), q18, d18) == lib.srl_apex_param_layout_noisy(A, 0, 0, int(noisy), o18, c18)
    assert list(q18) == list(o18) and list(d18) == list(c18)


@pytest.mark.parametrize('A,N', [(1, 2), (6, 200)])
def test_quantile_forward_is_the_formula(A, N):
    torch.manual_seed(5)
    net = AtariQNet(A, quantile=True, num_quantiles=N)
    obs = torch.randint(0, 256, (7, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        x = obs.double() / 255.0
        p = {n: t.double() for n, t in net.state_dict().items()}
        x = F.relu(F.conv2d(x, p['conv1.weight'], p['conv1.bias'], stride=4))
        x = F.relu(F.conv2d(x, p['conv2.weight'], p['conv2.bias'], stride=2))
        x = F.relu(F.conv2d(x, p['conv3.weight'], p['conv3.bias'], stride=1))
        h = F.relu(x.reshape(7, -1) @ p['fc.weight'].T + p['fc.bias'])
        theta = (h @ p['q.weight'].T + p['q.bias']).view(7, A, N)          # row a N + i: quantile i of action a
        want_q = theta.sum(2) / N
        got_t, got_q = net.quantiles(obs).double(), net(obs).double()
    assert got_t.shape == (7, A, N) and got_q.shape == (7, A)
    assert float((got_t - theta).abs().max()) <= 1e-5 * max(1.0, float(theta.abs().max()))
    assert float((got_q - want_q).abs().max()) <= 1e-5 * max(1.0, float(theta.abs().max()))
    # the oracle's network computes the same quantiles from the same state dict
    assert torch.equal(O.RefQNet(A, net.state_dict(), O.Head('quantile', num_quantiles=N))(obs), net.quantiles(obs))
    with pytest.raises(ValueError, match='quantile'):
        AtariQNet(A).quantiles(obs)


def test_quantile_c_argument_errors(lib):
    off, cnt = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    for args, msg in (((6, 0, 0, 1, 0), b'num_quantiles=1'), ((6, 0, 0, 257, 0), b'num_quantiles=257'), ((6, 0, 0, -1, 0), b'num_quantiles=-1'),
                      ((6, 1, 0, 51, 0), b'dueling=1'), ((6, 0, 51, 51, 0), b'num_atoms=51'), ((32, 0, 0, 51, 0), b'A=32'),
                      ((6, 0, 0, 51, 2), b'noisy=2')):
        assert lib.srl_apex_param_layout_quantile(*args, off, cnt) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_param_layout: ') and msg in m, m
    h = C.c_void_p()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    nan, inf = float('nan'), float('inf')
    # (A, num_envs, precision, dueling, num_atoms, v_min, v_max, num_quantiles, kappa, noisy, seed, params)
    for args, msg in (((6, 4, 0, 0, 0, 0.0, 1.0, 51, 1.0, 0, 0, None), b'NULL'),
                      ((6, 4, 0, 0, 0, 0.0, 1.0, 1, 1.0, 0, 0, p), b'num_quantiles=1'),
                      ((6, 4, 0, 0, 0, 0.0, 1.0, 257, 1.0, 0, 0, p), b'num_quantiles=257'),
                      ((6, 4, 0, 0, 0, 0.0, 1.0, 51, 0.0, 0, 0, p), b'kappa=0'),
                      ((6, 4, 0, 0, 0, 0.0, 1.0, 51, -1.0, 0, 0, p), b'kappa=-1'),
                      ((6, 4, 0, 0, 0, 0.0, 1.0, 51, nan, 0, 0, p), b'kappa=nan'),
                      ((6, 4, 0, 0, 0, 0.0, 1.0, 51, inf, 0, 0, p), b'kappa=inf'),
                      ((6, 4, 0, 1, 0, 0.0, 1.0, 51, 1.0, 0, 0, p), b'dueling=1'),
                      ((6, 4, 0, 0, 51, 0.0, 1.0, 51, 1.0, 0, 0, p), b'num_atoms=51'),
                      ((6, 4, 2, 0, 0, 0.0, 1.0, 51, 1.0, 0, 0, p), b'precision=2')):
        assert lib.srl_apex_actor_create_quantile(*args, C.byref(h)) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_actor_create: ') and msg in m and b'\n' not in m, m
    # each refusal has its own message
    msgs = set()
    for kw in (dict(num_quantiles=1), dict(kappa=0.0), dict(dueling=1), dict(num_atoms=51)):
        args = dict(dueling=0, num_atoms=0, num_quantiles=51, kappa=1.0)
        args.update(kw)
        assert lib.srl_apex_actor_create_quantile(6, 4, 0, args['dueling'], args['num_atoms'], 0.0, 1.0, args['num_quantiles'], args['kappa'],
                                                  0, 0, p, C.byref(h)) == -1
        msgs.add(lib.srl_last_error().replace(b'=51', b'').replace(b'=1', b'').replace(b'=0', b''))
    assert len(msgs) == 4, msgs
    # the learner's config check runs before any CUDA call
    for kw, msg in ((dict(num_quantiles=257), b'num_quantiles=257'), (dict(num_quantiles=1), b'num_quantiles=1'), (dict(kappa=0.0), b'kappa=0'),
                    (dict(kappa=nan), b'kappa=nan'), (dict(dueling=1), b'dueling=1'), (dict(num_atoms=51), b'num_atoms=51')):
        cfg = ApexHParams(quantile_dqn=True).to_c()
        for k, v in kw.items():
            setattr(cfg, k, v)
        assert lib.srl_apex_learner_create(C.addressof(cfg), p, p, p, p, p, C.byref(h)) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_learner: ') and msg in m, m
    # num_quantiles = 0 is not the quantile head: kappa is not read
    cfg = ApexHParams().to_c()
    assert (cfg.num_quantiles, cfg.kappa) == (0, 1.0)
    cfg.kappa = nan
    assert lib.srl_apex_learner_create(C.addressof(cfg), None, p, p, p, p, C.byref(h)) == -1
    assert b'NULL' in lib.srl_last_error()


@pytest.mark.parametrize('learner,msg', [(dict(quantile_dqn=False), 'quantile_dqn'), (dict(num_quantiles=51), 'num_quantiles'),
                                         (dict(quantile_kappa=0.5), 'quantile_kappa'), (dict(noisy_dqn=True), 'noisy_dqn')])
def test_sync_from_needs_the_same_head(learner, msg):
    hp = dict(num_actions=6, quantile_dqn=True, num_quantiles=200, quantile_kappa=1.0)
    hp.update(learner)
    L = unbuilt(B200ApexLearner, hp=ApexHParams(**hp), device=torch.device('cuda', 0))
    X = unbuilt(B200ApexActor, num_envs=4, num_actions=6, quantile_dqn=True, num_quantiles=200, quantile_kappa=1.0,
                 device=torch.device('cuda', 0), _h=None)
    with pytest.raises(ValueError, match=msg):
        X.sync_from(L)
    # and the other way round: a quantile learner, a plain actor
    X = unbuilt(B200ApexActor, num_envs=4, num_actions=6, device=torch.device('cuda', 0), _h=None)
    with pytest.raises(ValueError, match='quantile_dqn'):
        X.sync_from(unbuilt(B200ApexLearner, hp=ApexHParams(num_actions=6, quantile_dqn=True), device=torch.device('cuda', 0)))


# ---------------------------------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize('kappa', [1.0, 0.5])
@pytest.mark.parametrize('double', [False, True])
def test_written_dtheta_is_fp64_autograd(double, kappa):
    A, N, B = 4, 11, 6
    on, tg = default_q_state_dict(A, 0, num_quantiles=N), default_q_state_dict(A, 1, num_quantiles=N)
    g = torch.Generator().manual_seed(2)
    a, r, d, w = torch.randint(0, A, (B,), generator=g), torch.randn(B, generator=g), torch.rand(B, generator=g) < 0.3, torch.rand(B, generator=g) + 0.1
    obs = frames(B, 3)
    out = O.learn_step(on, tg, obs, a, r, frames(B, 4), d, weights=w, gamma=0.9, double_dqn=double, head=O.Head('quantile', num_quantiles=N, kappa=kappa))
    # fp64 autograd of mean(w loss) with respect to theta, from the oracle's own theta and targets
    theta = out['theta'].double().requires_grad_(True)
    ta = theta[torch.arange(B), a]
    loss = (w.double() * O.quantile_loss(ta, out['T'].double(), kappa)).mean()
    loss.backward()
    want = theta.grad.reshape(B, A * N)
    torch.testing.assert_close(out['dtheta'].double(), want, rtol=1e-5, atol=1e-9)
    torch.testing.assert_close(out['dtheta_autograd'].double(), want, rtol=1e-5, atol=1e-9)
    assert float(loss.detach()) == pytest.approx(out["loss"], rel=1e-6)
    assert float(out['loss']) == pytest.approx(float((w * out['loss_n']).mean()), rel=1e-6)
    # zero outside the taken action's rows; the q.bias gradient is the sum of the dtheta rows over transitions
    mask = torch.zeros(B, A, N, dtype=torch.bool)
    mask[torch.arange(B), a] = True
    assert not bool(out['dtheta'].view(B, A, N)[~mask].any())
    torch.testing.assert_close(out['grads']['q.bias'], out['dtheta'].sum(0), rtol=1e-5, atol=1e-8)
    assert bool((out['loss_n'] >= 0).all())


@pytest.mark.parametrize('kappa', [1.0, 0.5, 3.0])
def test_quantile_loss_closed_forms(kappa):
    g = torch.Generator().manual_seed(4)
    N = 17
    th, T = 2 * torch.randn(32, N, generator=g, dtype=torch.float64), 2 * torch.randn(32, N, generator=g, dtype=torch.float64)
    assert bool((O.quantile_loss(th, T, kappa) >= 0).all())
    # every theta_i equal to every T_j: u = 0 everywhere, no loss and no gradient
    c = torch.randn(32, 1, generator=g, dtype=torch.float64).expand(32, N)
    assert float(O.quantile_loss(c, c, kappa).abs().max()) == 0.0
    assert float(O.dtheta_written(c, c, kappa, torch.ones(32, dtype=torch.float64)).abs().max()) == 0.0
    # inside |u| <= kappa: rho = |tau - 1{u < 0}| u^2 / (2 kappa)
    small = th[:, :1] + (kappa / 3) * torch.rand(32, N, generator=g, dtype=torch.float64)
    u = small[:, None, :] - th[:, :1, None].expand(32, N, 1)
    tau = O.taus(N, torch.float64)[None, :, None]
    rho = O.rho(th[:, :1].expand(32, N), small, kappa)
    assert bool((u.abs() <= kappa).all())
    torch.testing.assert_close(rho, (tau - (u < 0).double()).abs() * u * u / (2 * kappa), rtol=1e-12, atol=0)
    # outside: rho = |tau - 1{u < 0}| (|u| - kappa / 2)
    far = th[:, :1] + 3 * kappa + torch.rand(32, N, generator=g, dtype=torch.float64)
    rho = O.rho(th[:, :1].expand(32, N), far, kappa)
    uf = far[:, None, :] - th[:, :1, None].expand(32, N, 1)
    torch.testing.assert_close(rho, tau * (uf.abs() - kappa / 2), rtol=1e-12, atol=1e-12)
    # tau_i is the midpoint of the i-th of N equal probability bins
    assert torch.equal(O.taus(4), torch.tensor([0.125, 0.375, 0.625, 0.875]))


def test_done_target_is_the_reward_whatever_s_prime_holds():
    n, A, N = 6, 3, 8
    bad = torch.full((n, A, N), math.inf)
    bad[1, 2, 3] = math.nan
    r = torch.arange(n, dtype=torch.float32) - 2.5
    done = torch.ones(n, dtype=torch.bool)
    T = O.targets(bad, r, done, 0.99, theta_next_online=bad)
    assert torch.equal(T, r[:, None].expand(n, N))
    # not done: r + gamma theta'(s')[a*], a* the first argmax of the quantile means (ties: the first index)
    g = torch.Generator().manual_seed(1)
    tn = torch.randn(n, A, N, generator=g)
    tn[:, 2] = tn[:, 0]
    tn[:, 0] += 5.0
    tn[:, 2] += 5.0
    T = O.targets(tn, r, torch.zeros(n, dtype=torch.bool), 0.99)
    torch.testing.assert_close(T, r[:, None] + torch.tensor(np.float32(0.99)) * tn[:, 0], rtol=0, atol=0)


def test_initial_priorities_are_the_learners_loss():
    A, N, n = 4, 21, 5
    sd = default_q_state_dict(A, 2, num_quantiles=N)
    head = O.Head('quantile', num_quantiles=N, kappa=0.5)
    s, ns = frames(n, 1), frames(n, 2)
    a = torch.tensor([0, 1, 2, 3, 1])
    Rw = torch.tensor([0.5, -1.0, 2.0, 0.0, 0.25])
    d = torch.tensor([0, 1, 0, 0, 1], dtype=torch.bool)
    p = O.initial_priorities(sd, s, a, Rw, ns, d, 0.5, 1e-3, head=head)
    out = O.learn_step(sd, sd, s, a, Rw, ns, d, gamma=0.5, head=head)
    assert torch.equal(p, out['loss_n'].double() + 1e-3)


def test_quantile_kernels_do_not_spill(lib):
    rep = srl_build.ptxas_report()
    want = {'dqn_qr.cu': ['qr_tail_kernel'], 'apex_actor.cu': ['apex_qr_priority_kernel', 'apex_act_kernelILNS_5QKindE3'],
            'dqn.cu': ['q_values_kernelILNS_5QKindE3']}
    for src, kernels in want.items():
        for k in kernels:
            hits = [(name, v) for name, v in rep[src].items() if k in name]
            assert len(hits) == 1, (src, k, list(rep[src]))
            name, v = hits[0]
            assert v['spill_stores'] == 0 and v['spill_loads'] == 0, (name, v)
