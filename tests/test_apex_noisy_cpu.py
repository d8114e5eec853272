"""Noisy networks for the Ape-X learner and actors without a GPU: the noisy_dqn / noisy_std switches and their checks, names, shapes and
Adam state order for all three heads, the 14 / 18-tensor flat layout and its C argument errors, sync_from's head check,
AtariQNet(noisy=True) against the formula written out (train mode), the plain network on mu (eval mode) and the initialisation of
Fortunato et al. 2018 section 3.2, the oracle's sigma gradient against dW * eps, and the new kernels' ptxas report."""
import ctypes as C
import math

import pytest
import torch
import torch.nn.functional as F

from oracle import apex_oracle as O
from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.apex import (APEX_NOISY_DUELING_PARAM_NAMES, APEX_NOISY_PARAM_NAMES, APEX_PARAM_NAMES, ApexHParams, AtariQNet,
                                          B200ApexActor, B200ApexLearner, NoisyLinear, apex_param_shapes, default_q_state_dict)
from scalerl_b200.algorithms.apex.learner import QHead, scale_noise
from tests.apex_cases import frames, unbuilt

HEADS = {'plain': dict(), 'dueling': dict(dueling=True), 'categorical': dict(categorical=True, num_atoms=5)}


@pytest.fixture(scope='module')
def lib():
    srl_build.build()
    return _lib.lib()


def test_noisy_switch_defaults_and_validation():
    hp = ApexHParams()
    assert hp.noisy_dqn is False and hp.noisy_std == 0.5 and hp.to_c().noisy == 0
    assert ApexHParams(noisy_dqn=True).to_c().noisy == 1
    assert ApexHParams(noisy_dqn=True, dueling_dqn=True).head == QHead(True, noisy=True)
    assert ApexHParams(noisy_dqn=True, categorical_dqn=True).head.noisy
    ApexHParams(noisy_dqn=True, noisy_std=0.0).validate()
    for bad in (1, 0, 'yes', None):
        with pytest.raises(ValueError, match='noisy_dqn'):
            ApexHParams(noisy_dqn=bad).validate()
    for bad in (-0.1, math.inf, math.nan, None, True):
        with pytest.raises(ValueError, match='noisy_std'):
            ApexHParams(noisy_dqn=True, noisy_std=bad).validate()
    with pytest.raises(ValueError, match='noisy_dqn'):
        B200ApexActor(4, 6, noisy_dqn=1)
    with pytest.raises(ValueError, match='noisy_std'):
        B200ApexActor(4, 6, noisy_dqn=True, noisy_std=-1.0)
    with pytest.raises(ValueError, match='categorical_dqn with dueling_dqn'):
        ApexHParams(noisy_dqn=True, dueling_dqn=True, categorical_dqn=True).validate()
    assert 'noisy_dqn=True' in str(ApexHParams(noisy_dqn=True).head)


@pytest.mark.parametrize('head', list(HEADS))
@pytest.mark.parametrize('A', [1, 6, 18])
def test_noisy_names_shapes_and_adam_order(A, head):
    kw = HEADS[head]
    dueling, K = kw.get('dueling', False), kw.get('num_atoms', 0)
    net = AtariQNet(A, noisy=True, **kw)
    want = APEX_NOISY_DUELING_PARAM_NAMES if dueling else APEX_NOISY_PARAM_NAMES
    assert len(want) == (18 if dueling else 14)
    assert tuple(n for n, _ in net.named_parameters()) == want and tuple(net.state_dict()) == want
    shapes = apex_param_shapes(A, dueling, K, noisy=True)
    assert {n: tuple(p.shape) for n, p in net.named_parameters()} == dict(shapes) and tuple(shapes) == want
    R = A * K if K else A
    assert shapes['fc.weight_sigma'] == (512, 3136) and shapes['fc.bias_sigma'] == (512,)
    if not dueling:
        assert shapes['q.weight_mu'] == (R, 512) and shapes['q.bias_sigma'] == (R,)
    hd = QHead.of(dueling, K > 0, K or 51, 0.0, 200.0 if K else 200.0, True)
    assert tuple(hd.names()) == want
    # torch.optim.Adam over the noisy net: integer keys in the same order
    opt = torch.optim.Adam(net.parameters())
    assert opt.state_dict()['param_groups'][0]['params'] == list(range(len(want)))
    # the noise buffers are not in the state dict, and the plain network is unchanged
    assert not any('eps' in n for n in net.state_dict())
    assert tuple(AtariQNet(A).state_dict()) == APEX_PARAM_NAMES
    sd = default_q_state_dict(A, 3, dueling, K, noisy=True)
    assert tuple(sd) == want and all(torch.equal(sd[n], default_q_state_dict(A, 3, dueling, K, noisy=True)[n]) for n in want)


@pytest.mark.parametrize('head', list(HEADS))
def test_noisy_train_forward_is_the_formula_and_eval_is_mu(head):
    kw = HEADS[head]
    A = 6
    torch.manual_seed(5)
    net = AtariQNet(A, noisy=True, **kw)
    obs = torch.randint(0, 256, (7, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    p = {n: t.double() for n, t in net.state_dict().items()}
    layers = [m for m in net.noisy_layers()]
    assert len(layers) == (3 if kw.get('dueling') else 2)

    def eff(name, train):
        m = getattr(net, name)
        if not train:
            return p[f'{name}.weight_mu'], p[f'{name}.bias_mu']
        eo, ei = m.eps_out.double(), m.eps_in.double()
        return p[f'{name}.weight_mu'] + p[f'{name}.weight_sigma'] * torch.outer(eo, ei), p[f'{name}.bias_mu'] + p[f'{name}.bias_sigma'] * eo

    for train in (True, False):
        net.train(train)
        with torch.no_grad():
            x = obs.double() / 255.0
            x = F.relu(F.conv2d(x, p['conv1.weight'], p['conv1.bias'], stride=4))
            x = F.relu(F.conv2d(x, p['conv2.weight'], p['conv2.bias'], stride=2))
            x = F.relu(F.conv2d(x, p['conv3.weight'], p['conv3.bias'], stride=1))
            h = F.relu(F.linear(x.reshape(7, -1), *eff('fc', train)))
            if kw.get('dueling'):
                v, adv = F.linear(h, *eff('value', train)), F.linear(h, *eff('advantage', train))
                want = v + adv - adv.mean(1, keepdim=True)
            elif kw.get('categorical'):
                pr = F.softmax(F.linear(h, *eff('q', train)).view(7, A, -1), dim=2)
                want = (pr * net.support.double()).sum(2)
                assert torch.allclose(net.dist(obs).double(), pr, rtol=1e-4, atol=1e-6)
            else:
                want = F.linear(h, *eff('q', train))
            got = net(obs).double()
        assert float((got - want).abs().max()) <= 1e-5 * float(want.abs().max()), (train, float((got - want).abs().max()))
    # eval mode is the plain network loaded with mu
    plain = AtariQNet(A, **kw)
    plain.load_state_dict({n.replace('_mu', ''): t for n, t in net.state_dict().items() if 'sigma' not in n})
    net.eval()
    with torch.no_grad():
        assert torch.equal(net(obs), plain(obs))
        net.train()
        noisy_q = net(obs)
        net.reset_noise()
        assert not torch.equal(net(obs), noisy_q)           # new noise, new Q


@pytest.mark.parametrize('std', [0.5, 0.1, 0.0])
def test_noisy_init_bounds_and_sigma(std):
    torch.manual_seed(0)
    net = AtariQNet(6, noisy=True, dueling=True, noisy_std=std)
    for m in net.noisy_layers():
        p = m.in_features
        for t in (m.weight_mu.detach(), m.bias_mu.detach()):
            assert float(t.abs().max()) <= 1 / math.sqrt(p)
            assert t.numel() < 64 or float(t.abs().max()) > 0.9 / math.sqrt(p)      # the whole range is used
        want = torch.tensor(std / math.sqrt(p), dtype=torch.float32)
        assert bool((m.weight_sigma == want).all()) and bool((m.bias_sigma == want).all())
        assert torch.equal(m.weight_epsilon, torch.outer(m.eps_out, m.eps_in)) and torch.equal(m.bias_epsilon, m.eps_out)
    if std == 0.0:                                          # sigma 0: the noisy net is its mean
        obs = torch.randint(0, 256, (3, 4, 84, 84), dtype=torch.uint8)
        with torch.no_grad():
            q = net(obs)
            net.eval()
            assert torch.equal(q, net(obs))
    # construction order under one seed fixes mu and the first noise
    torch.manual_seed(0)
    again = AtariQNet(6, noisy=True, dueling=True, noisy_std=std)
    assert all(torch.equal(a, b) for a, b in zip(net.state_dict().values(), again.state_dict().values()))


def test_scale_noise_and_set_noise():
    x = torch.tensor([-4.0, -0.25, 0.0, 0.25, 9.0])
    assert torch.equal(scale_noise(x), torch.tensor([-2.0, -0.5, 0.0, 0.5, 3.0]))
    m = NoisyLinear(3, 2)
    m.set_noise(torch.tensor([1.0, -2.0, 0.5]), torch.tensor([0.5, -1.0]))
    assert torch.equal(m.weight_epsilon, torch.tensor([[0.5, -1.0, 0.25], [-1.0, 2.0, -0.5]]))


@pytest.mark.parametrize('head', list(HEADS))
@pytest.mark.parametrize('A', [1, 6, 18, 31])
def test_noisy_flat_layout(A, head, lib):
    kw = HEADS[head]
    dueling, K = kw.get('dueling', False), kw.get('num_atoms', 0)
    for K_ in ((K,) if head != 'categorical' else (0, 51)):
        if head == 'categorical' and K_ == 0:
            continue
        total, off, cnt = _lib.apex_param_layout(A, dueling, K_, noisy=True)
        shapes = apex_param_shapes(A, dueling, K_, noisy=True)
        names = list(shapes)
        assert len(off) == len(cnt) == len(names) == (18 if dueling else 14)
        for (n, shp), c in zip(shapes.items(), cnt):
            assert c == int(torch.Size(shp).numel()), n
        assert all(o % 4 == 0 for o in off)
        spans = sorted(zip(off, cnt))
        for (o0, c0), (o1, _) in zip(spans, spans[1:]):
            assert o0 + c0 <= o1
        assert total == spans[-1][0] + spans[-1][1]
        assert spans[-1][0] == off[names.index('fc.weight_sigma')] and spans[-2][0] == off[names.index('fc.weight_mu')]
        if dueling:        # the mu rows and the sigma rows are one [(A + 1), 512] block each
            for s in ('mu', 'sigma'):
                assert off[names.index(f'advantage.weight_{s}')] == off[names.index(f'value.weight_{s}')] + 512
                assert off[names.index(f'advantage.bias_{s}')] == off[names.index(f'value.bias_{s}')] + 4
    # noisy = 0 through the new entry point is the existing layouts
    o, c = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    for d, k in ((0, 0), (1, 0), (0, 51)):
        t = lib.srl_apex_param_layout_noisy(A, d, k, 0, o, c)
        n = 12 if d else 10
        assert (t, list(o)[:n], list(c)[:n]) == _lib.apex_param_layout(A, bool(d), k)


def test_noisy_c_argument_errors(lib):
    off, cnt = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    for args, msg in (((6, 0, 0, 2), b'noisy=2'), ((6, 0, 0, -1), b'noisy=-1'), ((0, 0, 0, 1), b'A=0'), ((32, 1, 0, 1), b'A=32'),
                      ((6, 2, 0, 1), b'dueling=2'), ((6, 0, 1, 1), b'num_atoms=1'), ((6, 1, 51, 1), b'dueling=1 is not supported')):
        assert lib.srl_apex_param_layout_noisy(*args, off, cnt) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_param_layout: ') and msg in m, m
    with pytest.raises(ValueError, match='noisy=2'):
        _lib.check(-1 if lib.srl_apex_param_layout_noisy(6, 0, 0, 2, off, cnt) < 0 else 0, 'layout')
    h = C.c_void_p()
    buf = (C.c_float * 64)()
    p = C.addressof(buf)
    for args, msg in (((6, 4, 0, 0, 0, 0.0, 1.0, 1, 0, None), b'NULL'), ((6, 4, 0, 0, 0, 0.0, 1.0, 2, 0, p), b'noisy=2'),
                      ((6, 4, 0, 0, 0, 0.0, 1.0, -1, 0, p), b'noisy=-1'), ((0, 4, 0, 0, 0, 0.0, 1.0, 1, 0, p), b'A=0'),
                      ((6, 4, 0, 1, 51, 0.0, 1.0, 1, 0, p), b'dueling=1 is not supported'), ((6, 4, 2, 0, 0, 0.0, 1.0, 1, 0, p), b'precision=2')):
        assert lib.srl_apex_actor_create_noisy(*args, C.byref(h)) == -1
        m = lib.srl_last_error()
        assert m.startswith(b'apex_actor_create: ') and msg in m and b'\n' not in m, m
    cfg = ApexHParams(noisy_dqn=True).to_c()
    cfg.noisy = 2
    assert lib.srl_apex_learner_create(C.addressof(cfg), p, p, p, p, p, C.byref(h)) == -1
    assert b'noisy=2' in lib.srl_last_error()


@pytest.mark.parametrize('learner,actor', [(dict(noisy_dqn=True), dict(noisy_dqn=False)), (dict(noisy_dqn=False), dict(noisy_dqn=True)),
                                           (dict(noisy_dqn=True), dict(noisy_dqn=True, dueling_dqn=True)),
                                           (dict(noisy_dqn=True, categorical_dqn=True), dict(noisy_dqn=True))])
def test_sync_from_needs_the_same_noisy_head(learner, actor):
    L = unbuilt(B200ApexLearner, hp=ApexHParams(num_actions=6, **learner), device=torch.device('cuda', 0))
    X = unbuilt(B200ApexActor, num_envs=4, num_actions=6, device=torch.device('cuda', 0), _h=None, **actor)
    with pytest.raises(ValueError, match='noisy_dqn'):
        X.sync_from(L)


@pytest.mark.parametrize('head', list(HEADS))
def test_oracle_sigma_gradient_is_dW_times_eps(head):
    kw = HEADS[head]
    A, B = 5, 6
    dueling, K = kw.get('dueling', False), kw.get('num_atoms', 0)
    on = default_q_state_dict(A, 0, dueling, K, noisy=True)
    tg = default_q_state_dict(A, 1, dueling, K, noisy=True)
    R = A * K if K else A + dueling
    g = torch.Generator().manual_seed(2)
    nn_ = 3648 + 512 * (1 + dueling) + R
    n_on, n_tg = scale_noise(torch.randn(nn_, generator=g)), scale_noise(torch.randn(nn_, generator=g))
    batch = (frames(B, 3), torch.randint(0, A, (B,), generator=g), torch.randn(B, generator=g), frames(B, 4), torch.rand(B, generator=g) < 0.3)
    oh = O.Head('dueling' if dueling else 'categorical' if K else 'plain', noisy=True, num_atoms=K, v_min=-10.0, v_max=10.0)
    out = O.learn_step(on, tg, *batch, double_dqn=True, head=oh, noise_online=n_on, noise_target=n_tg)
    assert tuple(out['grads']) == O.names(dueling)
    # the gradient of the composed weight W is the mu gradient; sigma's is dW * eps (autograd's own rounding: bit for bit)
    for name, (ei, eo) in O.split_noise(n_on, A, dueling, K).items():
        gW, gb = out['grads'][f'{name}.weight_mu'], out['grads'][f'{name}.bias_mu']
        assert torch.equal(out['grads'][f'{name}.weight_sigma'], gW * torch.outer(eo, ei)), name
        assert torch.equal(out['grads'][f'{name}.bias_sigma'], gb * eo), name
        assert float(gW.abs().max()) > 0 or (name == 'advantage' and A == 1)
    # the oracle's composed weights are composed() in torch's order
    net = O.RefQNet(A, on, oh, n_on)
    for name, (W, b) in O.composed(on, n_on, A, dueling, K).items():
        w2, b2 = getattr(net, name).weights()
        assert torch.equal(W, w2) and torch.equal(b, b2)


def test_new_kernels_do_not_spill(lib):
    rep = srl_build.ptxas_report()
    kernels = rep['noisy.cu']
    assert {k for k in kernels if 'noisy_draw_kernel' in k or 'noisy_compose_kernel' in k or 'noisy_sigma_grad_kernel' in k} and len(kernels) == 3
    for k, v in kernels.items():
        assert v['spill_stores'] == 0 and v['spill_loads'] == 0 and v['regs'] is not None, (k, v)
