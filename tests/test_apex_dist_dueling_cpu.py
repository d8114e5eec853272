"""The distributional dueling head of the Ape-X learner and actors (Rainbow's per-atom dueling C51 and per-quantile dueling QR-DQN), on
the CPU: the settings and their refusals in Python and in C, the parameter layout against AtariQNet for every A, W and noise setting,
the reparametrisation the device runs (composed rows and decomposed gradients) in fp64, the oracle against the CPU network, and the
new kernels' register budget.  No GPU needed."""
import ctypes as C

import pytest
import torch

from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.apex import ApexHParams, AtariQNet
from scalerl_b200.algorithms.apex.learner import QHead, apex_param_shapes
from tests import apex_dist_dueling_ref as R

F64 = torch.float64


# ---------------------------------------------------------------------------------------------------------------- settings
def test_hparams_accept_the_head_with_either_distributional_head():
    c51 = ApexHParams(categorical_dqn=True, num_atoms=11, distributional_dueling=True)
    qr = ApexHParams(quantile_dqn=True, num_quantiles=32, distributional_dueling=True, noisy_dqn=True)
    assert c51.head == QHead(num_atoms=11, v_min=0.0, v_max=200.0, dist_dueling=True)
    assert qr.head == QHead(noisy=True, num_quantiles=32, kappa=1.0, dist_dueling=True)
    assert c51.to_c().dist_dueling == 1 and qr.to_c().dist_dueling == 1
    assert ApexHParams(categorical_dqn=True).to_c().dist_dueling == 0 and ApexHParams().to_c().dist_dueling == 0
    assert c51.head.names() == QHead(dueling=True).names()
    assert list(c51.head.shapes(6).items())[-4:] == [('value.weight', (11, 512)), ('value.bias', (11,)),
                                                     ('advantage.weight', (66, 512)), ('advantage.bias', (66,))]


@pytest.mark.parametrize('kw,msg', [
    (dict(distributional_dueling=True), 'distributional_dueling needs categorical_dqn or quantile_dqn'),
    (dict(distributional_dueling=True, dueling_dqn=True), 'distributional_dueling with dueling_dqn is not supported'),
    (dict(distributional_dueling=True, dueling_dqn=True, quantile_dqn=True), 'quantile_dqn with dueling_dqn is not supported'),
    (dict(distributional_dueling=True, dueling_dqn=True, categorical_dqn=True), 'categorical_dqn with dueling_dqn is not supported'),
    (dict(distributional_dueling=1, categorical_dqn=True), 'distributional_dueling must be a bool'),
    (dict(distributional_dueling='yes', quantile_dqn=True), 'distributional_dueling must be a bool'),
])
def test_hparams_refuse_bad_settings(kw, msg):
    with pytest.raises(ValueError, match=msg):
        ApexHParams(**kw).validate()
    with pytest.raises(ValueError, match=msg):
        ApexHParams(**kw).to_c()


def test_head_names_itself_only_when_set():
    """the existing heads' strings are unchanged, so sync_from names the mismatch with a dueling-distributional learner"""
    plain = QHead.of(False, True, 51, 0.0, 200.0)
    dd = QHead.of(False, True, 51, 0.0, 200.0, distributional_dueling=True)
    assert str(plain) == 'dueling_dqn=False, categorical_dqn=True, noisy_dqn=False, (num_atoms, v_min, v_max)=(51, 0.0, 200.0)'
    assert str(dd) == str(plain) + ', distributional_dueling=True'
    qr = QHead.of(False, False, 51, 0.0, 200.0, False, True, 200, 1.0, True)
    assert str(qr).endswith('quantile_dqn=True, (num_quantiles, quantile_kappa)=(200, 1.0), distributional_dueling=True')
    assert 'distributional' not in str(QHead.of(True, False, 51, 0.0, 200.0))
    assert plain != dd


def test_atari_qnet_builds_the_dueling_rows():
    net = AtariQNet(6, categorical=True, num_atoms=11, distributional_dueling=True)
    assert list(net.state_dict()) == list(QHead(dueling=True).names())
    assert tuple(net.value.weight.shape) == (11, 512) and tuple(net.advantage.weight.shape) == (66, 512)
    assert 'support' in dict(net.named_buffers()) and 'support' not in net.state_dict()
    noisy = AtariQNet(4, quantile=True, num_quantiles=8, noisy=True, distributional_dueling=True)
    assert list(noisy.state_dict()) == list(QHead(dueling=True, noisy=True).names()) and len(noisy.state_dict()) == 18
    assert 'taus' in dict(noisy.named_buffers()) and len(noisy.noisy_layers()) == 3
    with pytest.raises(ValueError, match='needs the categorical or the quantile head'):
        AtariQNet(6, distributional_dueling=True)
    with pytest.raises(ValueError, match='categorical head with the dueling head'):
        AtariQNet(6, dueling=True, categorical=True)
    with pytest.raises(ValueError, match='categorical head with the dueling head'):
        AtariQNet(6, dueling=True, categorical=True, distributional_dueling=True)


@pytest.mark.parametrize('head', ['categorical', 'quantile'])
def test_atari_qnet_rows_are_the_formula(head):
    torch.manual_seed(3)
    A, W = 5, 7
    net = AtariQNet(A, categorical=head == 'categorical', quantile=head == 'quantile', num_atoms=W, num_quantiles=W,
                    distributional_dueling=True, v_min=-10.0, v_max=10.0)
    obs = torch.randint(0, 256, (3, 4, 84, 84), dtype=torch.uint8)
    h = net._features(obs)
    v, adv = net.value(h), net.advantage(h).view(-1, A, W)
    rows = v[:, None, :] + adv - adv.mean(1, keepdim=True)
    with torch.no_grad():
        if head == 'categorical':
            assert torch.equal(net.dist(obs), torch.softmax(rows, dim=2))
            assert torch.equal(net(obs), (torch.softmax(rows, dim=2) * net.support).sum(2))
        else:
            assert torch.equal(net.quantiles(obs), rows)
            assert torch.equal(net(obs), rows.mean(2))


# ---------------------------------------------------------------------------------------------------------------- C refusals
def _cfg(**kw):
    c = ApexHParams(batch_size=32, num_actions=6).to_c()
    for k, v in kw.items():
        setattr(c, k, v)
    return c


@pytest.mark.parametrize('kw,msg', [
    (dict(dist_dueling=2, num_atoms=51), 'dist_dueling=2 must be 0 or 1'),
    (dict(dist_dueling=-1, num_quantiles=8), 'dist_dueling=-1 must be 0 or 1'),
    (dict(dist_dueling=1), 'dist_dueling=1 needs the categorical head (num_atoms > 0) or the quantile head (num_quantiles > 0)'),
    (dict(dist_dueling=1, dueling=1, num_atoms=51), 'dist_dueling=1 with dueling=1 is not supported'),
    (dict(dist_dueling=1, dueling=1, num_quantiles=8), 'dist_dueling=1 with dueling=1 is not supported'),
])
def test_c_refusals_before_any_cuda_call(kw, msg):
    """the learner and the actor refuse a bad setting from the config alone (no buffers, no device)"""
    L = _lib.lib()
    cfg = _cfg(**kw)
    h = C.c_void_p()
    assert L.srl_apex_learner_create(C.addressof(cfg), None, None, None, None, None, C.byref(h)) == -1
    assert L.srl_last_error().decode().startswith('apex_learner: ') and msg in L.srl_last_error().decode()
    fake = C.c_void_p(1 << 20)            # never dereferenced: the setting is refused first
    rc = L.srl_apex_actor_create_dist_dueling(6, 4, 0, cfg.dueling, cfg.num_atoms, 0.0, 10.0, cfg.num_quantiles, 1.0, cfg.dist_dueling, 0,
                                              0, fake, C.byref(h))
    assert rc == -1
    assert L.srl_last_error().decode().startswith('apex_actor_create: ') and msg in L.srl_last_error().decode()


def test_older_entry_points_keep_their_refusals():
    """dueling with the categorical or quantile head keeps its text through every entry point when dist_dueling is 0"""
    L = _lib.lib()
    off, cnt = (C.c_int64 * 18)(), (C.c_int64 * 18)()
    assert L.srl_apex_param_layout_dist_dueling(6, 1, 51, 0, 0, 0, off, cnt) == -1
    assert L.srl_last_error().decode() == 'apex_param_layout: the categorical head (num_atoms=51) with dueling=1 is not supported'
    assert L.srl_apex_param_layout_dist_dueling(6, 1, 0, 8, 0, 0, off, cnt) == -1
    assert L.srl_last_error().decode() == 'apex_param_layout: the quantile head (num_quantiles=8) with dueling=1 is not supported'
    assert L.srl_apex_param_layout_dist_dueling(6, 0, 51, 8, 1, 0, off, cnt) == -1
    assert 'with the categorical head (num_atoms=51) is not supported' in L.srl_last_error().decode()


# ---------------------------------------------------------------------------------------------------------------- layout
def _expected_layout(A, W, noisy):
    """the layout rule written out: state_dict names and shapes, and the memory order conv | fc bias | head weights | head biases |
    fc weight (noisy: conv | fc biases | head biases | head weights | fc weights, mu before sigma), each segment padded to 4 floats"""
    conv = [('conv1.weight', (32, 4, 8, 8)), ('conv1.bias', (32,)), ('conv2.weight', (64, 32, 4, 4)), ('conv2.bias', (64,)),
            ('conv3.weight', (64, 64, 3, 3)), ('conv3.bias', (64,))]
    rows = {'fc': 512, 'value': W, 'advantage': A * W}
    ins = {'fc': 3136, 'value': 512, 'advantage': 512}
    if noisy:
        sfx = ('weight_mu', 'weight_sigma', 'bias_mu', 'bias_sigma')
        state = conv + [(f'{l}.{s}', (rows[l], ins[l]) if s.startswith('weight') else (rows[l],)) for l in ('fc', 'value', 'advantage')
                        for s in sfx]
        memory = [n for n, _ in conv] + ['fc.bias_mu', 'fc.bias_sigma', 'value.bias_mu', 'advantage.bias_mu', 'value.bias_sigma',
                                          'advantage.bias_sigma', 'value.weight_mu', 'advantage.weight_mu', 'value.weight_sigma',
                                          'advantage.weight_sigma', 'fc.weight_mu', 'fc.weight_sigma']
    else:
        state = conv + [(f'{l}.{s}', (rows[l], ins[l]) if s == 'weight' else (rows[l],)) for l in ('fc', 'value', 'advantage')
                        for s in ('weight', 'bias')]
        memory = [n for n, _ in conv] + ['fc.bias', 'value.weight', 'advantage.weight', 'value.bias', 'advantage.bias', 'fc.weight']
    shapes = dict(state)
    off, o = {}, 0
    for n in memory:
        off[n] = o
        o += -(-torch.Size(shapes[n]).numel() // 4) * 4
    return state, off, o


@pytest.mark.parametrize('noisy', [False, True])
@pytest.mark.parametrize('kind,W', [('categorical', 2), ('categorical', 51), ('categorical', 64), ('quantile', 2), ('quantile', 200),
                                    ('quantile', 256)])
def test_layout_matches_atari_qnet_and_the_rule(kind, W, noisy):
    K, N = (W, 0) if kind == 'categorical' else (0, W)
    for A in range(1, 32):
        state, off_want, total_want = _expected_layout(A, W, noisy)
        total, off, cnt = _lib.apex_param_layout(A, False, K, noisy, N, dist_dueling=True)
        with torch.device('meta'):
            net = AtariQNet(A, categorical=K > 0, num_atoms=K or 51, quantile=N > 0, num_quantiles=N or 200, noisy=noisy,
                            distributional_dueling=True)
        sd = [(n, tuple(t.shape)) for n, t in net.state_dict().items()]
        assert sd == state, A
        assert list(apex_param_shapes(A, False, K, noisy, N, dist_dueling=True).items()) == state, A
        assert total == total_want, A
        assert off == [off_want[n] for n, _ in state], A
        assert cnt == [torch.Size(s).numel() for _, s in state], A
        assert all(o % 4 == 0 for o in off)
        o = dict(zip([n for n, _ in state], off))
        for mu in (('',) if not noisy else ('_mu', '_sigma')):
            assert o[f'advantage.weight{mu}'] == o[f'value.weight{mu}'] + W * 512, A          # one [(W + A W)][512] block
            assert o[f'advantage.bias{mu}'] == o[f'value.bias{mu}'] + -(-W // 4) * 4, A       # the biases grouped
    # the kernels' head: the same layout from the Python binding of the learner's settings
    hp = ApexHParams(num_actions=6, categorical_dqn=K > 0, num_atoms=K or 51, quantile_dqn=N > 0, num_quantiles=N or 200,
                     noisy_dqn=noisy, distributional_dueling=True)
    assert hp.head.layout(6) == _lib.apex_param_layout(6, False, K, noisy, N, dist_dueling=True)


# ---------------------------------------------------------------------------------------------------------------- the reparametrisation
def _compose(wv, ba_v, wa, ba, A, W, mean_over='actions'):
    """W_eff, b_eff in fp64 as the device composes them: (v + adv) - mean_a adv"""
    adv = wa.view(A, W, -1)
    advb = ba.view(A, W)
    if mean_over == 'actions':
        m, mb = adv.mean(0, keepdim=True), advb.mean(0, keepdim=True)
    else:                                               # a plausible mistake: the mean over the atoms / quantiles
        m, mb = adv.mean(1, keepdim=True), advb.mean(1, keepdim=True)
    return ((wv[None] + adv) - m).reshape(A * W, -1), ((ba_v[None] + advb) - mb).reshape(A * W)


def _decompose(gW, gb, A, W, minus_mean=True):
    g = gW.view(A, W, -1)
    gbb = gb.view(A, W)
    gv, gbv = g.sum(0), gbb.sum(0)
    if minus_mean:
        return gv, gbv, (g - g.mean(0, keepdim=True)).reshape(A * W, -1), (gbb - gbb.mean(0, keepdim=True)).reshape(A * W)
    return gv, gbv, gW, gb                              # a plausible mistake: the -1/A term dropped


def _rel(a, b):
    """|a - b| / |b| (|b| at least 1: the advantage gradients of A = 1 are exactly 0)"""
    return float((a - b).norm()) / max(float(b.norm()), 1.0)


@pytest.mark.parametrize('A,W', [(1, 2), (6, 51), (18, 200), (31, 64)])
def test_reparametrisation_in_fp64(A, W):
    g = torch.Generator().manual_seed(A * 100 + W)
    n = 9
    h = torch.randn(n, 512, generator=g, dtype=F64).relu()
    wv = torch.randn(W, 512, generator=g, dtype=F64, requires_grad=True)
    bv = torch.randn(W, generator=g, dtype=F64, requires_grad=True)
    wa = torch.randn(A * W, 512, generator=g, dtype=F64, requires_grad=True)
    ba = torch.randn(A * W, generator=g, dtype=F64, requires_grad=True)
    v, adv = (h @ wv.T + bv).view(n, 1, W), (h @ wa.T + ba).view(n, A, W)
    rows = v + adv - adv.mean(1, keepdim=True)                      # the head as written
    We, be = _compose(wv.detach(), bv.detach(), wa.detach(), ba.detach(), A, W)
    composed = (h @ We.T + be).view(n, A, W)
    assert _rel(composed, rows.detach()) < 1e-13
    dl = torch.randn(n, A * W, generator=g, dtype=F64)
    (rows.reshape(n, A * W) * dl).sum().backward()
    gW, gb = dl.T @ h, dl.sum(0)                                   # the gradients of W_eff and b_eff
    gv, gbv, gwa, gba = _decompose(gW, gb, A, W)
    for got, want in ((gv, wv.grad), (gbv, bv.grad), (gwa, wa.grad), (gba, ba.grad)):
        assert _rel(got, want) < 1e-13
    if A > 1:     # each mistake moves the check far past its bound
        Wb, bb = _compose(wv.detach(), bv.detach(), wa.detach(), ba.detach(), A, W, mean_over='atoms')
        assert _rel((h @ Wb.T + bb).view(n, A, W), rows.detach()) > 1e-2
        _, _, gwa_bad, gba_bad = _decompose(gW, gb, A, W, minus_mean=False)
        assert _rel(gwa_bad, wa.grad) > 1e-2 and _rel(gba_bad, ba.grad) > 1e-2


# ---------------------------------------------------------------------------------------------------------------- the oracle
@pytest.mark.parametrize('noisy', [False, True])
@pytest.mark.parametrize('kind', ['categorical', 'quantile'])
def test_oracle_agrees_with_atari_qnet(kind, noisy):
    A, W = 4, 9
    torch.manual_seed(11)
    net = AtariQNet(A, categorical=kind == 'categorical', quantile=kind == 'quantile', num_atoms=W, num_quantiles=W, noisy=noisy,
                    distributional_dueling=True, v_min=-10.0, v_max=10.0)
    net.eval()                      # noisy: the mean weights, and the oracle's zero noise
    head = R.Head(kind, noisy, num_atoms=W, v_min=-10.0, v_max=10.0, num_quantiles=W)
    assert head.num_actions(net.state_dict()) == A
    ref = R.RefQNet(A, net.state_dict(), head)
    assert [n for n, _ in ref.named_parameters()] == list(net.state_dict())
    obs = torch.randint(0, 256, (3, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        rows = ref(obs)
        got = net.dist(obs) if kind == 'categorical' else net.quantiles(obs)
        want = torch.softmax(rows, dim=2) if kind == 'categorical' else rows
    torch.testing.assert_close(got, want, rtol=1e-6, atol=1e-6)
    # the noise vector's head segments: value's and advantage's in, then W value and A W advantage rows out
    noise = torch.arange(3648 + 2 * 512 + W + A * W, dtype=torch.float32)
    sp = R.split_noise(noise, A, W)
    assert sp['value'][1].numel() == W and sp['advantage'][1].numel() == A * W
    assert float(sp['advantage'][0][0]) == 3648 + 512 and float(sp['advantage'][1][0]) == 3648 + 1024 + W


def test_oracle_statements_run_on_the_dueling_rows():
    """within installed() apex_oracle's learn_step and initial_priorities run on the dueling rows, with the 12 gradients of value
    and advantage; outside it, and for apex_oracle's own heads, its network is unchanged"""
    from oracle import apex_oracle as O
    from tests.apex_cases import batch
    A, W = 3, 5
    sd, tg = (AtariQNet(A, quantile=True, num_quantiles=W, distributional_dueling=True).state_dict() for _ in range(2))
    (obs, act, rew, nobs, done), w = batch(4, A, seed=1)
    head = R.Head('quantile', num_quantiles=W)
    with R.installed():
        out = O.learn_step(sd, tg, obs, act, rew, nobs, done, weights=w, head=head)
        p = O.initial_priorities(sd, obs, act, rew, nobs, done, 0.99, 1e-6, head=head)
        assert type(O.RefQNet(A, head=O.Head('quantile', num_quantiles=W))).forward is R.RefQNet.forward
    assert list(out['grads']) == list(sd) and p.shape == (4,)
    net = AtariQNet(A, quantile=True, num_quantiles=W, distributional_dueling=True)
    net.load_state_dict(sd)
    T = O.targets(R.RefQNet(A, tg, head)(nobs), rew, done, 0.99)
    with torch.no_grad():
        torch.testing.assert_close(out['T'], T, rtol=0, atol=0)
        torch.testing.assert_close(out['theta'], net.quantiles(obs), rtol=1e-6, atol=1e-6)
    assert O.RefQNet is R._RefQNet


def test_new_kernels_do_not_spill():
    import os
    path = os.path.join(srl_build.HERE, 'build', 'ptxas.log')
    if not os.path.exists(path):
        srl_build.build(force=True)
    rep = srl_build.ptxas_report(path)['dueling_rows.cu']
    kernels = {k: v for k, v in rep.items() if 'dist_dueling' in k}
    assert len(kernels) == 2, sorted(rep)
    for k, v in kernels.items():
        assert v['spill_stores'] == 0 and v['spill_loads'] == 0, (k, v)
