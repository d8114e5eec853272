"""CPU: the R2D2 oracle's statements against an fp64 loop and against the Ape-X oracle, the learner's settings and parameter layout, and
the new kernels' ptxas report."""
import ctypes as C
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import apex_oracle as AO
from oracle import r2d2_oracle as O
from scalerl_b200 import _lib
from scalerl_b200 import build as srl_build
from scalerl_b200.algorithms.r2d2 import R2D2HParams, R2D2QNet, r2d2_param_shapes


def test_rescale_inverse_roundtrip():
    x = np.concatenate([np.linspace(-1e4, 1e4, 20001), np.geomspace(1e-6, 1e4, 500), -np.geomspace(1e-6, 1e4, 500), [0.0]])
    for eps in (1e-3, 1e-2):
        back = O.rescale_h_inv(O.rescale_h(x, eps), eps)
        np.testing.assert_allclose(back, x, rtol=1e-11, atol=1e-11)


def _tail_case(B, A, burn_in, T, n, seed, dones=()):
    g = torch.Generator().manual_seed(seed)
    L = burn_in + T + n
    q_on = torch.randn(T + n, B, A, generator=g) * 3
    q_tg = torch.randn(T, B, A, generator=g) * 3
    la = torch.randint(0, A, (L, B), generator=g)
    rw = torch.randn(L, B, generator=g)
    dn = torch.zeros(L, B, dtype=torch.bool)
    for r, b in dones:
        dn[r, b] = True
    return q_on, q_tg, la, rw, dn


@pytest.mark.parametrize('rescale', [True, False])
def test_oracle_tail_equals_fp64_loop(rescale):
    """dones at every position of the n-window of trained row 0, at row 0, at the burn-in boundary and on the last row"""
    B, A, burn_in, T, n = 7, 5, 3, 6, 4
    L = burn_in + T + n
    dones = [(burn_in + k, k - 1) for k in range(1, n + 1)] + [(0, 4), (burn_in, 5), (L - 1, 6), (burn_in + 2, 6)]
    q_on, q_tg, la, rw, dn = _tail_case(B, A, burn_in, T, n, 0, dones)
    q_taken, y = O.tail(q_on, q_tg, la, rw, dn, burn_in, n, 0.997, rescale)
    y64, d64, p64 = O.tail_fp64_loop(q_on.numpy(), q_tg.numpy(), la.numpy(), rw.numpy(), dn.numpy(), burn_in, n, 0.997, rescale,
                                     eta=0.9, priority_eps=1e-6)
    np.testing.assert_allclose(y.numpy(), y64, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose((q_taken - y).numpy(), d64, rtol=1e-6, atol=1e-6)
    ad = (q_taken - y).abs().double()
    prio = 0.9 * ad.max(0)[0] + 0.1 * ad.mean(0) + 1e-6
    np.testing.assert_allclose(prio.numpy(), p64, rtol=1e-6)
    # the window of sequence k - 1 (done at trained row 0's k-th step) bootstraps nothing: y = the k-step return
    for k in range(1, n + 1):
        b = k - 1
        G = sum(0.997 ** (j - 1) * float(rw[burn_in + j, b]) for j in range(1, k + 1))
        want = O.rescale_h(G, 1e-3) if rescale else G
        assert abs(float(y[0, b]) - want) <= 1e-5 * max(1.0, abs(want))


def test_single_step_reproduces_apex_double_dqn():
    """burn_in 0, T 1, n 1, no rescaling: the sequence step on a feed-forward Q network equals apex_oracle's double-DQN step on the
    same encoder rows (frame[0] = s, frame[1] = s', last_action[1] = a, reward[1] = r, done[1] = d)"""
    torch.manual_seed(0)
    B, A = 5, 4
    sd_on = OrderedDict((k, v.clone()) for k, v in AO.RefQNet(A).state_dict().items())
    sd_tg = OrderedDict((k, v + 0.01 * torch.randn_like(v)) for k, v in sd_on.items())
    frame = torch.randint(0, 256, (2, B, 4, 84, 84), dtype=torch.uint8)
    la = torch.randint(0, A, (2, B))
    rw = torch.randn(2, B)
    dn = torch.tensor([[False] * B, [False, True, False, False, True]])
    w = torch.rand(B) + 0.5
    ref = AO.learn_step(sd_on, sd_tg, frame[0], la[1], rw[1], frame[1], dn[1], weights=w, gamma=0.9, double_dqn=True, lr=1e-3)
    on, tg = AO.RefQNet(A, sd_on), AO.RefQNet(A, sd_tg)
    wrap = lambda m: (lambda fr, a, r, d, s: (m(fr.reshape(-1, 4, 84, 84)).view(fr.shape[0], B, A), s))
    params = OrderedDict(on.named_parameters())
    got = O.sequence_step(wrap(on), wrap(tg), params, dict(frame=frame, last_action=la, reward=rw, done=dn, state=()), 0, 1, 0.9,
                          rescale=False, eta=0.9, weights=w, lr=1e-3, adam_eps=1e-8)
    torch.testing.assert_close(got['q_taken'][0], ref['q'], rtol=0, atol=0)
    torch.testing.assert_close(got['y'][0], ref['y'], rtol=1e-6, atol=1e-6)
    assert abs(got['loss'] - ref['loss']) <= 1e-6 * abs(ref['loss'])
    torch.testing.assert_close(got['priorities'].float(), ref['priorities'], rtol=1e-6, atol=1e-6)
    for k in ref['grads']:
        torch.testing.assert_close(got['grads'][k], ref['grads'][k], rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(params[k].detach(), ref['params'][k], rtol=1e-5, atol=1e-7)


def test_ref_network_matches_r2d2qnet():
    """the oracle's network on the reference's AtariNet layers and the package's CPU R2D2QNet compute the same Q rows"""
    torch.manual_seed(1)
    for dueling in (False, True):
        net = R2D2QNet(3, dueling)
        ref = O.RefR2D2Net(3, net.state_dict(), dueling)
        T, B = 3, 2
        frame = torch.randint(0, 256, (T, B, 4, 84, 84), dtype=torch.uint8)
        la, rw = torch.randint(0, 3, (T, B)), torch.randn(T, B) * 2
        dn = torch.tensor([[False, True], [True, False], [False, False]])
        st = tuple(torch.randn(2, B, 516) for _ in range(2))
        q1, (h1, c1) = net(frame, la, rw, dn, st)
        q2, (h2, c2) = ref(frame, la, rw, dn, st)
        torch.testing.assert_close(q1, q2)
        torch.testing.assert_close(h1, h2)
        torch.testing.assert_close(c1, c2)


@pytest.mark.parametrize('bad', [dict(precision='fp32_split'), dict(categorical_dqn=True), dict(quantile_dqn=True), dict(noisy_dqn=True),
                                 dict(distributional_dueling=True), dict(num_actions=32), dict(num_actions=0), dict(burn_in=-1),
                                 dict(seq_len=0), dict(n_step=0), dict(batch_size=600), dict(gamma=1.5), dict(priority_eta=1.2),
                                 dict(rescale_eps=0.0), dict(max_grad_norm=0.0), dict(learning_rate=0.0), dict(adam_beta2=1.0),
                                 dict(target_update_frequency=0), dict(priority_eps=-1.0)])
def test_hparams_validation(bad):
    with pytest.raises(ValueError):
        R2D2HParams(**bad).validate()


def test_hparams_paper_defaults():
    hp = R2D2HParams()
    hp.validate()
    assert (hp.batch_size, hp.burn_in, hp.seq_len, hp.n_step, hp.gamma) == (64, 40, 80, 5, 0.997)
    assert (hp.learning_rate, hp.adam_eps, hp.priority_eta, hp.rescale_eps) == (1e-4, 1e-3, 0.9, 1e-3)
    assert hp.value_rescaling and hp.dueling and hp.max_grad_norm is None and hp.target_update_frequency == 2500
    c = hp.to_c()
    assert (c.B, c.A, c.burn_in, c.T, c.n_step, c.dueling, c.value_rescaling) == (64, 18, 40, 80, 5, 1, 1)


def test_config_struct_size():
    assert C.sizeof(_lib.SrlR2d2Config) == 16 * 4


@pytest.mark.parametrize('A,dueling', [(1, False), (6, True), (18, True), (31, False), (31, True)])
def test_layout_matches_r2d2qnet(A, dueling):
    total, off, cnt = _lib.r2d2_param_layout(A, dueling)
    sd = R2D2QNet(A, dueling).state_dict()
    shapes = r2d2_param_shapes(A, dueling)
    assert list(sd) == list(shapes)
    assert [tuple(v.shape) for v in sd.values()] == [tuple(s) for s in shapes.values()]
    assert cnt == [v.numel() for v in sd.values()]
    assert all(o % 4 == 0 for o in off) and off == sorted(off)
    assert all(off[i] + cnt[i] <= off[i + 1] for i in range(len(off) - 1)) and off[-1] + cnt[-1] <= total


def test_layout_refuses_bad_arguments():
    L = _lib.lib()
    o, c = (C.c_int64 * 20)(), (C.c_int64 * 20)()
    assert L.srl_r2d2_param_layout(32, 0, o, c) == -1 and b'[1,31]' in L.srl_last_error()
    assert L.srl_r2d2_param_layout(6, 2, o, c) == -1
    cfg = R2D2HParams(batch_size=4, num_actions=6, burn_in=2, seq_len=3, n_step=2).to_c()
    cfg.priority_eta = 2.0
    h = C.c_void_p()
    assert L.srl_r2d2_learner_create(C.addressof(cfg), None, None, None, None, None, C.byref(h)) == -1
    assert b'priority_eta' in L.srl_last_error()
    cfg.priority_eta, cfg.B = 0.9, 60000
    assert L.srl_r2d2_learner_create(C.addressof(cfg), None, None, None, None, None, C.byref(h)) == -1
    assert b'65536' in L.srl_last_error()


def test_r2d2_kernels_compile_without_spills():
    path = os.path.join(srl_build.HERE, 'build', 'ptxas.log')
    if not os.path.exists(path):
        srl_build.build(force=True)
    rep = srl_build.ptxas_report(path)['r2d2.cu']
    kernels = {k: v for k, v in rep.items() if 'r2d2_' in k}
    assert len(kernels) == 9, sorted(kernels)       # head fwd x2, tail, dcore x2, wgrad x2, reduce x2
    bad = {k: v for k, v in kernels.items() if v['spill_stores'] or v['spill_loads'] or v['serialized']}
    assert not bad, bad

