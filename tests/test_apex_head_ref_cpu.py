"""tests/apex_head_ref.py on the CPU: its fp64 references are oracle/apex_oracle.py's statements (and float64 autograd through the loss
statements) evaluated in fp64; an fp32 evaluation in the kernel's order passes the bound of every stage that has one here (the logits
GEMM, the head-gradient GEMM, dqn_wgrad's slab / group order, q_dot and the dueling Q, both dcores, tail_loss, the C51 projection, CE,
KL and dlogits, the QR target quantiles and quantile loss, the distributional-dueling compose and split), and those bounds sit far
below the values they bound; every mistake moves its witness and the two neutral ones stay inside the bound.  Every input is seeded."""
import numpy as np
import pytest
import torch

from oracle import apex_oracle as O
from tests import apex_head_ref as R

F64 = torch.float64


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _scalar_case(kind, B, A, seed=0):
    g = _g(seed)
    h = torch.rand(B, 512, generator=g, dtype=F64)
    R_ = A + 1 if kind == 'dueling' else A
    net = lambda: {'W': torch.randn(R_, 512, generator=g, dtype=F64) * 0.05, 'b': torch.randn(1 if kind == 'dueling' else A, generator=g, dtype=F64),
                   'ba': torch.randn(A, generator=g, dtype=F64)}
    return h, torch.rand(B, 512, generator=g, dtype=F64), net(), net(), torch.randint(0, A, (B,), generator=g), \
        torch.randn(B, generator=g, dtype=F64), torch.rand(B, generator=g) < 0.3, torch.rand(B, generator=g, dtype=F64) + 0.1


@pytest.mark.parametrize('kind', ['plain', 'dueling'])
def test_scalar_tail_is_autograd_of_the_loss(kind):
    B, A, gamma = 37, 6, 0.97
    h, hn, on, tg, act, rew, done, w = _scalar_case(kind, B, A)
    Q, _ = R.scalar_q(kind, h, on)
    if kind == 'dueling':
        adv = h @ on['W'][1:].T + on['ba']
        want = (h @ on['W'][:1].T + on['b']) + adv - adv.mean(1, keepdim=True)
    else:
        want = h @ on['W'].T + on['b']
    assert torch.allclose(Q, want, rtol=1e-12, atol=1e-12)
    nx, _, _, _, _, a1 = R.scalar_targets(kind, None, hn, on, tg, False)
    assert torch.equal(a1, R.scalar_q(kind, hn, tg)[0].argmax(1))
    y, _ = R.td_target(rew, done, gamma, nx, torch.zeros(B, dtype=F64))
    q = R.take(Q, act)
    fq = R.from_qy(q, y, w, B, 0.0)
    # float64 autograd through the reference's loss statement (worker.py:156-157) -> dq, dcore, the head gradients
    hh = h.clone().requires_grad_(True)
    Wt = on['W'].clone().requires_grad_(True)
    bt, bat = on['b'].clone().requires_grad_(True), on['ba'].clone().requires_grad_(True)
    if kind == 'dueling':
        adv = hh @ Wt[1:].T + bat
        Qg = (hh @ Wt[:1].T + bt) + adv - adv.mean(1, keepdim=True)
    else:
        Qg = hh @ Wt.T + bt
    loss = (w * (Qg.gather(1, act[:, None])[:, 0] - y) ** 2).mean()
    loss.backward()
    assert abs(float(R.loss_ref(fq['l'], B)[0]) - float(loss.detach())) <= 1e-12 * float(loss.detach())
    dc, _ = R.scalar_dcore(kind, fq['dq'], act, on)
    assert torch.allclose(dc, hh.grad, rtol=1e-10, atol=1e-14)
    gW, _ = R.scalar_wgrad(kind, fq['dq'], act, h, A, B)
    want = torch.cat([Wt.grad, (bt.grad if kind == 'plain' else torch.cat([bt.grad, bat.grad]))[:, None]], 1)
    # the dueling head's 1 / A is the kernel's fp32 fl(1 / A)
    assert float((gW - want).abs().max()) <= (1e-7 if kind == 'dueling' else 1e-12) * float(want.abs().max())


@pytest.mark.parametrize('K,support', [(2, (-1.0, 1.0)), (51, (-10.0, 10.0)), (64, (-3.0, 7.0))])
def test_projection_and_c51_tail_are_the_oracles(K, support):
    B, A = 29, 3
    g = _g(K)
    x = torch.randn(B, A, K, generator=g, dtype=F64)
    rew = torch.randn(B, generator=g, dtype=F64) * 4
    done = torch.rand(B, generator=g) < 0.3
    gamma = 0.97
    z32, dz32 = O.support(K, *support)
    lo, hi = float(np.float32(support[0])), float(np.float32(support[1]))
    Q, _ = R.cat_q(x, z32)
    a = Q.argmax(1)
    p = torch.softmax(x, 2)[torch.arange(B), a]
    m, _ = R.project(p, p, rew, float(np.float32(gamma)) * (1 - done.to(F64)), z32, float(dz32), lo, hi)
    want = O.project_fp64_loop(p.numpy(), rew.numpy(), done.numpy(), float(np.float32(gamma)), lo, hi)
    # project_fp64_loop builds dz and the support in fp64; the reference takes the kernel's fp32 support
    assert np.abs(m.numpy() - want).max() <= 1e-5
    xs = x[:, 0]
    t = R.cat_tail(xs, m, z32, None, B)
    lp = torch.log_softmax(xs, 1)
    assert torch.allclose(t['ce'][0], -(m * lp).sum(1), rtol=1e-12)
    assert torch.allclose(t['kl'][0], O.kl(m, lp), rtol=1e-10, atol=1e-14)
    xg = xs.clone().requires_grad_(True)
    (-(m * torch.log_softmax(xg, 1)).sum(1)).mean().backward()
    assert torch.allclose(t['dl'][0], xg.grad, rtol=1e-10, atol=1e-15)


@pytest.mark.parametrize('N,kappa', [(2, 1.0), (33, 0.5), (256, 0.02)])
def test_qr_tail_is_the_oracles(N, kappa):
    B, A = 11, 3
    g = _g(N)
    th = torch.randn(B, A, N, generator=g, dtype=F64)
    tn = torch.randn(B, A, N, generator=g, dtype=F64)
    rew = torch.randn(B, generator=g, dtype=F64)
    done = torch.rand(B, generator=g) < 0.3
    w = torch.rand(B, generator=g, dtype=F64) + 0.1
    gamma = 0.97
    a = R.qr_q(tn)[0].argmax(1)
    T, _ = R.qr_targets(tn, a, rew, float(np.float32(gamma)) * (1 - done.to(F64)))
    assert torch.allclose(T, O.targets(tn, rew, done, gamma), rtol=1e-14)
    ta = th[:, 1]
    ln, _, d, _ = R.qr_loss(ta, T, kappa, w, B)
    assert torch.allclose(ln, O.quantile_loss(ta, T, kappa), rtol=1e-12)
    assert torch.allclose(d, O.dtheta_written(ta, T, kappa, w), rtol=1e-12, atol=1e-16)
    tg_ = ta.clone().requires_grad_(True)
    (w * O.quantile_loss(tg_, T, kappa)).mean().backward()
    assert torch.allclose(d, tg_.grad, rtol=1e-10, atol=1e-16)


def test_dist_dueling_compose_and_grad():
    A, V = 4, 7
    g = _g(3)
    wv, bv = torch.randn(V, 512, generator=g, dtype=F64), torch.randn(V, generator=g, dtype=F64)
    wa, ba = torch.randn(A * V, 512, generator=g, dtype=F64), torch.randn(A * V, generator=g, dtype=F64)
    W, b, _, _ = R.dd_compose(wv, bv, wa, ba, A)
    adv = wa.view(A, V, 512)
    assert torch.allclose(W.view(A, V, 512), wv[None] + adv - adv.mean(0, keepdim=True), rtol=1e-12)
    # the split is the chain rule through the composition: autograd of sum(G * rows) w.r.t. value and advantage
    G = torch.randn(A * V, 513, generator=g, dtype=F64)
    wvg, wag = wv.clone().requires_grad_(True), wa.clone().requires_grad_(True)
    a3 = wag.view(A, V, 512)
    rows = (wvg[None] + a3 - a3.mean(0, keepdim=True)).reshape(A * V, 512)
    (rows * G[:, :512]).sum().backward()
    gv, _, ga, _ = R.dd_grad(G[:, :512], G[:, 512], A, V)
    assert torch.allclose(gv[:, :512], wvg.grad, rtol=1e-12) and torch.allclose(ga[:, :512], wag.grad, rtol=1e-10, atol=1e-13)


def _fp32_gemm(h, W, b):
    """cat_gemm_kernel<false>'s order in fp32: one fma-free chain over j ascending from 0, then + b"""
    h32, W32 = h.float(), W.float()
    acc = torch.zeros(h.shape[0], W.shape[0])
    for j in range(512):
        acc = acc + h32[:, j:j + 1] * W32[:, j][None]
    return acc + b.float()


def test_fp32_evaluations_pass_the_bounds():
    """an fp32 CPU evaluation in each kernel's order is within every bound, and the bounds are far below the values they bound"""
    B, A, K = 70, 3, 11
    g = _g(9)
    h = torch.rand(B, 512, generator=g).double()
    W = (torch.randn(A * K, 512, generator=g) * 0.05).double()
    b = torch.randn(A * K, generator=g).double()
    x, S = R.gemm_rows(h, W, b)
    x32 = _fp32_gemm(h, W, b)
    assert R.ratio(x32, x, S, R.CHECK_C['logits']) <= 1.0
    assert float((R.CHECK_C['logits'] * R.U * S / x.abs().clamp(min=1e-3)).median()) < 0.1
    # the head gradient: one B-long chain in fp32
    dl = (torch.randn(B, A * K, generator=g) * 1e-3).double()
    gW, Sg = R.cat_wgrad(dl, h, B)
    hb = torch.cat([h, torch.ones(B, 1, dtype=F64)], 1).float()
    acc = torch.zeros(A * K, 513)
    for n in range(B):
        acc = acc + dl[n].float()[:, None] * hb[n][None]
    assert R.ratio(acc, gW, Sg, R.CHECK_C['head_grad']) <= 1.0
    # q_dot (16-term lane chains and the butterfly) in fp32, plain and dueling, and the dueling dcore
    for kind in ('plain', 'dueling'):
        hs, _, on, _, act, _, _, _ = _scalar_case(kind, 40, 6, 4)
        Q, SQ = R.scalar_q(kind, hs, on)
        lanes = (hs.float().view(40, 1, 16, 32) * on['W'].float().view(1, -1, 16, 32)).sum(2)      # [B, R, 32] lane partials
        dots = lanes.sum(2)
        if kind == 'plain':
            Q32 = dots + on['b'].float()
        else:
            adv = dots[:, 1:] + on['ba'].float()
            Q32 = (dots[:, :1] + on['b'].float() + adv) - adv.sum(1, keepdim=True) / 6
        assert R.ratio(Q32, Q, SQ, R.CHECK_C['q']) <= 1.0
    # the quantile Huber loss in fp32
    ta, T = torch.randn(9, 33, generator=g).double(), torch.randn(9, 33, generator=g).double()
    ln, Sln, d, Sd = R.qr_loss(ta, T, 0.5, None, 9)
    u = T.float()[:, None, :] - ta.float()[:, :, None]
    tau = ((2 * torch.arange(33) + 1) / torch.tensor(66.0))[None, :, None]
    wt = (tau - (u < 0).float()).abs()
    L = torch.where(u.abs() <= 0.5, 0.5 * (u * u), 0.5 * (u.abs() - 0.25))
    ln32 = (wt * L).sum(2).sum(1) / 0.5 / 33
    assert R.ratio(ln32, ln, Sln, R.CHECK_C['qr_loss']) <= 1.0


def _moves(m, got, ref, S, c):
    return R.sensitivity(got, ref, S, c) >= R.SENS


def test_mistakes_move_their_witnesses():
    """each mistake moves the reference of a small case of the kind its GPU witness runs by >= 20x the bound"""
    torch.manual_seed(17)
    B, A = 37, 6
    for kind in ('plain', 'dueling'):
        h, hn, on, tg, act, rew, done, w = _scalar_case(kind, B, A, 2)
        dq = torch.randn(B, dtype=F64) * 1e-2
        g0, S = R.scalar_wgrad(kind, dq, act, h, A, B)
        for m in ('wgrad_last_group', 'bias_dropped') + (('dueling_mean_A_minus_1',) if kind == 'dueling' else ()):
            assert _moves(m, R.scalar_wgrad(kind, dq, act, h, A, B, m)[0], g0, S, R.CHECK_C['head_grad']), (kind, m)
        nx, Sn, *_ = R.scalar_targets(kind, hn, hn * 0.5, on, tg, True)
        nxm = R.scalar_targets(kind, hn, hn * 0.5, on, tg, True, 'double_target_astar')[0]
        assert _moves('double_target_astar', nxm, nx, Sn, R.CHECK_C['y'])
    h, _, on, _, act, _, _, _ = _scalar_case('dueling', B, A, 3)
    dq = torch.randn(B, dtype=F64)
    d0, S = R.scalar_dcore('dueling', dq, act, on)
    for m in ('dueling_mean_A_minus_1', 'dueling_dcore_no_mean'):
        assert _moves(m, R.scalar_dcore('dueling', dq, act, on, m)[0], d0, S, R.CHECK_C['dcore_scalar'])
    l = torch.rand(5, dtype=F64)
    l0, Sl = R.loss_ref(l, 5)
    assert _moves('loss_last_block', R.loss_ref(l, 5, 'loss_last_block')[0], l0, Sl, R.CHECK_C['loss'])
    dl = torch.randn(33, 20, dtype=F64)
    hh = torch.rand(33, 512, dtype=F64)
    g0, S = R.cat_wgrad(dl, hh, 33)
    assert _moves('wgrad_last_kstage', R.cat_wgrad(dl, hh, 33, 'wgrad_last_kstage')[0], g0, S, R.CHECK_C['head_grad'])
    Wg, bg = torch.randn(20, 512, dtype=F64), torch.zeros(20, dtype=F64)
    x, S = R.gemm_rows(hh, Wg, bg)
    xm = R.gemm_rows(hh, Wg, bg, 'gemm_row0_unstored')[0]
    assert torch.equal(xm[1:64], x[1:64]) and R.sensitivity(xm, x, S, 1) == float('inf')
    Q = torch.randn(9, 3, dtype=F64)
    assert R.sensitivity(R.q_values_mistake(Q, 'q_values_last_lane'), Q, Q.abs(), 2) == float('inf')
    # the projection: rewards on the support's atoms with g = 0 take the l == u branch
    K = 11
    z32, dz32 = O.support(K, -10.0, 10.0)
    p = torch.softmax(torch.randn(6, K, dtype=F64), 1)
    rew = torch.tensor([-15.0, 15.0, float(z32[0]), float(z32[-1]), float(z32[3]), 0.3], dtype=F64)
    g = torch.zeros(6, dtype=F64)
    m0, Sm = R.project(p, p, rew, g, z32, float(dz32), -10.0, 10.0)
    assert _moves('project_split_l_eq_u', R.project(p, p, rew, g, z32, float(dz32), -10.0, 10.0, 'project_split_l_eq_u')[0], m0, Sm,
                  R.CHECK_C['m'])
    ta, T = torch.randn(4, 32, dtype=F64), torch.randn(4, 32, dtype=F64)
    l0, S0, _, _ = R.qr_loss(ta, T, 1.0, None, 4)
    assert _moves('tau_i_over_N', R.qr_loss(ta, T, 1.0, None, 4, 'tau_i_over_N')[0], l0, S0, R.CHECK_C['qr_loss'])
    G = torch.randn(4 * 7, 513, dtype=F64)
    gv, Sv, ga, Sa = R.dd_grad(G[:, :512], G[:, 512], 4, 7)
    for m in ('dd_grad_mean_axis', 'dd_grad_A_minus_1'):
        assert _moves(m, R.dd_grad(G[:, :512], G[:, 512], 4, 7, m)[2], ga, Sa, R.CHECK_C['rows'])


def test_neutral_mistakes_stay_within_the_bound():
    """|u| < kappa changes no loss (both branches give kappa^2 / 2 at |u| = kappa), and an unclamped u only moves mass by b's rounding"""
    torch.manual_seed(18)
    ta = torch.tensor([[0.0, 0.5, -0.5]], dtype=F64)
    T = torch.tensor([[0.5, 1.0, 0.0]], dtype=F64)                # |u| = kappa = 0.5 on several pairs
    l0, S0, d0, Sd = R.qr_loss(ta, T, 0.5, None, 1)
    l1, _, d1, _ = R.qr_loss(ta, T, 0.5, None, 1, 'kappa_strict')
    assert R.sensitivity(l1, l0, S0, 2) < 1.0 and R.sensitivity(d1, d0, Sd, 2) < 1.0
    K = 64
    z32, dz32 = O.support(K, -10.0, 10.0)
    p = torch.softmax(torch.randn(3, K, dtype=F64), 1)
    rew = torch.tensor([10.0, 30.0, 9.9], dtype=F64)
    g = torch.zeros(3, dtype=F64)
    m0, Sm = R.project(p, p, rew, g, z32, float(dz32), -10.0, 10.0)
    m1 = R.project(p, p, rew, g, z32, float(dz32), -10.0, 10.0, 'project_u_unclamped')[0]
    assert R.sensitivity(m1, m0, Sm, R.CHECK_C['m']) < 1.0
    assert set(R.NEUTRAL) <= set(R.MISTAKES)


@pytest.mark.parametrize('K,support', [(2, (-1.0, 1.0)), (11, (-10.0, 10.0)), (41, (-5.0, 5.0))])
def test_projection_is_the_fp64_loop_on_exact_supports(K, support):
    """on supports whose dz and atoms are exact in fp32 the projection is project_fp64_loop to 1e-12, rewards on atoms included"""
    B = 40
    g = _g(K + 1)
    p = torch.softmax(torch.randn(B, K, generator=g, dtype=F64), 1)
    z32, dz32 = O.support(K, *support)
    rew = torch.cat([torch.randn(B - 8, generator=g, dtype=F64) * 4, z32[[0, -1, K // 2, 1]].double(),
                     torch.tensor([support[0] - 3, support[1] + 3, 0.25, -0.5], dtype=F64)])
    done = torch.rand(B, generator=g) < 0.4
    gamma = 0.5
    m, _ = R.project(p, p, rew, gamma * (1 - done.to(F64)), z32, float(dz32), *support)
    want = O.project_fp64_loop(p.numpy(), rew.numpy(), done.numpy(), gamma, *support)
    assert np.abs(m.numpy() - want).max() <= 1e-12


def _f(x):
    return torch.as_tensor(x).float()


def _near(bound, value):
    """the median of bound / |value| over the elements not near 0"""
    v = value.abs()
    keep = v > 1e-3 * float(v.max())
    return float((bound[keep] / v[keep]).median())


def test_fp32_tails_pass_the_bounds():
    """fp32 evaluations in the kernels' orders: dqn_wgrad's slabs and groups, both dcores, tail_loss, the projection and the C51 tail,
    the QR target quantiles, the distributional-dueling compose and split; each within its bound, each bound far below its value"""
    g = _g(23)
    U2 = lambda c, S: c * R.U * S
    # dqn_wgrad + reduce at B = 1000: 32 groups of 2 slabs (fmaf chains in slab order), then the groups added in order
    B, A = 1000, 6
    h = torch.rand(B, 512, generator=g, dtype=F64)
    act = torch.randint(0, A, (B,), generator=g)
    dq = torch.randn(B, generator=g, dtype=F64) * 1e-3
    for kind in ('plain', 'dueling'):
        gW, S = R.scalar_wgrad(kind, dq, act, h, A, B)
        hb = torch.cat([_f(h), torch.ones(B, 1)], 1)
        oh = torch.nn.functional.one_hot(act, A).float()
        coef = oh * _f(dq)[:, None] if kind == 'plain' else torch.cat([_f(dq)[:, None], _f(dq)[:, None] * (oh - _f(1.0 / A))], 1)
        spg, groups = R.wgrad_groups(B)
        part = []
        for gi in range(groups):
            acc = torch.zeros(coef.shape[1], 513)
            for n in range(gi * spg * 16, min(B, (gi + 1) * spg * 16)):
                acc = acc + coef[n][:, None] * hb[n][None]
            part.append(acc)
        tot = torch.zeros_like(part[0])
        for q in part:
            tot = tot + q
        assert R.ratio(tot, gW, S, R.CHECK_C['head_grad']) <= 1.0, kind
        assert _near(U2(R.CHECK_C['head_grad'], S), gW) < 1e-3
    # dcore of both scalar heads and tail_loss, on fp32 q, y
    for kind in ('plain', 'dueling'):
        _, _, on, _, act, _, _, w = _scalar_case(kind, 333, 6, 5)
        q, y = torch.randn(333, generator=g).double(), torch.randn(333, generator=g).double()
        fq = R.from_qy(q, y, w, 333, 0.0)
        dc, Sdc = R.scalar_dcore(kind, fq['dq'], act, on)
        d32 = _f(2.0 / 333) * _f(w) * (_f(q) - _f(y))
        W = _f(on['W'])
        col = W[act] if kind == 'plain' else (W[0] + W[1:][act]) - W[1:].sum(0) / 6
        assert R.ratio(d32[:, None] * col, dc, Sdc, R.CHECK_C['dcore_scalar']) <= 1.0, kind
        assert _near(U2(R.CHECK_C['dcore_scalar'], Sdc), dc) < 1e-5
        lo, Sl = R.loss_ref(fq['l'], 333)
        l32 = _f(w) * ((_f(q) - _f(y)) * (_f(q) - _f(y)))
        parts = torch.stack([(l32[i:i + 4].sum()) for i in range(0, 333, 4)])
        assert R.ratio(parts.sum() / 333, lo, Sl, R.CHECK_C['loss']) <= 1.0
    # the projection and the C51 tail in fp32 (atom order; expf, the division and the splits rounded one by one)
    K, Bc = 51, 64
    z32, dz32 = O.support(K, -10.0, 10.0)
    xt = torch.randn(Bc, K, generator=g)
    xs = torch.randn(Bc, K, generator=g)
    rew = torch.randn(Bc, generator=g) * 3
    gm = torch.where(torch.rand(Bc, generator=g) < 0.3, torch.tensor(0.0), _f(0.97))
    p32 = torch.softmax(xt, 1)
    b = (torch.clamp(rew[:, None] + gm[:, None] * z32[None], -10.0, 10.0) - _f(-10.0)) / dz32
    lo_i, up = b.floor().long().clamp(0, K - 1), b.ceil().long().clamp(0, K - 1)
    m32 = torch.zeros(Bc, K + 0)
    for j in range(K):
        eq = lo_i[:, j] == up[:, j]
        m32.scatter_add_(1, lo_i[:, j:j + 1], torch.where(eq, p32[:, j], p32[:, j] * (up[:, j].float() - b[:, j]))[:, None])
        m32.scatter_add_(1, up[:, j:j + 1], torch.where(eq, torch.zeros(Bc), p32[:, j] * (b[:, j] - lo_i[:, j].float()))[:, None])
    p64, _, Sp, _ = R.softmax_rows(xt.double())
    m, Sm = R.project(p64, Sp, rew.double(), gm.double(), z32, float(dz32), -10.0, 10.0)
    assert R.ratio(m32, m, Sm, R.CHECK_C['m']) <= 1.0
    t = R.cat_tail(xs.double(), m32.double(), z32, None, Bc)
    lp32 = torch.log_softmax(xs, 1)
    ce32 = -(m32 * lp32).sum(1)
    assert R.ratio(ce32, *t['ce'], R.CHECK_C['ce']) <= 1.0
    lm = torch.where(m32 > 0, m32.clamp(min=1e-30).log(), torch.zeros_like(m32))
    assert R.ratio((torch.where(m32 > 0, m32 * (lm - lp32), torch.zeros_like(m32))).sum(1), *t['kl'], R.CHECK_C['kl']) <= 1.0
    dl32 = _f(1.0 / Bc) * (torch.softmax(xs, 1) * m32.sum(1, keepdim=True) - m32)
    assert R.ratio(dl32, *t['dl'], R.CHECK_C['dlogits']) <= 1.0
    assert _near(U2(R.CHECK_C['m'], Sm), m) < 1e-3 and _near(U2(R.CHECK_C['dlogits'], t['dl'][1]), t['dl'][0]) < 1e-4
    # the QR target quantiles
    tn = torch.randn(Bc, 3, 17, generator=g)
    a = R.qr_q(tn.double())[0].argmax(1)
    T, ST = R.qr_targets(tn.double(), a, rew.double(), gm.double())
    T32 = rew[:, None] + gm[:, None] * tn[torch.arange(Bc), a]
    assert R.ratio(T32, T, ST, R.CHECK_C['target_quantiles']) <= 1.0
    # the distributional-dueling compose and split
    Ad, V = 7, 9
    wv, bv = torch.randn(V, 512, generator=g), torch.randn(V, generator=g)
    wa, ba = torch.randn(Ad * V, 512, generator=g), torch.randn(Ad * V, generator=g)
    W, bb, SW, Sb = R.dd_compose(wv.double(), bv.double(), wa.double(), ba.double(), Ad)
    a3 = wa.view(Ad, V, 512)
    acc = torch.zeros(V, 512)
    for i in range(Ad):
        acc = acc + a3[i]
    W32 = ((wv[None] + a3) - acc[None] / Ad).reshape(Ad * V, 512)
    assert R.ratio(W32, W, SW, R.CHECK_C['rows']) <= 1.0 and _near(U2(2, SW), W) < 1e-5
    G = torch.randn(Ad * V, 513, generator=g)
    gv, Sv, ga, Sa = R.dd_grad(G[:, :512].double(), G[:, 512].double(), Ad, V)
    G3 = G.view(Ad, V, 513)
    acc = torch.zeros(V, 513)
    for i in range(Ad):
        acc = acc + G3[i]
    assert R.ratio(acc, gv, Sv, R.CHECK_C['rows_sum']) <= 1.0
    assert R.ratio((G3 - acc[None] / Ad).reshape(Ad * V, 513), ga, Sa, R.CHECK_C['rows']) <= 1.0
