"""fp64 references of the Ape-X Q-head kernels (csrc/dqn.cu, dqn_cat.cu / .cuh, dqn_qr.cu / .cuh, dueling_rows.cu, apex_actor.cu), on
whichever operands the caller passes, with the per-element rounding bound of each output and the kernel mistakes a check has to see.

torch float64 on any device, vectorised over the batch.  The GPU check (tests/test_gpu_apex_head_exact.py) runs each stage on the
operands the GPU itself read, so every bound stays local: the scalar heads on the kernel's core rows (priority, dcore, loss and the
head gradients on the kernel's own q and y), the logits / quantile GEMM on the core rows, the C51 / QR tail on the kernel's logits
(ce, KL, y and dlogits on its own m; qr_loss and dtheta on its own target quantiles), dcore and the head gradients on its own
dlogits / dtheta, the distributional-dueling split on its own composed-row gradient.  tests/test_apex_head_ref_cpu.py proves the
references against oracle/apex_oracle.py, shows a CPU fp32 evaluation in each kernel's order passes every bound, and that every
mistake below moves its witness case.

Bounds.  Every bound is per element, CHECK_C[check] * U * S (+ ETA): U = 2^-24, S in units of U.  For a plain sum S = n_chain *
sum|terms|, n_chain the longest chain of roundings in the kernel's order, and c = 1.01 (gamma_n = n U / (1 - n U) <= 1.01 n U for
n U <= 0.01; Higham, Accuracy and Stability, eq. 4.4).  For a composite quantity S is the first-order propagation of every rounding
(each written next to it) and c = 2 covers the second-order terms.  The chains:
  q_dot            16 fmaf per lane + a 5-step butterfly + the bias add = 22
  dqn_wgrad        spg * 16 fmaf in one group (spg slabs of 16 transitions) + `groups` adds in the reduce
  cat_gemm<false>  512 fmaf + the bias add = 513
  cat_gemm<true>   B fmaf, one chain over every transition (ascending n)
  cat_transition   K adds of the softmax sum, K fmaf of q / y / ce / KL, K adds of sum m
  qr_transition    N adds per S_i / G_i, then <= 8 lane adds (QR_PER_LANE) + 5 butterfly + / kappa + / N
  tail_loss        w * loss (+ the square), 2 block levels, ceil(blocks / 32) lane-strided adds, 5 butterfly, / B
  dueling mean     A adds + one division (dueling_q, dist_dueling_*)
expf is within 2 ulp and logf within 1 ulp (CUDA C Programming Guide, Mathematical Functions); the project builds without fast-math.

Discrete choices.  a* is an argmax.  pick() returns the fp64 first argmax, the runner-up and the rows whose two lie within their
bounds (the tie set): the caller accepts such a row under either action and counts it (<= MAX_TIE_FRAC).  Exact fp64 ties (equal
rows, tests/apex_cases.py's _tie_*) are not in the tie set: they resolve to the first index, as in the kernels.
"""
import functools
import math

import torch

from tests import exact as E
from tests.exact import U

F64 = torch.float64
ETA = 2.0 ** -126
SENS = 20.0
MAX_TIE_FRAC = 1e-3
HEAD_GROUPS, DQN_SLAB, CG_BK, CG_BM = 32, 16, 16, 64
QR_PER_LANE = 8

CHECK_C = {
    # plain sums (S = n_chain * sum|terms|)
    'logits': 1.01, 'theta': 1.01, 'head_grad': 1.01, 'dcore': 1.01, 'loss': 1.01, 'rows_sum': 1.01,
    # composites (S = the first-order propagation); 2x for second order
    'q': 2, 'y': 2, 'priority': 2, 'dcore_scalar': 2, 'm': 2, 'target_quantiles': 2, 'ce': 2, 'kl': 2, 'qr_loss': 2, 'dlogits': 2,
    'rows': 2,
}

MISTAKES = {
    'wgrad_last_group': 'dqn_wgrad_reduce_kernel sums groups - 1 partials (the last group of slabs dropped)',
    'wgrad_last_kstage': 'cat_gemm_kernel<true> loops k0 + CG_BK < Kdim (the last k-stage, n >= 16 floor((B - 1) / 16), dropped)',
    'bias_dropped': 'the bias column j = 512 of the head gradient left at 0',
    'gemm_row0_unstored': 'cat_gemm_kernel<false> does not store rows m = 0 (mod 64)',
    'dueling_mean_A_minus_1': 'the dueling mean divided by A - 1',
    'dueling_dcore_no_mean': 'the -mean term left out of the dueling dcore',
    'double_target_astar': 'a* taken from the target network under double DQN',
    'project_u_unclamped': 'cat_project with u = ceil(b) not clamped at K - 1',
    'project_split_l_eq_u': "cat_project's l == u branch splitting the mass (p (u - b) + p (b - l) = 0)",
    'tau_i_over_N': 'tau_i = i / N in place of (2 i + 1) / (2 N)',
    'kappa_strict': '|u| < kappa in place of |u| <= kappa',
    'loss_last_block': "tail_loss drops the last block's partial",
    'q_values_last_lane': 'q_values_kernel stores only lanes < A - 1 (the last action\'s column keeps what the output held: NaN here)',
    'dd_grad_mean_axis': 'the distributional-dueling gradient takes its mean over the atoms k instead of the actions a',
    'dd_grad_A_minus_1': 'dist_dueling_grad_kernel divides by A - 1',
}
# mistakes that change no value a kernel computes: both Huber branches give kappa^2 / 2 at |u| = kappa (and the same clamp), and b <= K - 1
# after the clamp of Tz to v_max, so u = ceil(b) exceeds K - 1 only by a rounding of b (moving mass p (b - (K - 1)), below the bound).
# The CPU test asserts they stay within the bound on every case rather than claiming a witness.
NEUTRAL = ('kappa_strict', 'project_u_unclamped')


def t64(x, device=None):
    x = torch.as_tensor(x)
    return x.to(device or x.device, F64)


# max |got - ref| / (c (U S + ETA)) on the tensors' device, and how far a mistake moves the reference in those units; an output NaN
# on both sides agrees
ratio = functools.partial(E.ratio, eta=ETA, nan_equal=True)
sensitivity = functools.partial(E.sensitivity, eta=ETA, nan_equal=True)


def n_loss(B):
    """tail_loss's chain after the per-transition product: 2 block levels + ceil(blocks / 32) + 5 + the division"""
    return 2 + -(-((B + 3) // 4) // 32) + 5 + 1


def wgrad_groups(B):
    """launch_q_wgrad's split: (slabs per group, groups)"""
    nslab = -(-B // DQN_SLAB)
    spg = -(-nslab // HEAD_GROUPS)
    return spg, -(-nslab // spg)


# ------------------------------------------------------------------------------------------------ argmax
def pick(Q, S, c=CHECK_C['q']):
    """-> (first argmax, runner-up, tie rows): a row ties when 0 < Q[a1] - Q[a2] <= the two bounds"""
    A = Q.shape[1]
    a1 = Q.argmax(1)
    if A == 1:
        return a1, a1, torch.zeros_like(a1, dtype=torch.bool)
    Qm = Q.clone()
    Qm.scatter_(1, a1[:, None], -math.inf)
    a2 = Qm.argmax(1)
    q1, q2 = Q.gather(1, a1[:, None])[:, 0], Q.gather(1, a2[:, None])[:, 0]
    s1, s2 = S.gather(1, a1[:, None])[:, 0], S.gather(1, a2[:, None])[:, 0]
    gap = q1 - q2
    return a1, a2, (gap > 0) & (gap <= c * U * (s1 + s2))


def q_values_mistake(Q, mistake):
    """q_values_kernel's output under a mistake: 'q_values_last_lane' leaves column A - 1 as the NaN the caller filled it with"""
    Q = Q.clone()
    if mistake == 'q_values_last_lane':
        Q[:, -1] = math.nan
    return Q


def take(x, a):
    return x.gather(1, a[:, None])[:, 0]


# ------------------------------------------------------------------------------------------------ the scalar heads
def lin(h, W, b):
    """h W^T + b and sum|terms|"""
    h, W, b = t64(h), t64(W).to(h.device), t64(b).to(h.device)
    return h @ W.T + b, h.abs() @ W.abs().T + b.abs()


def scalar_q(kind, h, net, mistake=None):
    """Q [B, A] of the plain (net = {W [A][512], b}) or dueling head (net = {W [(A + 1)][512] value row first, b [1], ba [A]}) ->
    (Q, S): q_dot's 22 roundings per dot product; dueling: + A adds and the division of the mean, then + and - (3 roundings)"""
    if kind == 'plain':
        Q, S = lin(h, net['W'], net['b'])
        return Q, 22 * S
    W = t64(net['W']).to(h.device)
    V, SV = lin(h, W[:1], net['b'])
    adv, Sa = lin(h, W[1:], net['ba'])
    A = adv.shape[1]
    mean = adv.sum(1, keepdim=True) / (A - 1 if mistake == 'dueling_mean_A_minus_1' else A)
    Q = (V + adv) - mean
    S = 22 * (SV + Sa + Sa.mean(1, keepdim=True)) + (A + 1) * adv.abs().mean(1, keepdim=True) + (V + adv).abs() + Q.abs() + mean.abs()
    return Q, S


def scalar_targets(kind, hn, hnt, on, tg, double, mistake=None):
    """Q_target(s')[a*] for a* = the fp64 first argmax and its runner-up -> (nx1, S1, nx2, S2, ties, a1)"""
    Qt, St = scalar_q(kind, hnt, tg)
    if double and mistake != 'double_target_astar':
        Qo, So = scalar_q(kind, hn, on)
        a1, a2, tie = pick(Qo, So)
    else:
        a1, a2, tie = pick(Qt, St)
    return take(Qt, a1), take(St, a1), take(Qt, a2), take(St, a2), tie, a1


def td_target(rew, done, gamma, nx, Snx):
    """y = r + (gamma nx) (1 - d): the product and the add rounded, nx's error scaled by gamma -> (y, S)"""
    g = float(gamma) * (1 - t64(done).to(nx.device))
    gn = g * nx
    y = t64(rew).to(nx.device) + gn
    return y, gn.abs() + y.abs() + g * Snx


def from_qy(q, y, w, B, eps):
    """what the scalar tail computes from its own q and y: delta = q - y (1 rounding), dq = (2 / B) w delta (3 roundings: 2 / B, * w,
    * delta), the priority |delta| + eps in double (delta's rounding) and the loss terms w delta^2 (2 roundings)"""
    q, y = t64(q), t64(y)
    w = torch.ones_like(q) if w is None else t64(w).to(q.device)
    d = q - y
    return {'delta': d, 'dq': 2 * w * d / B, 'dq_rel': 4.0, 'prio': (d.abs() + eps, d.abs()), 'l': w * d * d}


def loss_ref(l, B, mistake=None):
    """tail_loss on the per-transition terms l (each off by <= 2 roundings when squared, 1 otherwise: counted in S) -> (loss, S)"""
    if mistake == 'loss_last_block':
        l = l[:((B - 1) // 4) * 4]
    return l.sum() / B, (n_loss(B) + 3) * l.abs().sum() / B


def scalar_dcore(kind, dq, act, on, mistake=None):
    """dL/dh [B, 512]: plain dq W[a] (dq within 4 roundings, the product 1); dueling dq ((w_v + W_adv[a]) - wsum / A), wsum the A-add
    column sum -> (dcore, S)"""
    W = t64(on['W']).to(dq.device)
    if kind == 'plain':
        t = dq[:, None] * W[act]
        return t, 5 * t.abs()
    Wv, Wa = W[0], W[1:]
    A = Wa.shape[0]
    mean = Wa.sum(0) / (A - 1 if mistake == 'dueling_mean_A_minus_1' else A)
    col = (Wv + Wa[act]) - (0 if mistake == 'dueling_dcore_no_mean' else mean)
    t = dq[:, None] * col
    S = dq.abs()[:, None] * (5 * col.abs() + (Wv.abs() + Wa[act].abs()) + (A + 1) * Wa.abs().mean(0) + (Wv + Wa[act]).abs())
    return t, S


def scalar_wgrad(kind, dq, act, h, A, B, mistake=None):
    """the head gradient [R][513] (column 512: the bias) of dqn_wgrad + reduce: plain row a = sum_n 1[a_n = a] dq_n [h_n | 1]; dueling row
    0 = sum_n dq_n [h_n | 1], row 1 + a = sum_n dq_n (1[a_n = a] - fl(1 / A)) [h_n | 1] -> (g, S)"""
    spg, groups = wgrad_groups(B)
    hb = torch.cat([t64(h), torch.ones(B, 1, dtype=F64, device=dq.device)], 1)
    if mistake == 'bias_dropped':
        hb[:, 512] = 0
    if mistake == 'wgrad_last_group':
        keep = torch.arange(B, device=dq.device) < (groups - 1) * spg * DQN_SLAB
        dq = torch.where(keep, dq, torch.zeros_like(dq))
    oh = torch.nn.functional.one_hot(act, A).to(F64)
    if kind == 'plain':
        coef, extra = oh * dq[:, None], 4
    else:
        inv = float(torch.tensor(1.0 / (A - 1 if mistake == 'dueling_mean_A_minus_1' else A), dtype=torch.float32))
        coef, extra = torch.cat([dq[:, None], dq[:, None] * (oh - inv)], 1), 6
    g = coef.T @ hb
    return g, (spg * DQN_SLAB + groups + extra) * (coef.abs().T @ hb.abs())


# ------------------------------------------------------------------------------------------------ C51 and QR logits / quantiles
def gemm_rows(h, W, b, mistake=None):
    """cat_gemm_kernel<false>: [N][R] = h W^T + b, one 512-fmaf chain + the bias add -> (x, S)"""
    x, S = lin(h, W, b)
    if mistake == 'gemm_row0_unstored':
        x = x.clone()
        x[0::CG_BM] = math.nan
    return x, 513 * S


def cat_wgrad(dl, h, B, mistake=None):
    """cat_gemm_kernel<true>: gW [R][513] = dl^T [h | 1], one B-fmaf chain per output in ascending n -> (g, S)"""
    dl = t64(dl)
    hb = torch.cat([t64(h).to(dl.device), torch.ones(B, 1, dtype=F64, device=dl.device)], 1)
    if mistake == 'bias_dropped':
        hb[:, 512] = 0
    if mistake == 'wgrad_last_kstage':
        dl = dl.clone()
        dl[CG_BK * ((B - 1) // CG_BK):] = 0
    return dl.T @ hb, B * (dl.abs().T @ hb.abs())


def row_dcore(dl, W, width):
    """dL/dh = sum_k d_k W[act width + k] (k ascending, width fmaf) on the kernel's own dense row dl [B, R] (zero outside the taken
    action's block, which the caller checks) -> (dcore, S)"""
    dl = t64(dl)
    W = t64(W).to(dl.device)
    return dl @ W, width * (dl.abs() @ W.abs())


# ------------------------------------------------------------------------------------------------ C51
def softmax_rows(x):
    """p, log p of rows [..., K] and the first-order error of p in units of U: expf 2 ulp, x - max, the K-add sum, the division"""
    K = x.shape[-1]
    mx = x.max(-1, keepdim=True).values
    lse = torch.log(torch.exp(x - mx).sum(-1, keepdim=True))
    lp = (x - mx) - lse
    p = lp.exp()
    Sp = p * ((x - mx).abs() + K + 4)
    Slp = (x - mx).abs() + lp.abs() + lse.abs() + K + 3                # x - mx, - lse, logf 1 ulp, the sum inside the log
    return p, lp, Sp, Slp


def cat_q(x, z):
    """Q [..., A] = sum_k z_k p_k (K fmaf) of logits [..., A, K] -> (Q, S).  Each p_k = e_k / se carries its own errors (x_k - max, expf's
    2 ulp, the division: |x_k - max| + 3) and the one relative error of se's K adds, common to every p_k, which scales Q as a whole:
    (K + 1) |Q|; then the K fmaf"""
    p, _, _, _ = softmax_rows(x)
    z = t64(z).to(x.device)
    K = x.shape[-1]
    mx = x.max(-1, keepdim=True).values
    Q = (p * z).sum(-1)
    return Q, (z.abs() * p * ((x - mx).abs() + 3)).sum(-1) + (K + 1) * Q.abs() + K * (p * z).abs().sum(-1)


def project(p, Sp, rew, g, z, dz, lo, hi, mistake=None):
    """Algorithm 1 on rows p [B, K] (cat_project): Tz_j = clamp(r + g z_j), b_j = (Tz_j - lo) / dz, l / u = floor / ceil clamped to
    [0, K - 1] -> (m, S).  b_j's error: g z (1), + r (1), - lo (1), / dz (1); m moves by p_j per unit of b_j, also on the neighbours of l
    and u (b_j near an integer); the split products and differences (2); the K adds into m_k."""
    B, K = p.shape
    dev = p.device
    z = t64(z).to(dev)
    rew, g = t64(rew).to(dev)[:, None], t64(g).to(dev)[:, None]
    gz = g * z[None]
    tz = (rew + gz).clamp(lo, hi)
    b = (tz - lo) / dz
    Sb = ((gz.abs() + (rew + gz).abs() + (tz - lo).abs()) / dz + b.abs())
    lo_i = b.floor().long().clamp(0, K - 1)
    up_raw = b.ceil().long().clamp(min=0)
    up = up_raw if mistake == 'project_u_unclamped' else up_raw.clamp(max=K - 1)
    eq = lo_i == up
    if mistake == 'project_split_l_eq_u':
        wl, wu = p * (up.to(F64) - b), p * (b - lo_i.to(F64))
    else:
        wl = torch.where(eq, p, p * (up.to(F64) - b))
        wu = torch.where(eq, torch.zeros_like(p), p * (b - lo_i.to(F64)))
    m = torch.zeros(B, K + 1, dtype=F64, device=dev)                  # column K: mass past the support (the unclamped mistake)
    m.scatter_add_(1, lo_i, wl)
    m.scatter_add_(1, up.clamp(max=K), wu)
    m = m[:, :K]
    e = Sp + p * Sb + 2 * p
    S = torch.zeros(B, K, dtype=F64, device=dev)
    for off in (-1, 0, 1):
        S.scatter_add_(1, (lo_i + off).clamp(0, K - 1), e)
        S.scatter_add_(1, (up.clamp(max=K - 1) + off).clamp(0, K - 1), e)
    return m, S + K * m


def cat_tail(xs, m, z, w, B):
    """the rest of cat_transition on the online logits of s at the taken action xs [B, K] and the kernel's own m [B, K] -> dict of
    (value, S): ce = -sum m lp, kl = sum_{m > 0} m (log m - lp) (the priority max(kl, 0) + eps), q = sum z p, y = sum z m, and the
    dense dlogits (w fl(1 / B)) (p sum m - m)"""
    xs, m = t64(xs), t64(m).to(xs.device)
    z = t64(z).to(xs.device)
    K = xs.shape[1]
    p, lp, Sp, Slp = softmax_rows(xs)
    w = torch.ones(B, dtype=F64, device=xs.device) if w is None else t64(w).to(xs.device)
    ce = -(m * lp).sum(1)
    lm = torch.where(m > 0, torch.log(torch.where(m > 0, m, torch.ones_like(m))), torch.zeros_like(m))
    klt = torch.where(m > 0, m * (lm - lp), torch.zeros_like(m))
    kl = klt.sum(1)
    msum = m.sum(1, keepdim=True)
    wB = (w / B)[:, None]
    dl = wB * (p * msum - m)
    return {
        'ce': (ce, (m * Slp).sum(1) + K * (m * lp).abs().sum(1)),
        'kl': (kl, (m * (Slp + lm.abs() + 1)).sum(1) + K * klt.abs().sum(1)),
        'q': cat_q(xs[:, None], z)[0][:, 0], 'q_S': cat_q(xs[:, None], z)[1][:, 0],
        'y': ((m * z).sum(1), K * (m * z).abs().sum(1)),
        'dl': (dl, wB.abs() * (Sp * msum + p * K * msum + 5 * (p * msum).abs() + (p * msum - m).abs() + m.abs())),
    }


# ------------------------------------------------------------------------------------------------ QR
def qr_q(x):
    """Q [..., A] = (sum_i x_i) / N of quantiles [..., A, N] -> (Q, S): N adds + the division"""
    N = x.shape[-1]
    return x.sum(-1) / N, (N * x.abs().sum(-1) + x.sum(-1).abs()) / N


def qr_targets(xt, a, rew, g):
    """T_j = r + g theta'_{a*,j} (2 roundings; g = 0: T = r exactly) -> (T, S)"""
    t = t64(xt)[torch.arange(xt.shape[0], device=xt.device), a]
    g = t64(g).to(t.device)[:, None]
    gt = g * t
    T = t64(rew).to(t.device)[:, None] + gt
    return T, gt.abs() + T.abs()


def qr_taus(N, device, mistake=None):
    i = torch.arange(N, dtype=F64, device=device)
    return i / N if mistake == 'tau_i_over_N' else (2 * i + 1) / (2 * N)


def qr_loss(ta, T, kappa, w, B, mistake=None, chunk=2048):
    """qr_transition on the online quantiles of the taken action ta [B, N] and the kernel's own target quantiles T [B, N] -> (loss_n, S,
    dtheta [B, N], S).  Per pair: u = T_j - theta_i (1), wt = |tau_i - 1{u < 0}| (tau 1, the difference 1), L = u^2 / 2 (1 + u's
    error times |u|) or kappa (|u| - kappa / 2) (2 + kappa times u's), wt L (1); S_i over j (N adds), <= 8 lane adds + 5 butterfly +
    / kappa + / N.  dtheta_i = -(w fl(1 / B)) (G_i / fl(kappa N)): clamp(u) is 1-Lipschitz, wt clamp(u) (1), N adds, 5 roundings after."""
    ta, T = t64(ta), t64(T).to(ta.device)
    Bn, N = ta.shape
    k = float(kappa)
    w = torch.ones(Bn, dtype=F64, device=ta.device) if w is None else t64(w).to(ta.device)
    tau = qr_taus(N, ta.device, mistake)[None, :, None]
    out = [[], [], [], []]
    for s in range(0, Bn, chunk):
        u = T[s:s + chunk, None, :] - ta[s:s + chunk, :, None]        # [b, i, j]
        au = u.abs()
        wt = (tau - (u < 0).to(F64)).abs()
        quad = (au < k) if mistake == 'kappa_strict' else (au <= k)
        L = torch.where(quad, 0.5 * u * u, k * (au - 0.5 * k))
        SL = torch.where(quad, L + u * u, 2 * k * au + L)
        rho = wt * L
        Srho = wt * SL + L * (tau + wt) + rho
        loss = rho.sum((1, 2)) / (k * N)
        Sloss = (Srho.sum((1, 2)) + (N + QR_PER_LANE + 5 + 2) * rho.sum((1, 2))) / (k * N)
        c = u.clamp(-k, k)
        gi = wt * c
        Sg = wt * au * (au <= k) + c.abs() * (tau + wt) + gi.abs()
        sc = (w[s:s + chunk] / B)[:, None] / (k * N)
        d = -sc * gi.sum(2)
        Sd = sc.abs() * (Sg.sum(2) + (N + 5) * gi.abs().sum(2))
        for o, v in zip(out, (loss, Sloss, d, Sd)):
            o.append(v)
    return tuple(torch.cat(o) for o in out)


# ------------------------------------------------------------------------------------------------ distributional dueling
def dd_compose(wv, bv, wa, ba, A, mistake=None):
    """dist_dueling_compose_kernel: rows[a V + k] = (v[k] + adv[a V + k]) - (sum_a' adv[a' V + k]) / A, columns j < 512 and the bias ->
    (W [A V][512], b [A V], S_W, S_b): A adds + the division for the mean, then + and - (2 roundings)"""
    out = []
    for v, a in ((t64(wv), t64(wa)), (t64(bv)[:, None], t64(ba)[:, None])):
        V = v.shape[0]
        a3 = a.to(v.device).view(A, V, -1)
        mean = a3.sum(0) / A
        r = (v[None] + a3) - mean[None]
        S = (A + 1) * a3.abs().mean(0)[None] + (v[None] + a3).abs() + r.abs()
        out += [r.reshape(A * V, -1), S.reshape(A * V, -1)]
    return out[0], out[2][:, 0], out[1], out[3][:, 0]


def dd_grad(gW, gb, A, V, mistake=None):
    """dist_dueling_grad_kernel on the kernel's own composed-row gradient [A V][513] (column 512: the bias): g_v[k] = sum_a g[a V + k]
    (A adds), g_adv[a V + k] = g[a V + k] - g_v[k] / A (the division and the difference) -> (g_v [V][513], S, g_adv [A V][513], S)"""
    g = torch.cat([t64(gW).view(A * V, 512), t64(gb).to(gW.device).view(A * V, 1)], 1).view(A, V, 513)
    gv = g.sum(0)
    if mistake == 'dd_grad_mean_axis':
        mean = g.sum(1, keepdim=True).expand(A, V, 513) / V
    else:
        mean = (gv / (A - 1 if mistake == 'dd_grad_A_minus_1' else A))[None].expand(A, V, 513)
    ga = g - mean
    Sv = A * g.abs().sum(0)
    Sa = (A + 1) * g.abs().mean(0)[None] + ga.abs()
    return gv, Sv, ga.reshape(A * V, 513), Sa.reshape(A * V, 513)
