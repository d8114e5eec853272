"""fp64 references of the V-trace and IMPALA loss-tail kernels (csrc/vtrace.cu), on whichever operands the caller passes, with the
per-element rounding bound of each output and the kernel mistakes a check has to be able to see.

Plain numpy, vectorised over the batch (or rows), looping over T only.  The GPU check (tests/test_gpu_tail_exact.py) evaluates each
stage on the GPU's own output of the stage before it, so every bound stays local: pg on the kernel's vs, dlogits and the pg loss on
the kernel's pg, dbaseline and the baseline loss on the kernel's vs, from_logits' vs / pg on its own log_rhos.
tests/test_tail_ref_cpu.py proves the references (against oracle.impala_oracle's fp64 V-trace and float64 autograd through the
reference's loss statements), shows the bounds hold for the fp32 CPU oracle and that every mistake below moves its witness case.

Bounds.  Every bound is per element, `c * U * S`: U = 2^-24 (fp32's unit roundoff), S the fp64 sum of the |terms| that reach the
output, and c is written next to each check (CHECK_C) with the reason for it.  Summed losses use S = n_chain * sum|terms| (+ the
per-term bounds), n_chain the longest chain of roundings in that kernel's summation order (n_chain_*).  expf is within 2 ulp and
logf within 1 ulp (CUDA C Programming Guide, Mathematical Functions); the project compiles without fast-math.

MISTAKES are plausible kernel errors; each must move the reference of its witness case by at least SENS x the bound on some element.
"""
import functools

import numpy as np

from tests import exact as E
from tests.exact import U

ETA = 2.0 ** -126           # fp32's smallest normal: a result that underflows keeps only an absolute accuracy, c * ETA is added to each bound
SENS = 20.0

# c of each check: the multiple of U * S an fp32 kernel may be off by, and why
CHECK_C = {
    # the recursion: per step <= 4 roundings and expf's 2 ulp in rho, which also enter the products of the c_t; the scan kernels
    # compose the affine maps in a 5-level tree (one product and one fma per level): 32 covers both orders
    'vs': 32,
    # gamma * vs', + r, - V, * prho: four roundings and expf's 2 ulp, doubled
    'pg': 8,
    # x - max, - lse, logf, and the A expf / adds of the sum inside the log (counted in S): 2x the first-order count
    'logp': 4,
    'log_rhos': 4,
    # sum_a p log p: S already carries the propagated logp / exp errors to first order; 2x for second-order terms
    'entropy': 2,
    'dlogits': 2,
    # -cost * (vs - V): one subtraction, one product
    'dbaseline': 4,
    # summation trees: S = n_chain * sum|terms| is the first-order bound of the tree (Higham, Accuracy and Stability, eq. 4.4); 2x
    'loss': 2,
    # reduce_sum: the same tree bound, with the square and the scale counted in n_chain: gamma_n = n U / (1 - n U) <= 1.01 n U for
    # n U <= 0.01 (n_chain <= 16397 here)
    'reduce_sum': 1.01,
}

MISTAKES = {
    'cbar_rho': 'c_t clipped at the rho threshold instead of 1',
    'clips_swapped': 'the rho and pg-rho thresholds swapped',
    'pg_values': 'V_{t+1} in place of vs_{t+1} in the pg advantages',
    'boot_zero': 'the bootstrap value taken as 0',
    'chunk_carry': 'the carry into a 32-step chunk dropped',
    'discount_row_t': 'the discount read from trajectory row t instead of t + 1',
    'action_row_t': 'the action read from trajectory row t instead of t + 1',
    'no_reward_clip': 'the reward clip omitted',
    'entropy_dropped': 'the entropy term left out of dlogits',
    'entropy_sign': 'the entropy term of dlogits with its sign flipped',
    'baseline_no_half': 'the 0.5 of the baseline loss dropped',
    'dbaseline_sign': 'dbaseline with its sign flipped',
    'entropy_loss_sign': 'the entropy loss with its sign flipped',
}


def f64(x):
    return np.asarray(x.cpu() if hasattr(x, 'cpu') else x, dtype=np.float64)


# ------------------------------------------------------------------------------------------------ rows
def clamp_actions(a, A):
    """the action a kernel reads (ld_action): clamped to [0, A)"""
    return np.clip(np.asarray(a.cpu() if hasattr(a, 'cpu') else a, dtype=np.int64), 0, A - 1)


def rows(x):
    """log_softmax of rows [..., A] (vtrace.py:31-40) and sum_a p log p (loss_fn.py:9-13) -> dict(lp, p, ent, mx, lse, s_lp, s_ent).
    s_lp [..., A]: |x_a| + |max| + |lse| + A + 1 (the A expf / adds inside the log each move lse by <= U, logf by <= U |lse|).
    s_ent [...]: the first-order bound of the kernel's sum_a expf(lp) lp, lp within CHECK_C['logp'] U s_lp, over U."""
    x = f64(x)
    A = x.shape[-1]
    mx = x.max(-1, keepdims=True)
    lse = np.log(np.exp(x - mx).sum(-1, keepdims=True))
    lp = (x - mx) - lse
    p = np.exp(lp)
    e_lp = CHECK_C['logp'] * (np.abs(x) + np.abs(mx) + np.abs(lse) + A + 1)
    s_ent = (p * ((1 + np.abs(lp)) * e_lp + 2 * np.abs(lp))).sum(-1) + A * np.abs(p * lp).sum(-1)
    return {'lp': lp, 'p': p, 'ent': (p * lp).sum(-1), 'mx': mx[..., 0], 'lse': lse[..., 0], 's_lp': e_lp / CHECK_C['logp'],
            'e_lp': e_lp, 's_ent': s_ent}


def gather(v, a):
    return np.take_along_axis(v, a[..., None], -1)[..., 0]


def policy_grad(rw, act, w_logp, w_ent, mistake=None):
    """d/dlogits of sum_n w_logp[n] logp[n] + w_ent[n] ent[n] (policy_rows_bwd_kernel): w_logp (1{a} - p) + w_ent p (lp - ent);
    None weights are zeros, act None means no action.  -> (d, S)"""
    p, lp, ent, e_lp = rw['p'], rw['lp'], rw['ent'][..., None], rw['e_lp']
    d = np.zeros_like(p)
    S = np.zeros_like(p)
    if w_logp is not None:
        wl = f64(w_logp)[..., None]
        oh = np.zeros_like(p)
        np.put_along_axis(oh, act[..., None], 1.0, -1)
        if mistake != 'logp_p_dropped':
            d += wl * (oh - p)
        else:
            d += wl * oh
        S += np.abs(wl) * (p * (e_lp + 2) + np.abs(oh - p) * 2)
    if w_ent is not None:
        we = f64(w_ent)[..., None]
        sgn = -1.0 if mistake == 'entropy_sign' else 1.0
        d += sgn * we * p * (lp - ent)
        S += np.abs(we) * p * (np.abs(lp - ent) * (e_lp + 4) + e_lp + rw['s_ent'][..., None])
    return d, S


def reduce_sum(x, square, scale):
    """scale * sum x (or x^2) -> (value, S): S = n_chain * sum|terms| of reduce_sum_kernel's order (n_chain_reduce)"""
    x = f64(x).reshape(-1)
    t = x * x if square else x
    return scale * t.sum(), n_chain_reduce(x.size, square) * abs(scale) * np.abs(t).sum()


def n_chain_reduce(n, square):
    """reduce_sum_kernel: 1024 threads each add ceil(n / 1024) terms, then a 5-level warp sum, then the 32 warp partials in a second
    5-level warp sum, then the scale (and the square of each term)"""
    return -(-n // 1024) + 5 + 5 + 1 + (1 if square else 0)


def sample_ref(x, u):
    """the inverse CDF of sample_actions_kernel in fp64: the first a with u * sum_j e_j < sum_{j <= a} e_j, e_j = exp(x_j - max) ->
    (action, margin, bound): margin = the distance of the target from the nearest CDF boundary, bound = what the kernel's fp32 target
    and boundaries may be off by (expf 2 ulp each, one rounding per add and for u * se; first order, then 2x)"""
    x = f64(x)
    e = np.exp(x - x.max(-1, keepdims=True))
    C = np.cumsum(e, -1)
    se = C[..., -1]
    tgt = f64(u) * se
    act = np.minimum((tgt[..., None] >= C).sum(-1), x.shape[-1] - 1)
    margin = np.abs(tgt[..., None] - C[..., :-1]).min(-1) if x.shape[-1] > 1 else np.full(se.shape, np.inf)
    bound = 2 * U * (5 * se + 2 * C.sum(-1))
    return act, margin, bound


# ------------------------------------------------------------------------------------------------ V-trace
def _clipf(rho, thr):
    return rho if thr is None else np.minimum(rho, thr)


def vtrace_vs(log_rhos, discounts, rewards, values, boot, clip_rho=1.0, clip_pg=1.0, lr_err=None, mistake=None):
    """vs of vtrace.py:135-169 in fp64 -> (vs, S).  M_t = rhobar_t (|r_t| + |g_t V_{t+1}| + |V_t|) + |g_t c_t| M_{t+1} is the recursion on
    magnitudes; S_t = (1 + L_t) rhobar_t (|r_t| + |g_t V_{t+1}| + |V_t|) + |g_t c_t| (S_{t+1} + L_t M_{t+1}), plus |V_t| + |vs_t|, is its
    first-order error over U: L_t = lr_err (the log_rho's own bound over U; 0 for given log_rhos) enters rhobar_t and c_t once, so it
    scales the step's own delta and the carried magnitude M_{t+1}, not the carried error S_{t+1}"""
    lr, g, r, v = (f64(a) for a in (log_rhos, discounts, rewards, values))
    boot = np.zeros_like(f64(boot)) if mistake == 'boot_zero' else f64(boot)
    T = lr.shape[0]
    rho = np.exp(lr)
    crho = _clipf(rho, clip_pg if mistake == 'clips_swapped' else clip_rho)
    cs = _clipf(rho, clip_rho) if mistake == 'cbar_rho' else np.minimum(rho, 1.0)
    L = np.zeros_like(lr) if lr_err is None else f64(lr_err)
    vs, S = np.empty_like(lr), np.empty_like(lr)
    acc, s, m = np.zeros_like(boot), np.zeros_like(boot), np.zeros_like(boot)
    vnext = boot
    for t in range(T - 1, -1, -1):
        if mistake == 'chunk_carry' and (t + 1) % 32 == 0:
            acc = np.zeros_like(acc)
        acc = crho[t] * (r[t] + g[t] * vnext - v[t]) + g[t] * cs[t] * acc
        delta = crho[t] * (np.abs(r[t]) + np.abs(g[t] * vnext) + np.abs(v[t]))
        gc = np.abs(g[t] * cs[t])
        s = (1 + L[t]) * delta + gc * (s + L[t] * m)
        m = delta + gc * m
        vs[t] = acc + v[t]
        S[t] = s + np.abs(v[t]) + np.abs(vs[t])
        vnext = v[t]
    return vs, S


def vtrace_pg(log_rhos, discounts, rewards, values, boot, vs, clip_rho=1.0, clip_pg=1.0, lr_err=None, mistake=None):
    """pg advantages on the given vs (vtrace.py:166-169) -> (pg, S), S = (1 + L_t) prho_t (|r_t| + |g_t vs_{t+1}| + |V_t|)"""
    lr, g, r, v, vs = (f64(a) for a in (log_rhos, discounts, rewards, values, vs))
    boot = np.zeros_like(f64(boot)) if mistake == 'boot_zero' else f64(boot)
    nxt = np.concatenate([(v if mistake == 'pg_values' else vs)[1:], boot[None]], 0)
    prho = _clipf(np.exp(lr), clip_rho if mistake == 'clips_swapped' else clip_pg)
    L = np.zeros_like(lr) if lr_err is None else f64(lr_err)
    return prho * (r + g * nxt - v), (1 + L) * prho * (np.abs(r) + np.abs(g * nxt) + np.abs(v))


# ------------------------------------------------------------------------------------------------ the fused tail
def n_chain_tail(kernel, T, B):
    """the longest chain of roundings of a loss in each tail kernel's summation order, the term's own product and the cost included:
    warp:   lane over ceil(T/32) chunks, warp sum (5), (w0 + w1) + (w2 + w3) (2), lane over ceil(nblocks/32) block partials, warp sum (5)
    thread: thread over T steps, warp sum (5), block (2), the fp64 sum of the block partials rounded once (1)
    column: lane over ceil(T/32) chunks, warp sum (5), lane over ceil(B/32) column partials, warp sum (5)"""
    ch = -(-T // 32)
    if kernel == 'warp':
        core = ch + 5 + 2 + -(-(-(-B // 4)) // 32) + 5
    elif kernel == 'thread':
        core = T + 5 + 2 + 1
    else:
        core = ch + 5 + -(-B // 32) + 5
    return core + 2


def tail(bl, tl, baseline, action, reward, done, hp, kernel, vs_k=None, pg_k=None, mistake=None):
    """impala_atari.py:293-330 + loss_fn.py:5-23 + the head gradients on [T+1, B] rows: model rows t (target logits, baseline), trajectory
    rows t + 1 (behaviour logits, action, reward, done), bootstrap = baseline[T].  vs_k / pg_k: the kernel's vs / pg, on which pg,
    dbaseline, dlogits and the losses are evaluated (None: this function's own).  hp: discounting, clip_reward, clip_rho, clip_pg,
    baseline_cost, entropy_cost.  -> dict of (value, S) pairs: vs, pg, dlogits, dbaseline, loss_pg, loss_baseline, loss_entropy, total"""
    bl, tl, base, rew = f64(bl), f64(tl), f64(baseline), f64(reward)
    done = np.asarray(done.cpu() if hasattr(done, 'cpu') else done).astype(bool)
    T1, B, A = tl.shape
    T = T1 - 1
    act_all = clamp_actions(action, A)
    row = slice(0, T) if mistake in ('action_row_t',) else slice(1, T1)
    act = act_all[row]
    drow = slice(0, T) if mistake == 'discount_row_t' else slice(1, T1)
    r = rew[1:] if (mistake == 'no_reward_clip' or not hp['clip_reward']) else np.clip(rew[1:], -1, 1)
    g = np.where(done[drow], 0.0, hp['discounting'])
    tr, br = rows(tl[:T]), rows(bl[1:])
    talp, balp = gather(tr['lp'], act), gather(br['lp'], act)
    lr = talp - balp
    lr_err = gather(tr['e_lp'], act) + gather(br['e_lp'], act) + 2
    v, boot = base[:T], base[T]
    vtm = mistake if mistake in ('cbar_rho', 'clips_swapped', 'boot_zero', 'chunk_carry') else None
    vs, vs_S = vtrace_vs(lr, g, r, v, boot, hp['clip_rho'], hp['clip_pg'], lr_err, vtm)
    vsk = vs if vs_k is None else f64(vs_k)
    pgm = vtm if vtm != 'chunk_carry' else None
    if mistake == 'pg_values':
        pgm = 'pg_values'
    pg, pg_S = vtrace_pg(lr, g, r, v, boot, vsk, hp['clip_rho'], hp['clip_pg'], lr_err, pgm)
    adv = pg if pg_k is None else f64(pg_k)
    ec, bc = hp['entropy_cost'], hp['baseline_cost']
    w_ent = None
    if mistake != 'entropy_dropped':
        w_ent = np.full(adv.shape, ec)
    dl, dl_S = policy_grad(tr, act, -adv, w_ent, 'entropy_sign' if mistake == 'entropy_sign' else None)
    d = vsk - v
    db, db_S = (bc if mistake == 'dbaseline_sign' else -bc) * d, abs(bc) * (np.abs(vsk) + np.abs(v))
    n = n_chain_tail(kernel, T, B)
    t_pg = -talp * adv
    l_pg = (t_pg.sum(), n * np.abs(t_pg).sum() + (np.abs(adv) * gather(tr['e_lp'], act)).sum())
    half = 1.0 if mistake == 'baseline_no_half' else 0.5
    t_bl = half * d * d
    l_bl = (bc * t_bl.sum(), abs(bc) * ((n + 4) * np.abs(t_bl).sum()))
    l_ent = ((-ec if mistake == 'entropy_loss_sign' else ec) * tr['ent'].sum(), abs(ec) * (n * np.abs(tr['ent']).sum() + tr['s_ent'].sum()))
    tot = (l_pg[0] + l_bl[0] + l_ent[0], l_pg[1] + l_bl[1] + l_ent[1] + 2 * (abs(l_pg[0]) + abs(l_bl[0]) + abs(l_ent[0])))
    return {'vs': (vs, vs_S), 'pg': (pg, pg_S), 'dlogits': (dl, dl_S), 'dbaseline': (db, db_S), 'loss_pg': l_pg, 'loss_baseline': l_bl,
            'loss_entropy': l_ent, 'total': tot}


TAIL_LOSSES = ('loss_pg', 'loss_baseline', 'loss_entropy', 'total')
TAIL_CHECK_C = {'vs': 'vs', 'pg': 'pg', 'dlogits': 'dlogits', 'dbaseline': 'dbaseline', 'loss_pg': 'loss', 'loss_baseline': 'loss',
                'loss_entropy': 'loss', 'total': 'loss'}
# which mistakes each tail output can show
TAIL_MISTAKES = {'vs': ('cbar_rho', 'clips_swapped', 'boot_zero', 'chunk_carry', 'discount_row_t', 'action_row_t', 'no_reward_clip'),
                 'pg': ('clips_swapped', 'pg_values', 'boot_zero', 'discount_row_t', 'action_row_t', 'no_reward_clip'),
                 'dlogits': ('entropy_dropped', 'entropy_sign', 'action_row_t'),
                 'dbaseline': ('dbaseline_sign',), 'loss_pg': ('action_row_t',), 'loss_baseline': ('baseline_no_half',),
                 'loss_entropy': ('entropy_loss_sign',), 'total': ('baseline_no_half', 'entropy_loss_sign', 'action_row_t')}


# ------------------------------------------------------------------------------------------------ comparisons
# max |got - ref| / (c (U S + ETA)), and how far a mistake moves the reference in those units; an output NaN on both sides is NaN, so
# its check fails
ratio = functools.partial(E.ratio, eta=ETA, nan_equal=False)
sensitivity = functools.partial(E.sensitivity, eta=ETA, nan_equal=False)


# ------------------------------------------------------------------------------------------------ shared case table and inputs
def _disc(rng, T, B, regime):
    if regime == 'p05':            # gamma = 0.99 with 5 % dones
        return ((rng.rand(T, B) > 0.05) * 0.99).astype(np.float32)
    if regime == 'one':            # gamma = 1, no dones
        return np.ones((T, B), np.float32)
    return np.zeros((T, B), np.float32)


def _lr(rng, T, B, regime):
    if regime == 'n08':
        return (rng.randn(T, B) * 0.8).astype(np.float32)
    return np.clip(rng.randn(T, B) * 3, -20, 20).astype(np.float32)


# from_importance_weights: name -> (T, B, variant, (clip_rho, clip_pg), discounts, log_rhos, 4-byte offset, kernel, witnesses, edge)
IW_CASES = {
    'scan_T1': (1, 67, 1, (1.0, 1.0), 'p05', 'n08', False, 'scan', (), 'the scan kernel with one step: lane 0 alone, no recursion'),
    'scan_T31': (31, 67, 1, (2.0, 0.5), 'p05', 'n08', False, 'scan', ('cbar_rho', 'clips_swapped', 'pg_values'),
                 'one partial chunk (lane 31 idle); thresholds (2, 0.5)'),
    'scan_T32': (32, 67, 1, (None, None), 'one', 'n3', False, 'scan', ('boot_zero',), 'exactly one chunk; no clipping, wide log_rhos'),
    'scan_T33': (33, 67, 1, (0.5, 2.0), 'p05', 'n08', False, 'scan', ('chunk_carry', 'clips_swapped'),
                 'two chunks, the second with one step: the carry'),
    'scan_T64': (64, 67, 1, (1.0, 1.0), 'one', 'n08', False, 'scan', ('chunk_carry', 'boot_zero'), 'two full chunks, gamma = 1'),
    'scan_T65': (65, 67, 1, (2.0, 0.5), 'zero', 'n3', False, 'scan', (), 'three chunks, all discounts zero: no recursion at all'),
    'scan_T128': (128, 67, 1, (2.0, 0.5), 'one', 'n08', False, 'scan', ('chunk_carry', 'cbar_rho'),
                  'SCAN_MAX_T: 66 KB of shared memory, four chunks, gamma = 1 and no dones'),
    'scan_T129': (129, 67, 1, (1.0, 1.0), 'p05', 'n08', False, 'seq1', (),
                  'one past SCAN_MAX_T: variant 1 falls back to the sequential kernel, bit for bit variant 0'),
    'seq4': (20, 67584, 0, (1.0, 1.0), 'p05', 'n08', False, 'seq4', ('boot_zero',), 'B = 4 x 128 x 132: the 4-wide sequential kernel'),
    'seq1_offset': (20, 67584, 0, (2.0, 0.5), 'p05', 'n08', True, 'seq1', ('cbar_rho', 'clips_swapped'),
                    'the same B with operands at a 4-byte offset: the 1-wide fallback'),
    'seq1_B67585': (20, 67585, 0, (None, None), 'p05', 'n3', False, 'seq1', (), 'B % 4 = 1: the 1-wide fallback'),
    'seq_B1': (7, 1, 0, (0.5, 2.0), 'p05', 'n08', False, 'seq1', (), 'one column'),
    'seq_B33': (45, 33, 0, (2.0, 0.5), 'one', 'n08', False, 'seq1', ('cbar_rho', 'clips_swapped', 'pg_values'), 'a partial block'),
    'seq_B4099': (20, 4099, 0, (1.0, 1.0), 'p05', 'n3', False, 'seq1', (), 'ragged B, wide log_rhos'),
}


def iw_inputs(name):
    """float32 numpy operands of an IW_CASES case: log_rhos, discounts, rewards, values, bootstrap"""
    T, B = IW_CASES[name][:2]
    _, _, _, _, disc, lrg = IW_CASES[name][:6]
    rng = np.random.RandomState(sum(map(ord, name)))
    return (_lr(rng, T, B, lrg), _disc(rng, T, B, disc), rng.randn(T, B).astype(np.float32), rng.randn(T, B).astype(np.float32),
            rng.randn(B).astype(np.float32))


def logit_rows(rng, shape, regime):
    """float32 logits [..., A]: 'n1' N(0, 1), 'n30' N(0, 30) (near one-hot), 'big' 1000 + N(0, 1), 'equal' rows of equal logits"""
    if regime == 'n1':
        return rng.randn(*shape).astype(np.float32)
    if regime == 'n30':
        return (rng.randn(*shape) * 30).astype(np.float32)
    if regime == 'big':
        return (1000 + rng.randn(*shape)).astype(np.float32)
    return np.repeat(rng.randn(*shape[:-1], 1), shape[-1], -1).astype(np.float32)


LOGIT_REGIMES = ('n1', 'n30', 'big', 'equal')

# from_logits: name -> (T, B, A, logit regime, (clip_rho, clip_pg), out-of-range actions, edge)
LOGITS_CASES = {
    'A1_n1': (9, 37, 1, 'n1', (1.0, 1.0), False, 'one action: every log-prob is 0, rho = 1'),
    'A2_n30': (9, 37, 2, 'n30', (2.0, 0.5), False, 'two actions, near one-hot rows'),
    'A18_big': (9, 37, 18, 'big', (None, None), False, 'logits near 1000: the max shift carries the row'),
    'A100_equal': (9, 37, 100, 'equal', (0.5, 2.0), False, 'rows of equal logits: lse = log 100 exactly'),
    'A18_oob': (9, 37, 18, 'n1', (1.0, 1.0), True, 'actions -1, A and 2^40: the kernel reads the clamped action'),
    'A100_n30': (33, 5, 100, 'n30', (2.0, 0.5), False, 'a hundred actions, near one-hot'),
}


def logits_inputs(name):
    T, B, A, reg, _, oob, _ = LOGITS_CASES[name]
    rng = np.random.RandomState(sum(map(ord, name)))
    bl, tl = logit_rows(rng, (T, B, A), reg), logit_rows(rng, (T, B, A), reg)
    act = rng.randint(0, A, size=(T, B)).astype(np.int64)
    if oob:
        act[0, :] = -1
        act[1, :] = A
        act[2, :] = 1 << 40
    return (bl, tl, act, _disc(rng, T, B, 'p05'), rng.randn(T, B).astype(np.float32), rng.randn(T, B).astype(np.float32),
            rng.randn(B).astype(np.float32))


COSTS = {
    'default': dict(discounting=0.99, clip_rho=1.0, clip_pg=1.0, baseline_cost=0.5, entropy_cost=0.0006),
    'alt': dict(discounting=1.0, clip_rho=2.0, clip_pg=0.5, baseline_cost=1.0, entropy_cost=0.05),
    'off': dict(discounting=0.99, clip_rho=None, clip_pg=None, baseline_cost=0.0, entropy_cost=0.0),
}

# impala_loss_and_head_grads: name -> (T, B, A, rewards, clip_reward, dones, costs, witnesses, edge)
TAIL_CASES = {
    'w_T1_B1_A1': (1, 1, 1, 'u3', True, 'row1', 'default', (), 'the smallest tail: one step, one column, one action'),
    'w_T31_B5_A6': (31, 5, 6, 'u3', True, 'rowT', 'alt', ('cbar_rho', 'clips_swapped', 'no_reward_clip', 'entropy_dropped', 'entropy_sign',
                                                                   'dbaseline_sign', 'entropy_loss_sign'),
                    'warp kernel, a partial chunk, the other costs'),
    'w_T32_B33_A18': (32, 33, 18, 'pm1', True, 'twice', 'default', ('baseline_no_half', 'action_row_t'),
                      'one full chunk, rewards exactly +-1, dones twice in a row'),
    'w_T33_B2048_A6': (33, 2048, 6, 'u3', False, 'p05', 'alt', ('chunk_carry', 'discount_row_t', 'action_row_t', 'pg_values', 'boot_zero'),
                       'B = 2048: the last warp-kernel size; the chunk carry'),
    'w_T100_B5_A33': (100, 5, 33, 'u3', True, 'p05', 'off', (), 'four chunks, 33 actions, no clipping and no baseline / entropy cost'),
    'w_T33_B1_A1': (33, 1, 1, 'pm1', False, 'p05', 'alt', (), 'one action: pg loss and entropy vanish'),
    'w_T20_B33_A6': (20, 33, 6, 'u3', True, 'p05', 'default', ('no_reward_clip',), 'the default learner setting'),
    'w_T100_B33_A6': (100, 33, 6, 'u3', True, 'twice', 'alt', ('chunk_carry',), 'gamma = 1 over four chunks'),
    't_T20_B2049_A6': (20, 2049, 6, 'u3', True, 'p05', 'alt', ('cbar_rho', 'clips_swapped', 'entropy_dropped', 'entropy_sign',
                                                               'discount_row_t', 'no_reward_clip', 'baseline_no_half',
                                                               'dbaseline_sign', 'entropy_loss_sign'),
                       'B = 2049: the first thread-per-column size'),
    't_T3_B4099_A4': (3, 4099, 4, 'pm1', False, 'twice', 'default', ('action_row_t',), 'thread kernel, ragged B'),
    't_T100_B2049_A18': (100, 2049, 18, 'u3', True, 'rowT', 'off', ('pg_values',), 'thread kernel, a long column, no clipping'),
    't_T1_B4099_A33': (1, 4099, 33, 'u3', True, 'row1', 'alt', (), 'thread kernel, one step'),
}


def tail_inputs(T, B, A, rewards='u3', dones='p05', seed=0):
    """[T+1, B] rows of a tail call: behaviour logits, target logits, baseline, action, reward, done (numpy float32 / int64 / bool).
    dones: 'p05' 5 % at random; 'row1' / 'rowT' also every column done at trajectory row 1 / T; 'twice' also rows t0, t0 + 1."""
    rng = np.random.RandomState(seed)
    bl, tl = logit_rows(rng, (T + 1, B, A), 'n1'), logit_rows(rng, (T + 1, B, A), 'n1')
    base = rng.randn(T + 1, B).astype(np.float32)
    act = rng.randint(0, A, size=(T + 1, B)).astype(np.int64)
    rew = (rng.uniform(-3, 3, size=(T + 1, B)) if rewards == 'u3' else rng.choice([-1.0, 1.0], size=(T + 1, B))).astype(np.float32)
    done = rng.rand(T + 1, B) < 0.05
    if dones == 'row1':
        done[1] = True
    elif dones == 'rowT':
        done[T] = True
    elif dones == 'twice':
        t0 = max(1, T // 2)
        done[t0, ::2] = True
        done[min(T, t0 + 1), ::2] = True
    return bl, tl, base, act, rew, done


def tail_case(name):
    """-> (inputs, hp, kernel) of a TAIL_CASES case"""
    T, B, A, rw, clip, dn, costs = TAIL_CASES[name][:7]
    hp = dict(COSTS[costs], clip_reward=clip)
    return tail_inputs(T, B, A, rw, dn, seed=sum(map(ord, name))), hp, ('warp' if B <= 2048 else 'thread')


# the learner at each tail boundary: (T, B, A) -> (costs, kernel, edge); bf16, learning_rate = 0
LEARNER_CASES = {
    (20, 1, 8): ('default', 'column8', 'A = 8: the last size of the 8-action column kernel'),
    (20, 3, 9): ('alt', 'column32', 'A = 9: the first size of the 32-action column kernel'),
    (20, 3, 31): ('off', 'column32', 'A = 31: the widest learner'),
    (89, 2, 6): ('alt', 'column8', 'T = 89: the last T whose column fits 200 KB of shared memory at A = 6'),
    (90, 2, 6): ('default', 'warp', 'T = 90: one past it, the three-kernel path'),
    (57, 2, 31): ('alt', 'column32', 'T = 57: the last T that fits at A = 31'),
    (58, 2, 31): ('off', 'warp', 'T = 58: one past it'),
    (20, 512, 6): ('default', 'column8', 'B = 512: the widest column-kernel batch'),
    (3, 513, 6): ('alt', 'warp', 'B = 513: the three-kernel path with the warp tail'),
    (2, 2049, 4): ('default', 'thread', 'B = 2049: the three-kernel path with the thread tail'),
}
