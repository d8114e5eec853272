"""fp64 references of the clip and optimizer kernels (csrc/optim.cu), on whichever operands the caller passes, with the per-element
rounding bound of each output and the kernel mistakes a check has to be able to see.

Plain numpy.  Operands are the float32 values a kernel received: hyperparameters as float32, 1 - a formed in fp64 from the float a
(the C ABI passes floats and the kernels compute 1.f - a, exact for a in [0.5, 1]).  The GPU check (tests/test_gpu_optim_exact.py)
keeps every bound local: square_avg / exp_avg / exp_avg_sq / the momentum buffer from the step's inputs and the GPU's clip
coefficient, the parameters on the GPU's own new state, coefficient and lr; the coefficient bit for bit on the GPU's own norm.
tests/test_optim_ref_cpu.py proves the references against torch.optim / clip_grad_norm_ / LambdaLR in float64, shows the bounds hold
for the same torch optimizers in fp32 and that every mistake below moves its witness case.

Bounds.  Every bound is per element, `c * U * S + c * ETA`: U = 2^-24, S the fp64 sum of the |terms| that reach the output (a term
that passes through k roundings more than the others enters S k times), c written next to each check (CHECK_C) with the reason for
it.  A clipped gradient (or exp_avg) in fp32's subnormal range is only accurate to ETA absolutely; where a quotient by sqrt(v) + eps
scales it, S carries ETA / U / (sqrt(v) + eps).  sqrtf and the division are correctly rounded (no fast-math).  The norm's sum of squares uses S = n_chain * sum g^2, n_chain the
longest chain of roundings in the kernel's summation order (n_chain_norm).
"""
import functools

import numpy as np

from tests import exact as E
from tests.exact import U

ETA = 2.0 ** -149           # fp32's smallest subnormal: a rounding in the subnormal range is off by at most half of it, absolutely
SENS = 20.0

# c of each check: the multiple of U * S (and of ETA) an fp32 kernel may be off by, and why
CHECK_C = {
    # a v + (1 - a) gk^2: gk = g c rounded (twice in gk^2), gk gk, (1 - a) *, the add: 5 roundings on the g term, 2 on a v;
    # FMA contraction only removes roundings; +1 for the second-order terms
    'v': 6,
    # b1 m + (1 - b1) gk: gk, the product, the add: 3; +1
    'm': 4,
    # mu buf + gk / (sqrtf(v') + eps), v' the fp64 one: gk 1, v' off by CHECK_C['v'] halved by the root (3), sqrtf 1, + eps 1,
    # the division 1, the add 1: 8 on the quotient, 2 on mu buf; +1
    'buf': 9,
    # p - delta on the GPU's own state: the subtraction 1 on |p'|, delta's own roundings in S (RMSprop 5: gk, sqrtf, + eps, /, lr *;
    # momentum 1: lr *; Adam 11: inv_bc1 2 (the float 1 - b1^t, the reciprocal), lr * inv_bc1 1, inv_sqrt_bc2 2.5 (the float
    # 1 - b2^t halved by the root, sqrtf, the reciprocal), sqrtf(v') 1, * inv_sqrt_bc2 1, + eps 1, / 1, the outer * 1); 2x for the
    # second-order terms
    'p': 2,
    # the sum of squares: gamma_n = n U / (1 - n U) <= 1.01 n U for n U <= 0.01 (Higham eq. 3.4); every term is >= 0, so S = n_chain sum g^2
    'sumsq': 1.01,
}
DELTA_C = {'rmsprop': 5, 'momentum': 1, 'adam': 11}

MISTAKES = {
    'eps_in_sqrt': 'eps inside the square root: sqrt(v + eps)',
    'unclipped_update': 'the unclipped gradient in the update',
    'unclipped_v': 'the unclipped gradient in the second moment only',
    'bias_t_plus_1': "Adam's bias corrections of step t + 1",
    'bias_no_second': "Adam's bias correction without its second factor 1 / sqrt(1 - b2^t)",
    'old_v': 'the update taken from the old second moment',
    'lr_in_momentum': 'lr folded into the momentum buffer (buf = mu buf + lr q; p -= buf)',
    'lr_prev_step': 'the lr of step t - 1',
    'clip_no_1e6': 'the clip coefficient without its 1e-6: max_norm / norm',
    'norm_no_tail': 'the norm without the n % 4 tail',
    'norm_no_hold_slot': 'the norm without the second register-held float4 slot',
}


def f64(x):
    return np.asarray(x.detach().cpu() if hasattr(x, 'detach') else x, dtype=np.float64)


def f32(x):
    return np.float32(x)


def one_minus(a):
    """1 - a of the float a, in fp64 (the kernels' 1.f - a is exact for a in [0.5, 1])"""
    return 1.0 - float(np.float32(a))


# ------------------------------------------------------------------------------------------------ the norm and the clip
def n_chain_norm(n, blocks, fused=True):
    """the longest chain of roundings of the sum of squares in the kernel's order: each thread adds ceil(n4 / stride) float4s of 4
    squares (+1 for the n % 4 tail in block 0), a 5-level warp sum, the WARPS warp sums in order (16 fused, 8 stand-alone), the fp64
    sum of the block partials (1), the float root squared (2).  stride = blocks x the block's threads (512 fused, 256 stand-alone)"""
    threads, warps = (512, 16) if fused else (256, 8)
    n4 = n // 4
    per_thread = -(-n4 // (blocks * threads)) * 4 + (1 if n % 4 else 0)
    return per_thread + 5 + warps + 1 + 2


def sumsq(g, blocks, fused=True, mistake=None):
    """sum g^2 of the kernel's operand (fp64) -> (value, S); the mistakes drop the n % 4 tail, or the float4s of HOLD slot 1 (indices
    [stride, 2 stride) of the fused kernel)"""
    g = f64(g).reshape(-1)
    n = g.size
    keep = np.ones(n, bool)
    if mistake == 'norm_no_tail':
        keep[(n // 4) * 4:] = False
    elif mistake == 'norm_no_hold_slot':
        stride = blocks * 512
        keep[4 * stride:8 * stride] = False
    s = float((g[keep] * g[keep]).sum())
    return s, n_chain_norm(n, blocks, fused) * float((g * g).sum())


def clip_coef32(norm, max_norm):
    """the kernel's clip coefficient on its own float norm, in fp32, bit for bit: min(max_norm / (norm + 1e-6f), 1); max_norm < 0, NaN
    or +inf: 1; a NaN norm: NaN (torch's clamp(max=1) keeps it)"""
    mn = np.float32(max_norm)
    if not mn >= 0 or np.isinf(mn):
        return np.float32(1.0)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        c = mn / (np.float32(norm) + np.float32(1e-6))
    return c if (c < 1 or np.isnan(c)) else np.float32(1.0)


def clip_coef_ref(norm, max_norm, mistake=None):
    """the fp64 coefficient of a given norm (the clip_no_1e6 mistake's witness is the coefficient itself)"""
    if not max_norm >= 0 or np.isinf(max_norm):
        return 1.0
    d = norm if mistake == 'clip_no_1e6' else norm + float(np.float32(1e-6))
    return min(float(np.float32(max_norm)) / d, 1.0) if d > 0 else 1.0


# ------------------------------------------------------------------------------------------------ the schedule and the snapshot
def lr_at(lr, t, schedule='constant', frames_per_step=0.0, total_frames=None, lr_end=0.0):
    """the float32 lr of the 1-based step t, the closed form the kernels evaluate (scalerl_b200.learner.scheduled_lr on float32 lr and
    lr_end, rounded to float32)"""
    from scalerl_b200.learner import scheduled_lr
    return np.float32(scheduled_lr(float(np.float32(lr)), schedule, int(t), frames_per_step, total_frames, float(np.float32(lr_end))))


def snapshot_copies(losses):
    """the weight snapshot copies when there is no loss to look at or the step's total loss (losses[3]) is finite"""
    return losses is None or bool(np.isfinite(np.float32(losses[3])))


# ------------------------------------------------------------------------------------------------ RMSprop and Adam
def _gk(g, c, mistake, where):
    g = f64(g)
    return g if mistake == f'unclipped_{where}' else g * float(c)


def rmsprop(p, g, v, c, lr, alpha, eps, buf=None, mu=0.0, v_k=None, buf_k=None, lr_prev=None, mistake=None):
    """torch.optim.RMSprop(centered=False[, momentum=mu]) on the clipped gradient g c -> {'v', ['buf'], 'p'}: (value, S) pairs.
    v' and buf' from the step's inputs; p' on v_k / buf_k (the kernel's own v' / buf'; None: this function's).  lr_prev: the lr of
    the previous step (the lr_in_momentum mistake keeps lr_prev in the buffer it was given)"""
    p, v = f64(p), f64(v)
    a, e, lr = float(np.float32(alpha)), float(np.float32(eps)), float(np.float32(lr))
    if mistake == 'lr_prev_step' and lr_prev is not None:
        lr = float(np.float32(lr_prev))
    gv, gu = _gk(g, c, mistake, 'v'), _gk(g, c, mistake, 'update')
    terms_v = (a * np.abs(v), one_minus(alpha) * gv * gv)
    v1 = a * v + one_minus(alpha) * gv * gv
    out = {'v': (v1, terms_v[0] + terms_v[1])}
    vu = v if mistake == 'old_v' else (v1 if v_k is None else f64(v_k))
    den = np.sqrt(vu + e) if mistake == 'eps_in_sqrt' else np.sqrt(vu) + e
    # a gk in the subnormal range keeps only an absolute accuracy (ETA / 2): the quotient by the denominator scales it
    sub = ETA / U / den
    if buf is None:
        d = lr * (gu / den)
        p1 = p - d
        out['p'] = (p1, np.abs(p1) + DELTA_C['rmsprop'] * np.abs(d) + lr * sub)
        return out
    b, m = f64(buf), float(np.float32(mu))
    den_own = np.sqrt(v1 + e) if mistake == 'eps_in_sqrt' else np.sqrt(v if mistake == 'old_v' else v1) + e
    q = gu / den_own
    if mistake == 'lr_in_momentum':
        # the buffer holds lr_prev (mu buf + q) of the steps before: buf' = mu buf_folded + lr q, p -= buf'
        lp = float(np.float32(lr_prev if lr_prev is not None else lr))
        b1 = (m * lp * b + lr * q) / lr
    else:
        b1 = m * b + q
    out['buf'] = (b1, m * np.abs(b) + np.abs(q) + ETA / U / den_own)
    bu = b1 if buf_k is None else f64(buf_k)
    d = lr * bu
    p1 = p - d
    out['p'] = (p1, np.abs(p1) + DELTA_C['momentum'] * np.abs(d))
    return out


def adam_bias(b1, b2, t, mistake=None):
    """1 / (1 - b1^t) and 1 / sqrt(1 - b2^t) in fp64 of the float betas"""
    if mistake == 'bias_t_plus_1':
        t = t + 1
    b1, b2 = float(np.float32(b1)), float(np.float32(b2))
    i1 = 1.0 / (1.0 - b1 ** t)
    i2 = 1.0 if mistake == 'bias_no_second' else 1.0 / np.sqrt(1.0 - b2 ** t)
    return i1, i2


def adam(p, g, m, v, c, lr, b1, b2, eps, t, m_k=None, v_k=None, lr_prev=None, mistake=None):
    """torch.optim.Adam on the clipped gradient g c at the 1-based step t -> {'m', 'v', 'p'}: (value, S) pairs; p' on m_k / v_k (the
    kernel's own; None: this function's)"""
    p, m, v = f64(p), f64(m), f64(v)
    B1, B2, e, lr = float(np.float32(b1)), float(np.float32(b2)), float(np.float32(eps)), float(np.float32(lr))
    if mistake == 'lr_prev_step' and lr_prev is not None:
        lr = float(np.float32(lr_prev))
    gv, gu = _gk(g, c, mistake, 'v'), _gk(g, c, mistake, 'update')
    m1 = B1 * m + one_minus(b1) * gu
    v1 = B2 * v + one_minus(b2) * gv * gv
    out = {'m': (m1, B1 * np.abs(m) + one_minus(b1) * np.abs(gu)), 'v': (v1, B2 * np.abs(v) + one_minus(b2) * gv * gv)}
    mu_, vu = (m1 if m_k is None else f64(m_k)), (v1 if v_k is None else f64(v_k))
    if mistake == 'old_v':
        vu = v
    i1, i2 = adam_bias(b1, b2, t, mistake)
    den = np.sqrt(vu + e) * i2 if mistake == 'eps_in_sqrt' else np.sqrt(vu) * i2 + e
    d = (lr * i1) * (mu_ / den)
    p1 = p - d
    # an exp_avg in the subnormal range keeps only ETA absolutely: the quotient by the denominator scales it
    out['p'] = (p1, np.abs(p1) + DELTA_C['adam'] * np.abs(d) + lr * i1 * ETA / U / den)
    return out


# ------------------------------------------------------------------------------------------------ comparisons
# max |got - ref| / (c (U S + ETA)), and how far a mistake moves the reference in those units; an output NaN on both sides agrees (a
# NaN gradient poisons the kernel's weights and the reference's alike)
ratio = functools.partial(E.ratio, eta=ETA, nan_equal=True)
sensitivity = functools.partial(E.sensitivity, eta=ETA, nan_equal=True)


def loose(v, S, c):
    """the fraction of the elements in fp32's normal range whose bound is at least |v|, and the median bound / |v| (a value below
    2^-126 has only an absolute accuracy in fp32: the ETA term of its bound)"""
    v, b = np.abs(f64(v)), c * (U * f64(S) + ETA)
    nz = v >= 2.0 ** -126
    if not nz.any():
        return 0.0, 0.0
    return float((b[nz] >= v[nz]).mean()), float(np.median(b[nz] / v[nz]))


# ------------------------------------------------------------------------------------------------ inputs
BIG = 1.0e4           # the marked elements: large enough to move the norm of a 3.4 M-float gradient by far more than its bound
HP = {'rmsprop': dict(lr=1e-3, a=0.99, b=0.0, eps=1e-5), 'adam': dict(lr=1e-3, a=0.9, b=0.999, eps=1e-8)}
MOMENTUM = 0.9
SCHEDULE = dict(frames_per_step=20.0, total_frames=63.0, lr_end=2e-4)      # the linear schedule reaches its floor at step 4


def marked(n, blocks):
    """the indices a dropped index shows at: the n % 4 tail, and the first and last element of every span of `stride` float4s
    (the HOLD slots and each iteration of the loop past them)"""
    n4, stride = n // 4, blocks * 512
    idx = list(range(4 * n4, n))
    k = 0
    while k * stride < n4:
        idx += [4 * k * stride, 4 * min((k + 1) * stride, n4) - 1]
        k += 1
    return np.unique(np.array([i for i in idx if 0 <= i < n], dtype=np.int64))


def grads(rng, n, blocks, scale=1.0):
    """float32 gradients: magnitudes log-uniform over 1e-20 .. 1e3 with random signs, 2 % zeros, 2 % -0.0 and 1 % subnormal (1e-44 ..
    1e-39), +-BIG at marked(n, blocks) (all times scale)"""
    g = 10.0 ** rng.uniform(-20, 3, n) * rng.choice([-1.0, 1.0], n)
    r = rng.rand(n)
    sub = (r >= 0.04) & (r < 0.05)
    g[sub] = 10.0 ** rng.uniform(-44, -39, int(sub.sum())) / scale
    g[r < 0.02] = 0.0
    g = (g * scale).astype(np.float32)
    g[(r >= 0.02) & (r < 0.04)] = np.float32(-0.0)
    mk = marked(n, blocks)
    g[mk] = (BIG * scale * rng.choice([-1.0, 1.0], mk.size)).astype(np.float32)
    return g


def state(rng, n, opt, kind):
    """float32 parameters and optimizer state: kind 'zero' (fresh state) or 'large' (v log-uniform over 1e2 .. 1e6, a nonzero
    exp_avg / momentum buffer) -> dict(p, s0, s1, buf)"""
    p = (rng.randn(n) * 0.05).astype(np.float32)
    z = np.zeros(n, np.float32)
    if kind == 'zero':
        return dict(p=p, s0=z.copy(), s1=z.copy() if opt == 'adam' else None, buf=z.copy())
    v = (10.0 ** rng.uniform(2, 6, n)).astype(np.float32)
    m = (rng.randn(n) * 10).astype(np.float32)
    if opt == 'adam':
        return dict(p=p, s0=m, s1=v, buf=None)
    return dict(p=p, s0=v, s1=None, buf=(rng.randn(n) * 1e-2).astype(np.float32))


# ------------------------------------------------------------------------------------------------ one step of a variant
# the checked outputs of each optimizer: name -> the CHECK_C key of its bound
OUTPUTS = {'rmsprop': {'square_avg': 'v', 'momentum_buffer': 'buf', 'p': 'p'}, 'adam': {'exp_avg': 'm', 'exp_avg_sq': 'v', 'p': 'p'}}


def step(opt, st, g, c, lr, t, mu=MOMENTUM, own=None, lr_prev=None, mistake=None):
    """one step of `opt` ('rmsprop' with momentum when st['buf'] is not None, or 'adam') on st = dict(p, s0, s1, buf) and the gradient
    g with clip coefficient c, lr (float32 operand) and 1-based step t.  own: the kernel's new state (s0, s1, buf), on which p' is
    evaluated.  -> {output name: (value, S, c)}"""
    hp = HP[opt]
    own = own or {}
    if opt == 'rmsprop':
        r = rmsprop(st['p'], g, st['s0'], c, lr, hp['a'], hp['eps'], buf=st['buf'], mu=mu, v_k=own.get('s0'), buf_k=own.get('buf'),
                    lr_prev=lr_prev, mistake=mistake)
        names = {'v': 'square_avg', 'buf': 'momentum_buffer', 'p': 'p'}
    else:
        r = adam(st['p'], g, st['s0'], st['s1'], c, lr, hp['a'], hp['b'], hp['eps'], t, m_k=own.get('s0'), v_k=own.get('s1'),
                 lr_prev=lr_prev, mistake=mistake)
        names = {'m': 'exp_avg', 'v': 'exp_avg_sq', 'p': 'p'}
    return {names[k]: (val, S, CHECK_C[OUTPUTS[opt][names[k]]]) for k, (val, S) in r.items()}


# which mistakes each kind of output can show
OUTPUT_MISTAKES = {'rmsprop': ('eps_in_sqrt', 'unclipped_update', 'unclipped_v', 'old_v', 'lr_in_momentum', 'lr_prev_step'),
                   'adam': ('eps_in_sqrt', 'unclipped_update', 'unclipped_v', 'old_v', 'bias_t_plus_1', 'bias_no_second', 'lr_prev_step')}
NORM_MISTAKES = ('norm_no_tail', 'norm_no_hold_slot')

# the witness of every mistake: opt, momentum, schedule, 1-based step, n (or n4 in strides of the witness's blocks: ('stride', k, d)
# = k stride + d float4s, then n % 4), state kind, max_norm ('clip': a third of the norm; -1: none), gradient scale
WITNESS = {
    'eps_in_sqrt': dict(opt='rmsprop', mom=False, sched='constant', t=1, n=4099, state='zero', max_norm=-1.0, scale=1.0),
    'unclipped_update': dict(opt='rmsprop', mom=True, sched='constant', t=2, n=4099, state='large', max_norm='clip', scale=1.0),
    'unclipped_v': dict(opt='rmsprop', mom=False, sched='constant', t=1, n=4099, state='zero', max_norm='clip', scale=1.0),
    'bias_t_plus_1': dict(opt='adam', mom=False, sched='constant', t=1, n=4099, state='zero', max_norm=40.0, scale=1.0),
    'bias_no_second': dict(opt='adam', mom=False, sched='linear', t=2, n=4099, state='large', max_norm='clip', scale=1.0),
    'old_v': dict(opt='adam', mom=False, sched='constant', t=1, n=4099, state='zero', max_norm=-1.0, scale=1.0),
    'lr_in_momentum': dict(opt='rmsprop', mom=True, sched='linear', t=3, n=4099, state='large', max_norm=40.0, scale=1.0),
    'lr_prev_step': dict(opt='adam', mom=False, sched='linear', t=2, n=4099, state='large', max_norm=-1.0, scale=1.0),
    'clip_no_1e6': dict(opt='rmsprop', mom=False, sched='constant', t=1, n=4099, state='zero', max_norm='clip', scale=1e-9),
    'norm_no_tail': dict(opt='adam', mom=False, sched='constant', t=1, n=(1, 5, 3), state='zero', max_norm=40.0, scale=1.0),
    'norm_no_hold_slot': dict(opt='rmsprop', mom=True, sched='linear', t=1, n=(2, -1, 0), state='zero', max_norm='clip', scale=1.0),
}


def n_of(spec, blocks):
    """n of a case: an int, or (k, d, r) = 4 (k blocks 512 + d) + r"""
    if isinstance(spec, int):
        return spec
    k, d, r = spec
    return 4 * (k * blocks * 512 + d) + r


def max_norm_of(spec, g):
    """the float max_norm of a case: 'clip' is a third of the fp64 norm of g"""
    if spec == 'clip':
        return float(np.float32(np.sqrt((f64(g) ** 2).sum()) / 3))
    return float(spec)


def lr_of(opt, sched, t):
    """the float32 lr of step t under the case's schedule"""
    lr = HP[opt]['lr']
    if sched == 'constant':
        return np.float32(lr)
    return lr_at(lr, t, 'linear', SCHEDULE['frames_per_step'], SCHEDULE['total_frames'], SCHEDULE['lr_end'])


def mistake_sensitivity(mistake, opt, st, g, c, norm, max_norm, blocks, fused, t, lr, lr_prev, own=None, norm_k=None):
    """how far `mistake` moves the references of one step, in bounds: the norm mistakes on the sum of squares, clip_no_1e6 on the
    coefficient (in units of U |c|), the others on the outputs of step()"""
    if mistake in NORM_MISTAKES:
        ref, S = sumsq(g, blocks, fused)
        return sensitivity(sumsq(g, blocks, fused, mistake)[0], ref, S, CHECK_C['sumsq'])
    if mistake == 'clip_no_1e6':
        c0 = clip_coef_ref(norm, max_norm)
        return abs(clip_coef_ref(norm, max_norm, mistake) - c0) / (U * abs(c0)) if c0 else 0.0
    ref = step(opt, st, g, c, lr, t, own=own, lr_prev=lr_prev)
    pert = step(opt, st, g, c, lr, t, own=own, lr_prev=lr_prev, mistake=mistake)
    return max(sensitivity(pert[k][0], ref[k][0], ref[k][1], ref[k][2]) for k in ref)
