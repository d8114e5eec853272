"""CPU: the fp64 references of tests/optim_ref.py, their bounds and their mistakes.
  * the references equal torch.optim.RMSprop (momentum 0 and 0.9), torch.optim.Adam, clip_grad_norm_ and LambdaLR run in float64,
    to 1e-12, over several steps;
  * the same torch optimizers in fp32 stay within every bound, each step on torch's own clip coefficient and new state, and
    clip_grad_norm_'s fp32 coefficient is within one ulp of optim_ref.clip_coef32 on its own norm;
  * every bound is far below the value it bounds on almost every element, so each check checks;
  * every mistake moves its witness case by at least 20x the bound;
  * the non-finite cases: one NaN gradient poisons every clipped gradient, an Inf one gives the coefficient 0, and the snapshot
    copies exactly when the total loss is finite."""
import math

import numpy as np
import pytest
import torch

from tests import optim_ref as R

N = 4099
BLOCKS = 4               # the nominal grid of the CPU cases: stride 2048 float4s


def _case(opt, kind, seed, scale=1.0, n=N):
    rng = np.random.RandomState(seed)
    return R.grads(rng, n, BLOCKS, scale), R.state(rng, n, opt, kind)


def _torch_opt(opt, params, mom, dtype, lr):
    hp = R.HP[opt]
    f = lambda v: float(np.float32(v))
    if opt == 'rmsprop':
        return torch.optim.RMSprop(params, lr=f(lr), alpha=f(hp['a']), eps=f(hp['eps']), momentum=f(R.MOMENTUM) if mom else 0.0)
    return torch.optim.Adam(params, lr=f(lr), betas=(f(hp['a']), f(hp['b'])), eps=f(hp['eps']))


def _load_state(opt, torch_opt, prm, st, dtype, t):
    """put st's optimizer state (after t - 1 steps) into torch's"""
    if t == 1 and not (st['s0'] != 0).any():
        return
    s = torch_opt.state[prm]
    s['step'] = torch.tensor(float(t - 1), dtype=torch.float32)
    if opt == 'rmsprop':
        s['square_avg'] = torch.from_numpy(st['s0'].astype(dtype))
        if st['buf'] is not None:
            s['momentum_buffer'] = torch.from_numpy(st['buf'].astype(dtype))
    else:
        s['exp_avg'], s['exp_avg_sq'] = torch.from_numpy(st['s0'].astype(dtype)), torch.from_numpy(st['s1'].astype(dtype))


def _torch_step(opt, mom, g, st, max_norm, dtype, lr, t):
    """clip_grad_norm_(max_norm) (not called for max_norm < 0 or +inf: no clip) + one step of the torch optimizer in `dtype` from st
    at the 1-based step t -> (norm or None, the clipped gradient, the new state)"""
    prm = torch.nn.Parameter(torch.from_numpy(st['p'].astype(dtype)))
    o = _torch_opt(opt, [prm], mom, dtype, lr)
    _load_state(opt, o, prm, st, dtype, t)
    prm.grad = torch.from_numpy(g.astype(dtype))
    norm = float(torch.nn.utils.clip_grad_norm_([prm], max_norm)) if max_norm >= 0 and not math.isinf(max_norm) else None
    clipped = prm.grad.clone()
    o.step()
    s = o.state[prm]
    new = {'p': prm.detach().numpy().copy()}
    if opt == 'rmsprop':
        new['s0'] = s['square_avg'].numpy().copy()
        new['buf'] = s['momentum_buffer'].numpy().copy() if mom else None
    else:
        new['s0'], new['s1'] = s['exp_avg'].numpy().copy(), s['exp_avg_sq'].numpy().copy()
    return norm, clipped.numpy(), new


def _state64(st):
    return {k: (None if v is None else v.astype(np.float64)) for k, v in st.items()}


# ------------------------------------------------------------------------------------------------ the references are right
@pytest.mark.parametrize('opt,mom', [('rmsprop', False), ('rmsprop', True), ('adam', False)])
@pytest.mark.parametrize('max_norm', [40.0, 'clip', -1.0])
def test_fp64_refs_equal_torch_float64(opt, mom, max_norm):
    """three steps of the reference and of torch in float64 from a 'large' state, the lr of each step set to the float32 schedule"""
    g, st = _case(opt, 'large', 11)
    if not mom:
        st['buf'] = None
    mn = R.max_norm_of(max_norm, g)
    cur = _state64(st)
    for t in range(1, 4):
        lr = float(R.lr_of(opt, 'linear', t))
        gt = g * np.float32(0.5 + t)
        norm, _, new = _torch_step(opt, mom, gt, cur, mn, np.float64, lr, t + 5)
        s2, _ = R.sumsq(gt, BLOCKS)
        if norm is not None:
            assert abs(math.sqrt(s2) - norm) <= 1e-12 * norm
        c = R.clip_coef_ref(math.sqrt(s2), mn)
        if norm is not None:
            assert abs(c - min(mn / (norm + 1e-6), 1.0)) <= 1e-12
        ref = R.step(opt, cur, gt, c, lr, t + 5)
        want = {'p': new['p'], 'square_avg': new.get('s0'), 'momentum_buffer': new.get('buf'), 'exp_avg': new.get('s0'),
                'exp_avg_sq': new.get('s1')}
        for k, (val, _, _) in ref.items():
            w = want[k]
            assert np.max(np.abs(val - w)) <= 1e-12 * max(1.0, np.max(np.abs(w))), (k, t)
        cur = {'p': new['p'], 's0': new['s0'], 's1': new.get('s1'), 'buf': new.get('buf')}


def test_schedule_equals_lambdalr_float64():
    """the linear schedule's lr of steps 1..8 is LambdaLR's (stepped after every optimizer step) to 1e-12, and lr_at rounds it once"""
    from scalerl_b200.learner import scheduled_lr
    hp, sc = R.HP['adam'], R.SCHEDULE
    lr = float(np.float32(hp['lr']))
    end = float(np.float32(sc['lr_end']))
    prm = torch.nn.Parameter(torch.zeros(3, dtype=torch.float64))
    o = torch.optim.SGD([prm], lr=lr)
    F, tot = sc['frames_per_step'], sc['total_frames']
    sched = torch.optim.lr_scheduler.LambdaLR(o, lambda e: max(1 - min(e * F, tot) / tot, end / lr))
    for t in range(1, 9):
        want = o.param_groups[0]['lr']
        got = scheduled_lr(lr, 'linear', t, F, tot, end)
        assert abs(got - want) <= 1e-12 * lr, (t, got, want)
        assert R.lr_of('adam', 'linear', t) == np.float32(got)
        o.step()
        sched.step()
    assert R.lr_of('adam', 'linear', 8) == np.float32(end) and R.lr_of('adam', 'constant', 8) == np.float32(lr)


# ------------------------------------------------------------------------------------------------ fp32 torch is within every bound
@pytest.mark.parametrize('opt,mom', [('rmsprop', False), ('rmsprop', True), ('adam', False)])
@pytest.mark.parametrize('kind', ['zero', 'large'])
@pytest.mark.parametrize('max_norm', [40.0, 'clip', 0.0, -1.0])
def test_fp32_torch_within_bounds(opt, mom, kind, max_norm):
    g, st = _case(opt, kind, 3 + len(kind))
    if not mom:
        st['buf'] = None
    mn = R.max_norm_of(max_norm, g)
    for t in (1, 2, 10 ** 6):
        norm, clipped, new = _torch_step(opt, mom, g, st, mn, np.float32, float(R.HP[opt]['lr']), t)
        if norm is None:
            c = np.float32(1.0)
        else:
            # torch forms the coefficient on 0-dim tensors: within one ulp of the kernel's fp32 evaluation on the same norm
            c = torch.clamp(mn / (torch.tensor(norm, dtype=torch.float32) + 1e-6), max=1.0).numpy()
            assert abs(int(c.view(np.int32)) - int(R.clip_coef32(np.float32(norm), mn).view(np.int32))) <= 1
            assert np.array_equal(clipped.view(np.int32), (g * c).astype(np.float32).view(np.int32)), 'the clipped gradient is g * c in fp32'
            s2, S = R.sumsq(g, 1, fused=False)
            # torch's norm is a different order of the same sum: a chain of at most n squares and adds, bounded with n_chain = n
            assert abs(float(np.float32(norm)) ** 2 - s2) <= R.CHECK_C['sumsq'] * R.U * (g.size + 2) * s2
        own = {'s0': new['s0'], 's1': new.get('s1'), 'buf': new.get('buf')}
        ref = R.step(opt, st, g, c, np.float32(R.HP[opt]['lr']), t, own=own)
        got = {'p': new['p'], 'square_avg': new['s0'], 'momentum_buffer': new.get('buf'), 'exp_avg': new['s0'], 'exp_avg_sq': new.get('s1')}
        for k, (val, S, cc) in ref.items():
            q = R.ratio(got[k], val, S, cc)
            assert q <= 1.0, f'{k} at t={t}: {q:.3f} x the bound'


# ------------------------------------------------------------------------------------------------ every bound checks its elements
@pytest.mark.parametrize('opt,mom', [('rmsprop', False), ('rmsprop', True), ('adam', False)])
@pytest.mark.parametrize('kind', ['zero', 'large'])
@pytest.mark.parametrize('max_norm', [40.0, 'clip'])
def test_bounds_are_far_below_the_values(opt, mom, kind, max_norm):
    """below |value| on at least 95 % of the nonzero elements, and at most 1e-2 |value| on the median one"""
    g, st = _case(opt, kind, 5)
    if not mom:
        st['buf'] = None
    mn = R.max_norm_of(max_norm, g)
    c = R.clip_coef32(np.float32(np.sqrt(R.sumsq(g, BLOCKS)[0])), mn)
    for t in (1, 2):
        for k, (val, S, cc) in R.step(opt, st, g, c, np.float32(R.HP[opt]['lr']), t).items():
            frac, med = R.loose(val, S, cc)
            assert frac <= 0.05 and med <= 1e-2, f'{k}: the bound is >= |value| on {100 * frac:.1f} % of elements, median {med:.2e}'
    s2, S = R.sumsq(g, BLOCKS)
    assert R.CHECK_C['sumsq'] * R.U * S <= 1e-4 * s2


# ------------------------------------------------------------------------------------------------ every mistake is visible
def witness_sensitivity(mistake):
    """the sensitivity of `mistake` on its witness case, evaluated as the GPU suite evaluates it"""
    w = R.WITNESS[mistake]
    opt, t = w['opt'], w['t']
    n = R.n_of(w['n'], BLOCKS)
    rng = np.random.RandomState(sum(map(ord, mistake)))
    g = R.grads(rng, n, BLOCKS, w['scale'])
    st = R.state(rng, n, opt, w['state'])
    if not w['mom']:
        st['buf'] = None
    mn = R.max_norm_of(w['max_norm'], g)
    norm = np.float32(np.sqrt(R.sumsq(g, BLOCKS)[0]))
    c = R.clip_coef32(norm, mn)
    lr = R.lr_of(opt, w['sched'], t)
    lr_prev = R.lr_of(opt, w['sched'], t - 1) if t > 1 else None
    return R.mistake_sensitivity(mistake, opt, st, g, c, float(norm), mn, BLOCKS, True, t, lr, lr_prev)


def test_every_mistake_has_a_witness():
    assert set(R.WITNESS) == set(R.MISTAKES)


@pytest.mark.parametrize('mistake', list(R.MISTAKES))
def test_mistake_moves_its_witness(mistake):
    s = witness_sensitivity(mistake)
    assert s >= R.SENS, f'{mistake} ({R.MISTAKES[mistake]}) moves its witness by only {s:.1f} x the bound'


def test_lr_in_momentum_shows_over_steps_of_the_linear_schedule():
    """folding lr into the buffer is exact while lr is constant; over three steps of the linear schedule it moves p"""
    rng = np.random.RandomState(7)
    g = R.grads(rng, N, BLOCKS)
    st = R.state(rng, N, 'rmsprop', 'zero')
    hp = R.HP['rmsprop']
    p, v, b, folded = (R.f64(st[k]) for k in ('p', 's0', 'buf', 'buf'))
    pf = p.copy()
    vf = v.copy()
    a = float(np.float32(hp['a']))
    for t in (1, 2, 3):
        lr = float(R.lr_of('rmsprop', 'linear', t))
        r = R.rmsprop(p, g, v, 1.0, lr, hp['a'], hp['eps'], buf=b, mu=R.MOMENTUM)
        p, v, b = r['p'][0], r['v'][0], r['buf'][0]
        vf = a * vf + R.one_minus(hp['a']) * R.f64(g) ** 2
        folded = float(np.float32(R.MOMENTUM)) * folded + lr * (R.f64(g) / (np.sqrt(vf) + float(np.float32(hp['eps']))))
        pf = pf - folded
    assert R.sensitivity(pf, p, r['p'][1], R.CHECK_C['p']) >= R.SENS


# ------------------------------------------------------------------------------------------------ non-finite inputs
def test_nan_and_inf_gradients_follow_torch():
    g = np.linspace(-1, 1, 16).astype(np.float32)
    for bad, want_c in ((np.nan, np.nan), (np.inf, 0.0), (-np.inf, 0.0)):
        x = g.copy()
        x[5] = bad
        t = torch.from_numpy(x.copy())
        prm = torch.nn.Parameter(torch.zeros(16))
        prm.grad = t
        norm = float(torch.nn.utils.clip_grad_norm_([prm], 40.0))
        c = R.clip_coef32(np.float32(norm), 40.0)
        assert (np.isnan(c) and np.isnan(want_c)) or c == want_c
        want = (x * c).astype(np.float32)
        assert np.array_equal(np.isnan(prm.grad.numpy()), np.isnan(want)) and np.array_equal(prm.grad.numpy()[~np.isnan(want)], want[~np.isnan(want)])
    assert R.clip_coef32(np.float32(np.nan), -1.0) == 1.0 and R.clip_coef32(np.float32(np.nan), np.inf) == 1.0
    assert R.clip_coef32(np.float32(np.inf), np.inf) == 1.0


def test_snapshot_contract():
    big = float(np.float32(3.3e38))
    for loss, copies in ((np.nan, False), (np.inf, False), (-np.inf, False), (big, True), (-big, True), (1.5, True)):
        assert R.snapshot_copies([0, 0, 0, loss]) == copies, loss
    assert R.snapshot_copies(None)
