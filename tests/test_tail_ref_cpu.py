"""CPU: the fp64 references of tests/tail_ref.py, their bounds and their mistakes.
  * the fp64 V-trace equals oracle.impala_oracle.vtrace_from_importance_weights_np64 to 1e-12;
  * the fp64 dlogits / dbaseline equal float64 autograd through the reference's loss statements (oracle.impala_oracle.impala_losses);
  * the fp32 CPU oracle passes every bound on every case's inputs, each stage on its own output of the stage before: the bounds are
    not too tight for a correct fp32 implementation;
  * every bound is far below the value it bounds on almost every element, so each check checks;
  * every mistake moves the reference of its witness case by at least 20x the bound on some element: the inputs exercise every term;
  * a negative or NaN clip threshold is refused by the Python front ends and the C ABI, not read as None."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import impala_oracle as O
from tests import tail_ref as R

CASES_SMALL = [n for n, c in R.IW_CASES.items() if c[1] <= 4099]


def _t(x):
    return torch.from_numpy(np.ascontiguousarray(x))


def _within(name, got, ref, S, c):
    q = R.ratio(got, ref, S, c)
    assert q <= 1.0, f'{name}: {q:.3f} x the bound'
    return q


# ------------------------------------------------------------------------------------------------ the references are right
@pytest.mark.parametrize('name', CASES_SMALL)
def test_fp64_vtrace_equals_np64_oracle(name):
    lr, g, r, v, boot = R.iw_inputs(name)
    cr, cp = R.IW_CASES[name][3]
    vs, _ = R.vtrace_vs(lr, g, r, v, boot, cr, cp)
    pg, _ = R.vtrace_pg(lr, g, r, v, boot, vs, cr, cp)
    wvs, wpg = O.vtrace_from_importance_weights_np64(lr, g, r, v, boot, cr, cp)
    for got, want in ((vs, wvs), (pg, wpg)):
        assert np.max(np.abs(got - want)) <= 1e-12 * max(1.0, np.max(np.abs(want)))


@pytest.mark.parametrize('name', ['w_T31_B5_A6', 'w_T32_B33_A18', 'w_T100_B5_A33', 'w_T1_B1_A1'])
def test_fp64_head_grads_equal_float64_autograd(name):
    (bl, tl, base, act, rew, done), hp, kernel = R.tail_case(name)
    ref = R.tail(bl, tl, base, act, rew, done, hp, kernel)
    T = tl.shape[0] - 1
    logits = _t(tl[:T]).double().requires_grad_()
    values = _t(base[:T]).double().requires_grad_()
    vs, pg = (torch.from_numpy(ref[k][0]) for k in ('vs', 'pg'))
    losses = O.impala_losses(logits, _t(act[1:]), values, vs, pg, hp['baseline_cost'], hp['entropy_cost'])
    sum(losses).backward()
    assert np.max(np.abs(ref['dlogits'][0] - logits.grad.numpy())) <= 1e-12
    assert np.max(np.abs(ref['dbaseline'][0] - values.grad.numpy())) <= 1e-12
    for k, l in zip(R.TAIL_LOSSES, losses):
        assert abs(ref[k][0] - float(l)) <= 1e-12 * max(1.0, abs(float(l)))


def test_sample_ref_is_the_inverse_cdf():
    rng = np.random.RandomState(0)
    x = rng.randn(500, 7)
    u = rng.rand(500)
    act, _, _ = R.sample_ref(x, u)
    p = np.exp(x - x.max(-1, keepdims=True))
    p /= p.sum(-1, keepdims=True)
    want = [int(np.searchsorted(np.cumsum(pi), ui, side='right')) for pi, ui in zip(p, u)]
    assert np.array_equal(act, np.minimum(want, 6))


# ------------------------------------------------------------------------------------------------ the fp32 oracle is within every bound
@pytest.mark.parametrize('name', list(R.IW_CASES))
def test_fp32_oracle_within_vtrace_bounds(name):
    lr, g, r, v, boot = R.iw_inputs(name)
    cr, cp = R.IW_CASES[name][3]
    vs32, pg32 = O.vtrace_from_importance_weights(*(_t(a) for a in (lr, g, r, v, boot)), cr, cp)
    vs, S = R.vtrace_vs(lr, g, r, v, boot, cr, cp)
    _within('vs', vs32, vs, S, R.CHECK_C['vs'])
    pg, S = R.vtrace_pg(lr, g, r, v, boot, vs32, cr, cp)
    _within('pg', pg32, pg, S, R.CHECK_C['pg'])


@pytest.mark.parametrize('name', list(R.LOGITS_CASES))
def test_fp32_oracle_within_from_logits_bounds(name):
    bl, tl, act, g, r, v, boot = R.logits_inputs(name)
    A = tl.shape[-1]
    a = R.clamp_actions(act, A)
    cr, cp = R.LOGITS_CASES[name][4]
    vs32, pg32, lr32, balp32, talp32 = O.vtrace_from_logits(*(_t(x) for x in (bl, tl, a, g, r, v, boot)), cr, cp)
    tr, br = R.rows(tl), R.rows(bl)
    _within('talp', talp32, R.gather(tr['lp'], a), R.gather(tr['s_lp'], a), R.CHECK_C['logp'])
    _within('balp', balp32, R.gather(br['lp'], a), R.gather(br['s_lp'], a), R.CHECK_C['logp'])
    lr = R.gather(tr['lp'], a) - R.gather(br['lp'], a)
    _within('log_rhos', lr32, lr, R.gather(tr['s_lp'], a) + R.gather(br['s_lp'], a) + np.abs(lr), R.CHECK_C['log_rhos'])
    vs, S = R.vtrace_vs(lr32, g, r, v, boot, cr, cp)
    _within('vs', vs32, vs, S, R.CHECK_C['vs'])
    pg, S = R.vtrace_pg(lr32, g, r, v, boot, vs32, cr, cp)
    _within('pg', pg32, pg, S, R.CHECK_C['pg'])


def _oracle_tail(bl, tl, base, act, rew, done, hp):
    """the fp32 CPU oracle's tail, stage by stage, as the reference writes it (impala_atari.py:293-330)"""
    T = tl.shape[0] - 1
    A = tl.shape[-1]
    bl, tl, base, rew = (_t(x) for x in (bl, tl, base, rew))
    a = _t(R.clamp_actions(act, A))[1:]
    r = torch.clamp(rew[1:], -1, 1) if hp['clip_reward'] else rew[1:]
    g = (~_t(done)[1:]).float() * hp['discounting']
    vs, pg, *_ = O.vtrace_from_logits(bl[1:], tl[:T], a, g, r, base[:T], base[T], hp['clip_rho'], hp['clip_pg'])
    l = O.impala_losses(tl[:T], a, base[:T], vs, pg, hp['baseline_cost'], hp['entropy_cost'])
    dl, db = O.head_grads(tl[:T], a, base[:T], vs, pg, hp['baseline_cost'], hp['entropy_cost'])
    return {'vs': vs, 'pg': pg, 'dlogits': dl, 'dbaseline': db, 'loss_pg': l[0], 'loss_baseline': l[1], 'loss_entropy': l[2],
            'total': l[0] + l[1] + l[2]}


def _learner_case(shape):
    T, B, A = shape
    costs, kernel, _ = R.LEARNER_CASES[shape]
    hp = dict(R.COSTS[costs], clip_reward=True)
    return R.tail_inputs(T, B, A, 'u3', 'p05', seed=T + B + A), hp, ('column' if kernel.startswith('column') else kernel)


@pytest.mark.parametrize('name', list(R.TAIL_CASES) + [f'learner_{t}_{b}_{a}' for t, b, a in R.LEARNER_CASES])
def test_fp32_oracle_within_tail_bounds(name):
    if name.startswith('learner_'):
        inputs, hp, kernel = _learner_case(tuple(int(v) for v in name.split('_')[1:]))
    else:
        inputs, hp, kernel = R.tail_case(name)
    got = _oracle_tail(*inputs, hp)
    own = R.tail(*inputs, hp, kernel)
    ref = R.tail(*inputs, hp, kernel, vs_k=got['vs'], pg_k=got['pg'])
    _within('vs', got['vs'], *own['vs'], R.CHECK_C['vs'])
    for k in ('pg', 'dlogits', 'dbaseline') + R.TAIL_LOSSES:
        _within(k, got[k], *ref[k], R.CHECK_C[R.TAIL_CHECK_C[k]])


@pytest.mark.parametrize('A', [1, 2, 18, 100])
@pytest.mark.parametrize('regime', R.LOGIT_REGIMES)
def test_fp32_torch_within_row_bounds(A, regime):
    rng = np.random.RandomState(A)
    x = R.logit_rows(rng, (129, A), regime)
    act = rng.randint(0, A, size=129)
    wl, we = rng.randn(129).astype(np.float32), rng.randn(129).astype(np.float32)
    xt = _t(x).requires_grad_()
    lp = torch.log_softmax(xt, -1)
    logp = lp.gather(-1, _t(act)[:, None])[:, 0]
    ent = (lp.exp() * lp).sum(-1)
    (logp * _t(wl) + ent * _t(we)).sum().backward()
    rw = R.rows(x)
    _within('logp', logp.detach(), R.gather(rw['lp'], act), R.gather(rw['s_lp'], act), R.CHECK_C['logp'])
    _within('entropy', ent.detach(), rw['ent'], rw['s_ent'], R.CHECK_C['entropy'])
    d, S = R.policy_grad(rw, act, wl, we)
    _within('dlogits', xt.grad, d, S, R.CHECK_C['dlogits'])


@pytest.mark.parametrize('n,square', [(1025, False), (1 << 20, True), ((1 << 20) + 7, False)])
def test_fp32_sequential_sum_within_reduce_bound(n, square):
    """a plain sequential fp32 sum is a worse order than reduce_sum_kernel's tree: its chain is n long, so the bound with n_chain = n
    must hold for it"""
    x = np.random.RandomState(n).randn(n).astype(np.float32) + 1
    t = x * x if square else x
    s32 = np.float32(0)
    for c in np.array_split(t, 1024):           # 1024 sequential partials, then a sequential sum of them
        s32 = np.float32(s32 + np.cumsum(c, dtype=np.float32)[-1])
    val, S = R.reduce_sum(x, square, 1.0)
    chain = -(-n // 1024) + 1024 + 2
    assert abs(float(s32) - val) <= R.CHECK_C['reduce_sum'] * R.U * S * chain / R.n_chain_reduce(n, square)


# ------------------------------------------------------------------------------------------------ every bound checks its elements
def _loose(v, S, c):
    """the fraction of nonzero elements whose bound is at least |v| (there the check would pass 0 or 2v), and the median bound / |v|"""
    v, b = np.abs(R.f64(v)), c * (R.U * R.f64(S) + R.ETA)
    nz = v > 0
    if not nz.any():                 # all zero (one action, or a zero cost): nothing a bound could let through
        return 0.0, 0.0
    return float((b[nz] >= v[nz]).mean()), float(np.median(b[nz] / v[nz]))


TIGHT_CASES = [('iw', n) for n in CASES_SMALL] + [('logits', n) for n in R.LOGITS_CASES] + [('tail', n) for n in R.TAIL_CASES]


@pytest.mark.parametrize('table,name', TIGHT_CASES)
def test_bounds_are_far_below_the_values(table, name):
    """a bound as large as the value it bounds checks nothing: vs and pg (and the tail's dlogits and dbaseline) must have bounds below
    |value| on at least 95 % of their nonzero elements, and at most 1e-2 |value| on the median one"""
    if table == 'iw':
        lr, g, r, v, boot = R.iw_inputs(name)
        cr, cp = R.IW_CASES[name][3]
        vs, S = R.vtrace_vs(lr, g, r, v, boot, cr, cp)
        out = {'vs': (vs, S), 'pg': R.vtrace_pg(lr, g, r, v, boot, vs, cr, cp)}
    elif table == 'logits':
        bl, tl, act, g, r, v, boot = R.logits_inputs(name)
        a = R.clamp_actions(act, tl.shape[-1])
        lr = R.gather(R.rows(tl)['lp'], a) - R.gather(R.rows(bl)['lp'], a)
        cr, cp = R.LOGITS_CASES[name][4]
        vs, S = R.vtrace_vs(lr, g, r, v, boot, cr, cp)
        out = {'vs': (vs, S), 'pg': R.vtrace_pg(lr, g, r, v, boot, vs, cr, cp)}
    else:
        inputs, hp, kernel = R.tail_case(name)
        out = {k: v for k, v in R.tail(*inputs, hp, kernel).items() if k in ('vs', 'pg', 'dlogits', 'dbaseline')}
    for k, (val, S) in out.items():
        frac, med = _loose(val, S, R.CHECK_C[R.TAIL_CHECK_C[k]])
        assert frac <= 0.05 and med <= 1e-2, f'{k}: the bound is >= |value| on {100 * frac:.1f} % of elements, median bound / |value| {med:.2e}'


# ------------------------------------------------------------------------------------------------ every mistake is visible
def _iw_sens(name, mistake):
    lr, g, r, v, boot = R.iw_inputs(name)
    cr, cp = R.IW_CASES[name][3]
    vs, Svs = R.vtrace_vs(lr, g, r, v, boot, cr, cp)
    pg, Spg = R.vtrace_pg(lr, g, r, v, boot, vs, cr, cp)
    pvs, _ = R.vtrace_vs(lr, g, r, v, boot, cr, cp, mistake=mistake)
    ppg, _ = R.vtrace_pg(lr, g, r, v, boot, vs, cr, cp, mistake=mistake)
    return max(R.sensitivity(pvs, vs, Svs, R.CHECK_C['vs']), R.sensitivity(ppg, pg, Spg, R.CHECK_C['pg']))


def _tail_sens(name, mistake):
    inputs, hp, kernel = R.tail_case(name)
    own = R.tail(*inputs, hp, kernel)
    vs, pg = own['vs'][0], own['pg'][0]
    ref = R.tail(*inputs, hp, kernel, vs_k=vs, pg_k=pg)
    pert = R.tail(*inputs, hp, kernel, vs_k=vs, pg_k=pg, mistake=mistake)
    best = R.sensitivity(R.tail(*inputs, hp, kernel, mistake=mistake)['vs'][0], vs, own['vs'][1], R.CHECK_C['vs'])
    for k in ('pg', 'dlogits', 'dbaseline') + R.TAIL_LOSSES:
        best = max(best, R.sensitivity(pert[k][0], ref[k][0], ref[k][1], R.CHECK_C[R.TAIL_CHECK_C[k]]))
    return best


WITNESSES = [('iw', n, m) for n, c in R.IW_CASES.items() for m in c[8]] + \
            [('tail', n, m) for n, c in R.TAIL_CASES.items() for m in c[7]]


def test_every_mistake_has_a_witness():
    assert {m for _, _, m in WITNESSES} == set(R.MISTAKES)


@pytest.mark.parametrize('table,name,mistake', WITNESSES)
def test_mistake_moves_its_witness(table, name, mistake):
    s = (_iw_sens if table == 'iw' else _tail_sens)(name, mistake)
    assert s >= R.SENS, f'{mistake} ({R.MISTAKES[mistake]}) moves {name} by only {s:.1f} x the bound'


# ------------------------------------------------------------------------------------------------ clip thresholds
@pytest.mark.parametrize('bad', [-0.5, -1.0, float('nan')])
def test_bad_clip_threshold_is_refused(bad):
    from scalerl_b200 import _lib, ops
    from scalerl_b200.learner import ImpalaHParams
    assert ops._clip(None) == -1.0 and ops._clip(0) == 0.0 and ops._clip(2) == 2.0
    with pytest.raises(ValueError):
        ops._clip(bad)
    for field in ('clip_rho_threshold', 'clip_pg_rho_threshold'):
        hp = ImpalaHParams(**{field: bad})
        with pytest.raises(ValueError):
            hp.validate()
        with pytest.raises(ValueError):
            hp.to_c()
    if not math.isnan(bad):
        return
    # the C ABI keeps "< 0 means None" but refuses NaN, before it reads any pointer
    L = _lib.lib()
    for clips in ((bad, 1.0), (1.0, bad)):
        rc = L.srl_vtrace_from_importance_weights(None, None, None, None, None, 1, 1, *clips, None, None, 0, None)
        assert rc == -1 and b'NaN' in L.srl_last_error()
        rc = L.srl_vtrace_from_logits(None, None, None, None, None, None, None, 1, 1, 2, *clips, None, None, None, None, None, None)
        assert rc == -1 and b'NaN' in L.srl_last_error()
        rc = L.srl_impala_loss_and_head_grads(None, None, None, None, None, None, 1, 1, 2, 0.99, 1, *clips, 0.5, 0.01, None, None, None,
                                              None, None, None, None)
        assert rc == -1 and b'NaN' in L.srl_last_error()
        c = ImpalaHParams().to_c()
        c.clip_rho_threshold, c.clip_pg_rho_threshold = clips
        h = ctypes.c_void_p()
        rc = L.srl_learner_create(ctypes.byref(c), None, None, None, None, ctypes.byref(h))
        assert rc == -1 and b'NaN' in L.srl_last_error()
