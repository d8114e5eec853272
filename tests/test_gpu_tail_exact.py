"""Every kernel of csrc/vtrace.cu against an fp64 evaluation of its own operation (tests/tail_ref.py), element by element, on the operands
the GPU itself read, at every dispatch edge of the V-trace kernels, the fused loss tail, the learner's column kernel and the row operators.

  * Each stage is checked on the GPU's own output of the stage before it: pg on the kernel's vs, dlogits and the pg loss on the kernel's
    pg, dbaseline and the baseline loss on the kernel's vs, from_logits' vs / pg on its own log_rhos.  So every bound is local.
  * Every bound is per element, c * 2^-24 * S, S the fp64 sum of the |terms| that reach the output; c is tail_ref.CHECK_C.  Each of the
    four losses is checked on its own.
  * Sensitivity: each check records how far the mistakes of tail_ref.MISTAKES that it can show move its reference, in bounds; every
    case requires at least 20x for the mistakes it is a witness of.
  * Which kernel runs: each case of a dispatching entry point (V-trace, from_logits, the tails, the learner) asserts with
    torch.profiler that the kernel it is meant to reach ran.  The row operators, reduce_sum and sample_actions launch one kernel each.
  * The learner at each tail boundary (bf16, learning rate 0): its vs, pg, dlogits and dbaseline equal the stand-alone tail's on its own
    logits / baseline bit for bit, and everything, the losses included, is within the fp64 bounds.
  * sample_actions: with given uniforms every row whose fp64 target lies farther than the bound from each CDF boundary picks the fp64
    action; the other rows are counted (<= 0.1 %); no row picks an action whose probability is 0 in fp32.  Without uniforms: the first
    maximal index, ties built in.

The worst err / bound of every check, its margin and its sensitivity go to $SRL_RESULTS_DIR/tail_exact.json when SRL_RESULTS_DIR is
set (per case, and a summary per check)."""
import numpy as np
import pytest
import torch

from oracle import impala_oracle as O
from tests import exact as E
from tests import tail_ref as R

pytestmark = pytest.mark.gpu

RESULTS = 'tail_exact.json'
KERNELS = {'scan': 'vtrace_iw_scan_kernel', 'seq4': 'vtrace_iw_seq_kernel<4>', 'seq1': 'vtrace_iw_seq_kernel<1>',
           'logits': 'vtrace_logits_kernel', 'warp': 'impala_tail_warp_kernel', 'thread': 'impala_tail_kernel',
           'column8': 'column_step_kernel<4,8>', 'column32': 'column_step_kernel<4,32>'}
MAX_EXCLUDED = 1e-3

_summary = E.summary(RESULTS)


def _ran(fn, kernel, tries=3):
    """fn() under torch.profiler; asserts the kernel ran.  A profiler session now and then returns the runtime API records of a call
    without its kernel record, so fn (every caller's fn is deterministic and has no side effect a repeat would change) runs again
    under a new session, up to `tries` times; a kernel that does not run is missing from every one."""
    seen = set()
    for _ in range(tries):
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            out = fn()
            torch.cuda.synchronize()
        names = [e.name.replace(' ', '') for e in prof.events()]
        if any(KERNELS[kernel] in n for n in names):
            return out
        seen.update(names)
    raise AssertionError(f'{KERNELS[kernel]} did not run in {tries} profiled calls: {sorted(seen)[:12]}')


def _dev(x, offset=False):
    t = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    if not offset:
        return t
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device='cuda')
    buf[1:].copy_(t.reshape(-1))
    return buf[1:].view(t.shape)            # 4 bytes past a 16-byte boundary


def _host(t):
    return t.detach().cpu().numpy()


# ------------------------------------------------------------------------------------------------ from_importance_weights
def _vtrace_checks(Ck, lr, g, r, v, boot, cr, cp, vs, pg):
    """vs against the fp64 recursion, pg on the kernel's vs -> {mistake: sensitivity}"""
    ref_vs, S_vs = R.vtrace_vs(lr, g, r, v, boot, cr, cp)
    ref_pg, S_pg = R.vtrace_pg(lr, g, r, v, boot, vs, cr, cp)
    sens = {}
    for m in ('cbar_rho', 'clips_swapped', 'boot_zero', 'chunk_carry'):
        sens[m] = R.sensitivity(R.vtrace_vs(lr, g, r, v, boot, cr, cp, mistake=m)[0], ref_vs, S_vs, R.CHECK_C['vs'])
    sp = {m: R.sensitivity(R.vtrace_pg(lr, g, r, v, boot, vs, cr, cp, mistake=m)[0], ref_pg, S_pg, R.CHECK_C['pg'])
          for m in ('clips_swapped', 'pg_values', 'boot_zero')}
    Ck.bound('vs', vs, ref_vs, S_vs, R.CHECK_C['vs'], max(sens.values()))
    Ck.bound('pg', pg, ref_pg, S_pg, R.CHECK_C['pg'], max(sp.values()))
    for m, s in sp.items():
        sens[m] = max(sens.get(m, 0.0), s)
    return sens


@pytest.mark.parametrize('name', list(R.IW_CASES))
def test_from_importance_weights_exact(name):
    from scalerl_b200 import ops
    T, B, variant, (cr, cp), _, _, offset, kernel, witnesses, _ = R.IW_CASES[name]
    x = R.iw_inputs(name)
    d = [_dev(a, offset) for a in x]
    out = _ran(lambda: ops.from_importance_weights(*d, cr, cp, variant=variant), kernel)
    Ck = E.Checker(RESULTS, R)
    sens = _vtrace_checks(Ck, *x, cr, cp, _host(out.vs), _host(out.pg_advantages))
    Ck.require(name, sens, witnesses)
    if variant == 1 and T > 128:
        seq = ops.from_importance_weights(*d, cr, cp, variant=0)
        Ck.exact('vs_equals_variant0', out.vs, seq.vs)
        Ck.exact('pg_equals_variant0', out.pg_advantages, seq.pg_advantages)
    Ck.done(f'iw_{name}')


# ------------------------------------------------------------------------------------------------ from_logits
@pytest.mark.parametrize('name', list(R.LOGITS_CASES))
def test_from_logits_exact(name):
    from scalerl_b200 import ops
    x = R.logits_inputs(name)
    bl, tl, act, g, r, v, boot = x
    A = tl.shape[-1]
    cr, cp = R.LOGITS_CASES[name][4]
    out = _ran(lambda: ops.from_logits(*[_dev(a) for a in x], cr, cp), 'logits')
    a = R.clamp_actions(act, A)
    tr, br = R.rows(tl), R.rows(bl)
    talp, balp = R.gather(tr['lp'], a), R.gather(br['lp'], a)
    s_t, s_b = R.gather(tr['s_lp'], a), R.gather(br['s_lp'], a)
    Ck = E.Checker(RESULTS, R)
    nb = (a + 1) % A                                                          # the neighbouring action read by mistake
    sens = lambda pert, ref, S, c: R.sensitivity(pert, ref, S, c) if A > 1 else None
    Ck.bound('talp', _host(out.target_action_log_probs), talp, s_t, R.CHECK_C['logp'], sens(R.gather(tr['lp'], nb), talp, s_t, R.CHECK_C['logp']))
    Ck.bound('balp', _host(out.behavior_action_log_probs), balp, s_b, R.CHECK_C['logp'], sens(R.gather(br['lp'], nb), balp, s_b, R.CHECK_C['logp']))
    lr = talp - balp
    Ck.bound('log_rhos', _host(out.log_rhos), lr, s_t + s_b + np.abs(lr), R.CHECK_C['log_rhos'],
             sens(R.gather(tr['lp'], nb) - balp, lr, s_t + s_b + np.abs(lr), R.CHECK_C['log_rhos']))
    _vtrace_checks(Ck, _host(out.log_rhos), g, r, v, boot, cr, cp, _host(out.vs), _host(out.pg_advantages))
    Ck.done(f'logits_{name}')


# ------------------------------------------------------------------------------------------------ the fused tail
def _tail_checks(Ck, case, inputs, hp, kernel, out, witnesses):
    """out: vs, pg_advantages, dlogits, dbaseline, losses[4] of a tail on `inputs`"""
    vs, pg = _host(out['vs']), _host(out['pg_advantages'])
    own = R.tail(*inputs, hp, kernel)
    ref = R.tail(*inputs, hp, kernel, vs_k=vs, pg_k=pg)
    got = {'pg': pg, 'dlogits': _host(out['dlogits']), 'dbaseline': _host(out['dbaseline'])}
    got.update(zip(R.TAIL_LOSSES, _host(out['losses']).astype(np.float64)))
    sens = {}
    for m in R.MISTAKES:
        pert_own = R.tail(*inputs, hp, kernel, mistake=m)
        pert = R.tail(*inputs, hp, kernel, vs_k=vs, pg_k=pg, mistake=m)
        sens[m] = {'vs': R.sensitivity(pert_own['vs'][0], own['vs'][0], own['vs'][1], R.CHECK_C['vs'])}
        for k in got:
            sens[m][k] = R.sensitivity(pert[k][0], ref[k][0], ref[k][1], R.CHECK_C[R.TAIL_CHECK_C[k]])
    per_check = lambda k: max([sens[m][k] for m in R.TAIL_MISTAKES[k] if m in sens] or [0.0])
    Ck.bound('vs', vs, *own['vs'], R.CHECK_C['vs'], per_check('vs'))
    for k in got:
        Ck.bound(k, got[k], *ref[k], R.CHECK_C[R.TAIL_CHECK_C[k]], per_check(k))
    Ck.require(case, {m: max(s.values()) for m, s in sens.items()}, witnesses)


def _tail_call(inputs, hp):
    from scalerl_b200 import ops
    bl, tl, base, act, rew, done = (_dev(a) for a in inputs)
    return ops.impala_loss_and_head_grads(bl, tl, base, act, rew, done, discounting=hp['discounting'],
                                          reward_clipping='abs_one' if hp['clip_reward'] else 'none', clip_rho_threshold=hp['clip_rho'],
                                          clip_pg_rho_threshold=hp['clip_pg'], baseline_cost=hp['baseline_cost'],
                                          entropy_cost=hp['entropy_cost'])


@pytest.mark.parametrize('name', list(R.TAIL_CASES))
def test_impala_tail_exact(name):
    inputs, hp, kernel = R.tail_case(name)
    out = _ran(lambda: _tail_call(inputs, hp), kernel)
    Ck = E.Checker(RESULTS, R)
    _tail_checks(Ck, name, inputs, hp, kernel, out, R.TAIL_CASES[name][7])
    Ck.done(f'tail_{name}')


# ------------------------------------------------------------------------------------------------ the learner at each tail boundary
@pytest.mark.parametrize('T,B,A', list(R.LEARNER_CASES))
def test_learner_tail_exact(T, B, A):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    costs, kernel, _ = R.LEARNER_CASES[(T, B, A)]
    c = R.COSTS[costs]
    hp = dict(c, clip_reward=True)
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, learning_rate=0.0, precision='bf16',
                                        discounting=c['discounting'], baseline_cost=c['baseline_cost'], entropy_cost=c['entropy_cost'],
                                        clip_rho_threshold=c['clip_rho'], clip_pg_rho_threshold=c['clip_pg']),
                          init_state_dict=O.init_params(A, seed=T + A), process_group=False)
    try:
        L.set_option('column_fusion', 1)       # explicit: SRL_NO_COLUMN_FUSION in the environment would turn it off
        batch = {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=T + B + A, done_p=0.05).items()}
        batch['reward'] = torch.empty_like(batch['reward']).uniform_(-3, 3, generator=torch.Generator('cuda').manual_seed(B))
        _ran(lambda: L.forward_backward(batch), kernel)
        logits = L.debug_buffer('logits').view(T + 1, B, A).clone()
        baseline = L.debug_buffer('baseline').view(T + 1, B).clone()
        mine = {'vs': L._vs.clone(), 'pg_advantages': L._pg_adv.clone(), 'dlogits': L.debug_buffer('dlogits').view(T, B, A).clone(),
                'dbaseline': L.debug_buffer('dbaseline').view(T, B).clone(), 'losses': L._losses.clone()}
    finally:
        L.close()
    inputs = tuple(_host(t) for t in (batch['policy_logits'], logits, baseline, batch['action'], batch['reward'], batch['done']))
    alone = _tail_call(inputs, hp)
    Ck = E.Checker(RESULTS, R)
    for k in ('vs', 'pg_advantages', 'dlogits', 'dbaseline'):
        Ck.exact(f'{k}_equals_standalone', mine[k], alone[k])
    _tail_checks(Ck, f'learner {T}x{B}x{A}', inputs, hp, 'column' if kernel.startswith('column') else kernel, mine, ())
    Ck.done(f'learner_T{T}_B{B}_A{A}')


# ------------------------------------------------------------------------------------------------ row operators
@pytest.mark.parametrize('A', [1, 2, 18, 100])
@pytest.mark.parametrize('N', [1, 129, 100003])
def test_policy_rows_exact(N, A):
    from scalerl_b200 import ops
    rng = np.random.RandomState(N + A)
    Ck = E.Checker(RESULTS, R)
    for regime in R.LOGIT_REGIMES:
        x = R.logit_rows(rng, (N, A), regime)
        act = rng.randint(0, A, size=N).astype(np.int64)
        wl, we = rng.randn(N).astype(np.float32), rng.randn(N).astype(np.float32)
        xd, ad, wld, wed = _dev(x), _dev(act), _dev(wl), _dev(we)
        rw = R.rows(x)
        logp, ent = ops.policy_rows_forward(xd, ad, want_logp=True, want_entropy=True)
        off = R.gather(rw['lp'], (act + 1) % A)                              # the neighbouring action's log-prob
        s_lp = R.gather(rw['s_lp'], act)
        Ck.bound(f'logp_{regime}', _host(logp), R.gather(rw['lp'], act), s_lp, R.CHECK_C['logp'],
                 R.sensitivity(off, R.gather(rw['lp'], act), s_lp, R.CHECK_C['logp']))
        # mistakes: the entropy's sign flipped, or its sum taken over log p without the p
        s_ent = max(R.sensitivity(-rw['ent'], rw['ent'], rw['s_ent'], R.CHECK_C['entropy']),
                    R.sensitivity(rw['lp'].sum(-1), rw['ent'], rw['s_ent'], R.CHECK_C['entropy']))
        Ck.bound(f'entropy_{regime}', _host(ent), rw['ent'], rw['s_ent'], R.CHECK_C['entropy'], s_ent)
        s_logp = Ck.res[f'logp_{regime}']['sensitivity']
        if regime == 'n1' and A >= 2 and N >= 129 and min(s_ent, s_logp) < R.SENS:
            Ck.fails.append(f'{regime}: the mistakes move logp / the entropy by only {s_logp:.1f} / {s_ent:.1f} x the bound')
        only_ent = ops.policy_rows_forward(xd, None, want_logp=False, want_entropy=True)[1]
        only_logp = ops.policy_rows_forward(xd, ad, want_logp=True, want_entropy=False)[0]
        Ck.exact(f'entropy_alone_{regime}', only_ent, ent)
        Ck.exact(f'logp_alone_{regime}', only_logp, logp)
        for use_act in (False, True):
            for use_wl in ((False, True) if use_act else (False,)):
                for use_we in (False, True):
                    tag = f'dlogits_{regime}_{"a" if use_act else "-"}{"l" if use_wl else "-"}{"e" if use_we else "-"}'
                    got = ops.policy_rows_backward(xd, ad if use_act else None, wld if use_wl else None, wed if use_we else None)
                    d, S = R.policy_grad(rw, act if use_act else None, wl if use_wl else None, we if use_we else None)
                    sens = []
                    if use_we:
                        sens.append(R.sensitivity(R.policy_grad(rw, act, wl if use_wl else None, we, 'entropy_sign')[0], d, S,
                                                  R.CHECK_C['dlogits']))
                    if use_wl:
                        sens.append(R.sensitivity(R.policy_grad(rw, act, wl, we if use_we else None, 'logp_p_dropped')[0], d, S,
                                                  R.CHECK_C['dlogits']))
                    s = max(sens) if sens else None
                    Ck.bound(tag, _host(got), d, S, R.CHECK_C['dlogits'], s)
                    if s is not None and regime == 'n1' and A >= 2 and N >= 129 and s < R.SENS:
                        Ck.fails.append(f'{tag}: the mistakes move the reference by only {s:.1f} x the bound')
    Ck.done(f'rows_N{N}_A{A}')


@pytest.mark.parametrize('n', [0, 1, 1024, 1025, (1 << 20) + 7, (1 << 24) + 3])
def test_reduce_sum_exact(n):
    from scalerl_b200 import ops
    x = (np.random.RandomState(n % 1000).randn(n) + 1).astype(np.float32)
    xd = _dev(x)
    Ck = E.Checker(RESULTS, R)
    for square, scale in ((False, 1.0), (True, 0.5), (False, -0.25)):
        got = ops.reduce_sum(xd, square=square, scale=scale)
        val, S = R.reduce_sum(x, square, scale)
        sens = None
        if n >= 1024:                                # warp 0's partial (threads 0..31, every 1024th element) left out
            keep = (np.arange(n) % 1024) >= 32
            sens = R.sensitivity(R.reduce_sum(x[keep], square, scale)[0], val, S, R.CHECK_C['reduce_sum'])
            if sens < R.SENS:
                Ck.fails.append(f'reduce_sum n={n} square={square}: leaving out a warp moves the sum by only {sens:.1f} x the bound')
        Ck.bound(f'sum_square{int(square)}', float(got), val, S, R.CHECK_C['reduce_sum'], sens)
    Ck.done(f'reduce_n{n}')


# ------------------------------------------------------------------------------------------------ sample_actions
def _sample(xd, ud):
    from scalerl_b200 import _lib
    N, A = xd.shape
    out = torch.full((N,), -7, dtype=torch.int64, device='cuda')
    _lib.check(_lib.lib().srl_sample_actions(xd.data_ptr(), ud.data_ptr() if ud is not None else None, N, A, out.data_ptr(),
                                             torch.cuda.current_stream().cuda_stream), 'srl_sample_actions')
    return out


@pytest.mark.parametrize('A', [1, 2, 6, 18, 31])
def test_sample_actions_exact(A):
    N = 100003
    rng = np.random.RandomState(A)
    Ck = E.Checker(RESULTS, R)
    for regime in R.LOGIT_REGIMES:
        x = R.logit_rows(rng, (N, A), regime)
        u = rng.rand(N).astype(np.float32)
        top = np.nextafter(np.float32(1), np.float32(0))                    # the largest float below 1
        u[0], u[1] = 0.0, top
        if A >= 2:                          # rows whose last actions have probability 0 in fp32, at the top of the CDF: the A - 1 fallback
            x[2:34, A // 2:] = x[2:34, :A // 2].max(-1, keepdims=True) - 200
            u[2:34] = top
        xd, ud = _dev(x), _dev(u)
        got = _host(_sample(xd, ud))
        want, margin, bound = R.sample_ref(x, u)
        ok = margin > bound
        wrong = int((got[ok] != want[ok]).sum())
        e32 = np.exp((x - x.max(-1, keepdims=True)).astype(np.float64)).astype(np.float32)     # exp(x - max) rounded to fp32
        zero_pick = int((R.gather(e32, np.clip(got, 0, A - 1)) == 0).sum() + ((got < 0) | (got >= A)).sum())
        excluded = int((~ok).sum())
        Ck.count(f'sample_{regime}', wrong=wrong, excluded=excluded, excluded_frac=excluded / N, zero_probability_picks=zero_pick, n=N)
        if wrong or zero_pick or excluded > MAX_EXCLUDED * N:
            Ck.fails.append(f'sample {regime}: {wrong} decidable rows differ, {zero_pick} zero-probability picks, {excluded} excluded')
        # u = NULL: the first maximal index, with ties
        xt = x.copy()
        rows_t = np.arange(0, N, 2)
        src = rng.randint(0, A, size=rows_t.size)
        xt[rows_t, src] = xt[rows_t].max(-1)                                  # a second (or the same) maximal entry
        am = _host(_sample(_dev(xt), None))
        bad = int((am != np.argmax(xt, -1)).sum())
        Ck.count(f'argmax_{regime}', differ=bad, n=N)
        if bad:
            Ck.fails.append(f'argmax {regime}: {bad} rows are not the first maximal index')
    Ck.done(f'sample_A{A}')
