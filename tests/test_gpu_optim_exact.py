"""The clip and optimizer kernels of csrc/optim.cu against an fp64 evaluation of their own operation (tests/optim_ref.py), every element
of every output, on the operands the GPU itself read, at every grid and tail edge of the fused cooperative step.

  * The fused step through srl_test_clip_optim at any n: n = 1 .. 7, n4 = stride - 1 / stride / stride + 1 (n % 4 = 0 and 3),
    2 stride - 1 / 2 stride / 2 stride + 1, 3 stride + 1 (the loop past the two register-held float4s), the block count on both sides
    of the cap, and the product sizes, for all six variants (RMSprop +- momentum, Adam; constant / linear lr).  stride = blocks x 512
    float4s, blocks as the hook reports it.  Each case: step 1 from a fresh state, step 2 on the same buffers unrefilled, and a step
    at t = 10^6 (through the device step count, where b2^t underflows) from a large state; max_norm rotates over 40, a value that
    clips, 0, -1 (no clip) and +inf (no clip).
  * The stand-alone C-ABI ops on the same sizes: the norm twice on one scratch block (the ticket reset), RMSprop with coef = NULL and
    with the norm's coefficient, Adam at a 4-byte offset.
  * The product paths: the IMPALA learner (+- LSTM, RMSprop +- momentum, Adam, constant / linear lr, steps 1 - 3, a checkpoint at a
    large step) and the Ape-X learner (one step per head of tests/apex_cases.py) give the hook's bits on the same inputs, and those
    are within the fp64 bounds.
  * Non-finite inputs: one NaN gradient poisons every weight as torch's clip_grad_norm_ + step does (unless the step does not clip);
    one +-Inf gives the coefficient 0; the weight snapshot copies exactly when the total loss is finite.

Every bound is per element, optim_ref.CHECK_C x 2^-24 x S; the clip coefficient, the lr and the step count are exact.  Before each call
coef is filled with NaN, so an output the kernel does not write shows.  Every hook call asserts which of the six clip_optim_kernel
templates the launcher instantiated and launched (the hook reports its OPT, SCHED and MOM); a learner's step must give the bits of the
hook call on its own inputs.  The suite runs no torch.profiler session: after the IMPALA learner and the cooperative steps have run in a
process, later profiler sessions there returned no kernel records on the H100, and other suites rely on them.
The worst err / bound of every check, its margin and its weakest sensitivity go to $SRL_RESULTS_DIR/optim_exact.json (per case, and a
summary per check)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch

from scalerl_b200 import _lib
from tests import exact as E
from tests import optim_ref as R

pytestmark = pytest.mark.gpu

RESULTS = 'optim_exact.json'
VARIANTS = {'rms_const': ('rmsprop', False, 'constant'), 'rms_linear': ('rmsprop', False, 'linear'),
            'mom_const': ('rmsprop', True, 'constant'), 'mom_linear': ('rmsprop', True, 'linear'),
            'adam_const': ('adam', False, 'constant'), 'adam_linear': ('adam', False, 'linear')}
MAX_NORMS = (40.0, 'clip', 0.0, -1.0, math.inf)
BIG_T = 10 ** 6


def _variant_code(opt, mom, sched):
    """4 OPT + 2 SCHED + MOM of the clip_optim_kernel<OPT, SCHED, MOM> template a variant must launch"""
    return 4 * int(opt == 'adam') + 2 * int(sched == 'linear') + int(mom)


_summary = E.summary(RESULTS, kind=lambda name: name.split('@')[0])        # per check, over its steps and calls


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _host(t):
    return t.detach().cpu().numpy()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ the hook
class Bufs:
    """device buffers of one fused step: p, g, s0, s1, buf (momentum), coef[3], scratch, the device step count"""

    def __init__(self, g, st, opt, mom):
        self.p, self.g, self.s0 = _dev(st['p']), _dev(g), _dev(st['s0'])
        self.s1 = _dev(st['s1']) if opt == 'adam' else None
        self.buf = _dev(st['buf']) if mom else None
        self.coef = torch.full((3,), float('nan'), device='cuda')
        self.scratch = torch.zeros(1024, device='cuda')
        self.dstep = torch.zeros(1, dtype=torch.int32, device='cuda')

    def refill(self, st, t_before):
        for name in ('p', 's0', 's1', 'buf'):
            d = getattr(self, name)
            if d is not None:
                d.copy_(torch.from_numpy(st[name]))
        self.dstep.fill_(t_before)

    def state(self):
        """the host copy of p and the optimizer state"""
        return {k: (None if getattr(self, k) is None else _host(getattr(self, k))) for k in ('p', 's0', 's1', 'buf')}


def hook(opt, mom, sched, b, max_norm, lr=None, a=None, bb=None, eps=None, frames_per_step=None, total_frames=None, lr_end=None,
         momentum=R.MOMENTUM, dstep=True):
    """one fused step on Bufs b (coef refilled with NaN first) -> the block count launched"""
    hp = R.HP[opt]
    sc = R.SCHEDULE
    b.coef.fill_(float('nan'))
    blocks, variant = C.c_int(0), C.c_int(-1)
    _lib.check_hook(_lib.hooks().srl_test_clip_optim(
        1 if opt == 'adam' else 0, b.p.data_ptr(), b.g.data_ptr(), b.s0.data_ptr(), b.s1.data_ptr() if b.s1 is not None else None,
        b.p.numel(), float(max_norm), b.coef.data_ptr(), b.scratch.data_ptr(), hp['lr'] if lr is None else lr, hp['a'] if a is None else a,
        hp['b'] if bb is None else bb, hp['eps'] if eps is None else eps, 1, b.dstep.data_ptr() if dstep else None,
        1 if sched == 'linear' else 0, sc['lr_end'] if lr_end is None else lr_end, sc['frames_per_step'] if frames_per_step is None else frames_per_step,
        sc['total_frames'] if total_frames is None else total_frames, b.buf.data_ptr() if mom and b.buf is not None else None, momentum,
        C.byref(blocks), C.byref(variant), _stream()), 'srl_test_clip_optim')
    assert variant.value == _variant_code(opt, mom, sched), f'launched template {variant.value}, want {_variant_code(opt, mom, sched)}'
    return blocks.value


_CAP = {}


def cap(variant):
    """the most blocks the variant's cooperative launch uses on this GPU (occupancy x SMs, at most 592), as the hook reports it"""
    if variant not in _CAP:
        opt, mom, sched = VARIANTS[variant]
        n = 4 * (592 * 512 + 1)
        z = np.zeros(n, np.float32)
        b = Bufs(z, dict(p=z, s0=z, s1=z, buf=z), opt, mom)
        _CAP[variant] = hook(opt, mom, sched, b, 40.0)
        torch.cuda.synchronize()
    return _CAP[variant]


def _product_sizes():
    return {'impala': _lib.param_layout(6)[0], 'impala_lstm': _lib.param_layout(6, True)[0],
            'apex_noisy_c51': _lib.apex_param_layout(6, num_atoms=11, noisy=True)[0]}


def n_of(label, cp):
    """the n of a grid label at the cap cp (stride = cp x 512 float4s)"""
    s = cp * 512
    small = {'n1': 1, 'n2': 2, 'n3': 3, 'n4': 4, 'n5': 5, 'n7': 7}
    if label in small:
        return small[label]
    if label in ('impala', 'impala_lstm', 'apex_noisy_c51'):
        return _product_sizes()[label]
    n4, r = {'s-1_r0': (s - 1, 0), 's-1_r3': (s - 1, 3), 's_r0': (s, 0), 's_r3': (s, 3), 's+1_r0': (s + 1, 0), 's+1_r3': (s + 1, 3),
             '2s-1': (2 * s - 1, 2), '2s': (2 * s, 0), '2s+1': (2 * s + 1, 1), '3s+1': (3 * s + 1, 3),
             'cap-1_blocks': ((cp - 1) * 512, 1), 'cap_blocks+1': ((cp - 1) * 512 + 1, 0)}[label]
    return 4 * n4 + r


GRID = ['n1', 'n2', 'n3', 'n4', 'n5', 'n7', 's-1_r0', 's-1_r3', 's_r0', 's_r3', 's+1_r0', 's+1_r3', '2s-1', '2s', '2s+1', '3s+1',
        'cap-1_blocks', 'cap_blocks+1', 'impala', 'impala_lstm', 'apex_noisy_c51']


def want_blocks(n, cp, threads=512):
    return max(1, min(-(-(n // 4) // threads), cp))


# ------------------------------------------------------------------------------------------------ the checks of one step
def check_step(Ck, tag, opt, mom, sched, b, before, g, max_norm, t, blocks, cp, require=(), mistakes=True):
    """every output of the step Bufs b has just taken from `before` (host state) on g: the block count, the norm (sum of squares
    bound), the coefficient, lr and step count exactly, then each new state from the inputs and p on the GPU's own state"""
    Ck.equal(f'blocks@{tag}', blocks, want_blocks(g.size, cp))
    coef = _host(b.coef)
    norm = np.float32(coef[0])
    s2, S2 = R.sumsq(g, blocks)
    Ck.bound(f'sumsq@{tag}', float(norm) ** 2, s2, S2, R.CHECK_C['sumsq'])
    c = R.clip_coef32(norm, max_norm)
    Ck.exact(f'coef@{tag}', coef[1], c)
    lr = R.lr_of(opt, sched, t)
    writes_lr = sched == 'linear' or mom
    Ck.exact(f'lr@{tag}', coef[2], lr if writes_lr else np.float32(np.nan))
    Ck.equal(f'step@{tag}', int(b.dstep.item()), t)
    after = b.state()
    st = dict(before, buf=before['buf'] if mom else None)
    own = {'s0': after['s0'], 's1': after['s1'], 'buf': after['buf'] if mom else None}
    ref = R.step(opt, st, g, coef[1], lr, t, own=own)
    lr_prev = R.lr_of(opt, sched, t - 1) if t > 1 else None
    sens = {}
    if mistakes:
        ms = [m for m in R.OUTPUT_MISTAKES[opt] if (m != 'lr_in_momentum' or mom) and (m != 'lr_prev_step' or (sched == 'linear' and t > 1))
              and (g.size <= 1 << 21 or m in require)]
        for m in ms:
            pert = R.step(opt, st, g, coef[1], lr, t, own=own, lr_prev=lr_prev, mistake=m)
            for k in ref:
                sens.setdefault(k, {})[m] = R.sensitivity(pert[k][0], ref[k][0], ref[k][1], ref[k][2])
        n4, stride = g.size // 4, blocks * 512
        norm_ms = (['norm_no_tail'] if g.size % 4 else []) + (['norm_no_hold_slot'] if n4 > stride else [])
        sens['sumsq'] = {m: R.sensitivity(R.sumsq(g, blocks, mistake=m)[0], s2, S2, R.CHECK_C['sumsq']) for m in norm_ms}
        Ck.require(f'sumsq@{tag}', sens['sumsq'], norm_ms)
        if sens['sumsq']:
            Ck.res[f'sumsq@{tag}']['sensitivity'] = min(sens['sumsq'].values())
        best = {m: max(sens[k][m] for k in ref) for m in ms}
        Ck.require(f'step@{tag}', best, [m for m in require if m in best])
    got = {'p': after['p'], 'square_avg': after['s0'], 'exp_avg': after['s0'], 'exp_avg_sq': after['s1'], 'momentum_buffer': after['buf']}
    for k, (val, S, cc) in ref.items():
        Ck.bound(f'{k}@{tag}', got[k], val, S, cc, sens.get(k))
    return after


# ------------------------------------------------------------------------------------------------ the fused step over the grid
@pytest.mark.parametrize('label', GRID)
@pytest.mark.parametrize('variant', list(VARIANTS))
def test_fused_step_exact(variant, label):
    opt, mom, sched = VARIANTS[variant]
    cp = cap(variant)
    n = n_of(label, cp)
    blocks = want_blocks(n, cp)
    rng = np.random.RandomState(sum(map(ord, variant + label)))
    g = R.grads(rng, n, blocks)
    st = R.state(rng, n, opt, 'zero')
    k = GRID.index(label)
    mn1, mn3 = R.max_norm_of(MAX_NORMS[k % 5], g), R.max_norm_of(MAX_NORMS[(k + 2) % 5], g)
    b = Bufs(g, st, opt, mom)
    Ck = E.Checker(RESULTS, R)
    got_blocks = hook(opt, mom, sched, b, mn1)
    # step 1 from a fresh state: the mistakes every case that steps its small gradients must show (eps inside the root, the old v of a
    # fresh state); the cases of n < 64 hold marked elements only, and max_norm 0 steps nothing
    req = ('eps_in_sqrt', 'old_v') if n >= 64 and MAX_NORMS[k % 5] != 0.0 else ()
    after = check_step(Ck, 't1', opt, mom, sched, b, st, g, mn1, 1, got_blocks, cp, require=req)
    # step 2 on the same buffers, not refilled: the device step count advances
    blocks2 = hook(opt, mom, sched, b, mn1)
    check_step(Ck, 't2', opt, mom, sched, b, after, g, mn1, 2, blocks2, cp, mistakes=n <= 1 << 20)
    # a late step from a large state: b2^t underflows
    st3 = R.state(rng, n, opt, 'large')
    b.refill(st3, BIG_T - 1)
    blocks3 = hook(opt, mom, sched, b, mn3)
    check_step(Ck, 'tbig', opt, mom, sched, b, st3, g, mn3, BIG_T, blocks3, cp, mistakes=False)
    Ck.done(f'fused_{variant}_{label}')


# ------------------------------------------------------------------------------------------------ the stand-alone C-ABI ops
@pytest.mark.parametrize('label', GRID)
def test_standalone_ops_exact(label):
    L = _lib.lib()
    n = n_of(label, cap('rms_const'))
    rng = np.random.RandomState(sum(map(ord, 'standalone' + label)))
    blocks = max(1, min(-(-(n // 4) // 256), 592))
    g = R.grads(rng, n, blocks)
    gd = _dev(g)
    Ck = E.Checker(RESULTS, R)
    scratch = torch.zeros(1028, device='cuda')
    coef = torch.empty(2, device='cuda')
    mn = R.max_norm_of('clip', g)
    first = None
    for call in (1, 2):                   # one scratch block: the second call needs the ticket the first one reset
        coef.fill_(float('nan'))
        f = lambda: _lib.check(L.srl_grad_norm_clip_coef(gd.data_ptr(), n, mn, coef.data_ptr(), scratch.data_ptr(), _stream()), 'grad_norm')
        f()
        c = _host(coef)
        s2, S2 = R.sumsq(g, blocks, fused=False)
        sens = {m: R.sensitivity(R.sumsq(g, blocks, mistake=m)[0], s2, S2, R.CHECK_C['sumsq']) for m in (['norm_no_tail'] if n % 4 else [])}
        Ck.bound(f'sumsq@call{call}', float(np.float32(c[0])) ** 2, s2, S2, R.CHECK_C['sumsq'], sens)
        Ck.require(f'sumsq@call{call}', sens, list(sens))
        Ck.exact(f'coef@call{call}', c[1], R.clip_coef32(np.float32(c[0]), mn))
        if first is None:
            first = c
        else:
            Ck.exact('norm_twice', c, first)
    hp = R.HP['rmsprop']
    for use_coef in (False, True):
        st = R.state(rng, n, 'rmsprop', 'large' if use_coef else 'zero')
        p, v = _dev(st['p']), _dev(st['s0'])

        def f():
            p.copy_(torch.from_numpy(st['p']))
            v.copy_(torch.from_numpy(st['s0']))
            _lib.check(L.srl_rmsprop_step(p.data_ptr(), gd.data_ptr(), v.data_ptr(), n, coef.data_ptr() if use_coef else None, hp['lr'],
                                          hp['a'], hp['eps'], _stream()), 'rmsprop')
        f()
        c = np.float32(first[1]) if use_coef else np.float32(1.0)
        ref = R.step('rmsprop', dict(st, buf=None), g, c, np.float32(hp['lr']), 1, own={'s0': _host(v)})
        got = {'p': _host(p), 'square_avg': _host(v)}
        for k, (val, S, cc) in ref.items():
            Ck.bound(f'rmsprop_{k}@coef{int(use_coef)}', got[k], val, S, cc)
    hp = R.HP['adam']
    st = R.state(rng, n, 'adam', 'large')
    off = lambda x: torch.cat([torch.zeros(1), torch.from_numpy(x)]).cuda()[1:]         # 4 bytes past a 16-byte boundary
    p, gg, m, v = off(st['p']), off(g), off(st['s0']), off(st['s1'])
    for t in (1, BIG_T):
        before = {'p': _host(p), 's0': _host(m), 's1': _host(v), 'buf': None}
        def f():
            for d, k in ((p, 'p'), (m, 's0'), (v, 's1')):
                d.copy_(torch.from_numpy(before[k]))
            _lib.check(L.srl_adam_step(p.data_ptr(), gg.data_ptr(), m.data_ptr(), v.data_ptr(), n, coef.data_ptr(), hp['lr'], hp['a'],
                                       hp['b'], hp['eps'], t, _stream()), 'adam')
        f()
        ref = R.step('adam', before, g, np.float32(first[1]), np.float32(hp['lr']), t, own={'s0': _host(m), 's1': _host(v)})
        got = {'p': _host(p), 'exp_avg': _host(m), 'exp_avg_sq': _host(v)}
        for k, (val, S, cc) in ref.items():
            Ck.bound(f'adam_{k}@t{t}', got[k], val, S, cc)
    Ck.done(f'standalone_{label}')


# ------------------------------------------------------------------------------------------------ non-finite inputs
@pytest.mark.parametrize('bad,max_norm', [(math.nan, 40.0), (math.nan, -1.0), (math.nan, math.inf), (math.inf, 40.0), (-math.inf, 40.0)])
@pytest.mark.parametrize('variant', ['rms_const', 'mom_linear', 'adam_const'])
def test_non_finite_gradient(variant, bad, max_norm):
    """torch's clip_grad_norm_ then step: a NaN norm makes the coefficient NaN and poisons every weight; max_norm -1 / +inf does not
    clip (coefficient 1: only the NaN element's weight is poisoned); an Inf gives the coefficient 0 (its own element NaN, every other
    weight keeps its value, up to the momentum of earlier steps)"""
    opt, mom, sched = VARIANTS[variant]
    n = 4099
    rng = np.random.RandomState(1)
    g = rng.randn(n).astype(np.float32)
    g[1234] = bad
    st = R.state(rng, n, opt, 'large')
    b = Bufs(g, st, opt, mom)
    b.dstep.fill_(2)
    blocks = hook(opt, mom, sched, b, max_norm)
    coef = _host(b.coef)
    Ck = E.Checker(RESULTS, R)
    c = R.clip_coef32(np.float32(coef[0]), max_norm)
    Ck.exact('coef', coef[1], c)
    if math.isnan(bad) and max_norm == 40.0:
        Ck.equal('coef_is_nan', bool(np.isnan(coef[1])), True)
    if math.isinf(bad):
        Ck.equal('coef_is_zero', float(coef[1]), 0.0)
    after = b.state()
    own = {'s0': after['s0'], 's1': after['s1'], 'buf': after['buf'] if mom else None}
    lr = R.lr_of(opt, sched, 3)
    ref = R.step(opt, dict(st, buf=st['buf'] if mom else None), g, coef[1], lr, 3, own=own)
    got = {'p': after['p'], 'square_avg': after['s0'], 'exp_avg': after['s0'], 'exp_avg_sq': after['s1'], 'momentum_buffer': after['buf']}
    for k, (val, S, cc) in ref.items():
        Ck.bound(k, got[k], val, S, cc)
        Ck.equal(f'{k}_nan_count', int(np.isnan(got[k]).sum()), int(np.isnan(val).sum()))
    # torch on the CPU, in fp32: the same NaN pattern
    prm = torch.nn.Parameter(torch.from_numpy(st['p'].copy()))
    prm.grad = torch.from_numpy(g.copy())
    if max_norm >= 0 and not math.isinf(max_norm):
        torch.nn.utils.clip_grad_norm_([prm], max_norm)
    Ck.equal('torch_grad_nan_count', int(torch.isnan(prm.grad).sum()), int(np.isnan(g * coef[1]).sum()))
    Ck.done(f'nonfinite_{variant}_{bad}_{max_norm}')


@pytest.mark.parametrize('loss', [math.nan, math.inf, -math.inf, 3.3e38, -3.3e38, 1.5, None])
def test_snapshot_copies_when_the_loss_is_finite(loss):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=2, batch_size=2, num_actions=4), process_group=False)
    try:
        dst = torch.full((L.numel,), -7.0, device='cuda')
        losses = None if loss is None else torch.tensor([0.0, 0.0, 0.0, loss], dtype=torch.float32, device='cuda')
        _lib.check(L._L.srl_learner_snapshot_params(L._h, dst.data_ptr(), losses.data_ptr() if losses is not None else None, _stream()),
                   'snapshot')
        torch.cuda.synchronize()
        copies = R.snapshot_copies(None if losses is None else _host(losses))
        if copies:
            assert torch.equal(dst, L.flat_params), loss
        else:
            assert bool((dst == -7.0).all()), loss
    finally:
        L.close()


# ------------------------------------------------------------------------------------------------ the product paths
IMPALA_CASES = {
    'rms_const': dict(use_lstm=False, optimizer='rmsprop', momentum=0.0, sched='constant', start=0),
    'mom_linear': dict(use_lstm=False, optimizer='rmsprop', momentum=0.9, sched='linear', start=0),
    'adam_linear': dict(use_lstm=False, optimizer='adam', momentum=0.0, sched='linear', start=0),
    'lstm_rms_const': dict(use_lstm=True, optimizer='rmsprop', momentum=0.0, sched='constant', start=0),
    'lstm_mom_const': dict(use_lstm=True, optimizer='rmsprop', momentum=0.9, sched='constant', start=0),
    'lstm_adam_const': dict(use_lstm=True, optimizer='adam', momentum=0.0, sched='constant', start=0),
    'adam_checkpoint': dict(use_lstm=False, optimizer='adam', momentum=0.0, sched='constant', start=BIG_T),
    'mom_checkpoint': dict(use_lstm=False, optimizer='rmsprop', momentum=0.9, sched='linear', start=5),
}


def _as_bufs(p, g, s0, s1, buf, opt, mom):
    """Bufs over clones of a learner's flat tensors"""
    b = Bufs.__new__(Bufs)
    b.p, b.g, b.s0 = p.clone(), g.clone(), s0.clone()
    b.s1 = s1.clone() if opt == 'adam' else None
    b.buf = buf.clone() if mom else None
    b.coef = torch.full((3,), float('nan'), device='cuda')
    b.scratch = torch.zeros(1024, device='cuda')
    b.dstep = torch.zeros(1, dtype=torch.int32, device='cuda')
    return b


@pytest.mark.parametrize('name', list(IMPALA_CASES))
def test_impala_learner_step_is_the_hook(name):
    """impala_case(name) in a child process: after an IMPALA learner has run in a process, that process's later torch.profiler sessions
    return no kernel records (seen on the H100 with the learner's profiled and unprofiled steps alike), which would blind every later
    suite that asserts which kernel ran"""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    code = f'import sys; sys.path.insert(0, {root!r}); from tests.test_gpu_optim_exact import impala_case; impala_case({name!r})'
    r = subprocess.run([sys.executable] + (['-s'] if sys.flags.no_user_site else []) + ['-c', code], cwd=root, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]


def impala_case(name):
    """the IMPALA learner's steps of IMPALA_CASES[name] against the hook (bits) and the fp64 bounds"""
    from oracle import impala_oracle as O
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    c = IMPALA_CASES[name]
    opt, mom, sched = c['optimizer'], c['momentum'] != 0, c['sched']
    T, B, A = 5, 4, 6
    total = R.SCHEDULE['total_frames']
    kw = dict(lr_schedule='linear', total_frames=total, min_learning_rate=R.SCHEDULE['lr_end']) if sched == 'linear' else {}
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, use_lstm=c['use_lstm'], optimizer=opt, momentum=c['momentum'],
                       learning_rate=R.HP[opt]['lr'], **kw)
    L = B200ImpalaLearner(hp, process_group=False, seed=3)
    Ck = E.Checker(RESULTS, R)
    try:
        if c['start']:
            L._set_opt_step(c['start'])
            rng = np.random.RandomState(9)
            for flat in (L.opt_state0, L.opt_state1, L.opt_state2):
                if flat is not None:
                    flat.copy_(torch.from_numpy((10.0 ** rng.uniform(-4, 0, flat.numel())).astype(np.float32)))
        a, bb, eps = (hp.adam_beta1, hp.adam_beta2, hp.adam_eps) if opt == 'adam' else (hp.alpha, 0.0, hp.epsilon)
        for k in range(3):
            batch = {key: v.cuda() for key, v in O.synthetic_batch(T, B, A, seed=20 + k, done_p=0.1).items()}
            L.forward_backward(batch)
            torch.cuda.synchronize()
            t0 = L.device_opt_step()
            hb = _as_bufs(L.flat_params, L.flat_grads, L.opt_state0, L.opt_state1, L.opt_state2, opt, mom)
            hb.dstep.fill_(t0)
            before = hb.state()
            L.apply_gradients()
            torch.cuda.synchronize()

            # the same step through the hook on the learner's pre-step buffers, with the template it must launch: the learner's
            # step must be its bits
            blocks = hook(opt, mom, sched, hb, hp.max_grad_norm, lr=hp.learning_rate, a=a, bb=bb, eps=eps, frames_per_step=float(T * B),
                          total_frames=float(total), lr_end=hp.min_learning_rate if sched == 'linear' else 0.0, momentum=hp.momentum)
            torch.cuda.synchronize()
            tag = f'step{k + 1}'
            Ck.exact(f'p_is_hook@{tag}', _host(L.flat_params), _host(hb.p))
            Ck.exact(f's0_is_hook@{tag}', _host(L.opt_state0), _host(hb.s0))
            if opt == 'adam':
                Ck.exact(f's1_is_hook@{tag}', _host(L.opt_state1), _host(hb.s1))
            if mom:
                Ck.exact(f'buf_is_hook@{tag}', _host(L.opt_state2), _host(hb.buf))
            n_coef = 3 if (sched == 'linear' or mom) else 2
            Ck.exact(f'coef_is_hook@{tag}', _host(L._coef)[:n_coef], _host(hb.coef)[:n_coef])
            Ck.equal(f'step@{tag}', L.device_opt_step(), t0 + 1)
            g = _host(hb.g)
            check_step(Ck, tag, opt, mom, sched, hb, before, g, hp.max_grad_norm, t0 + 1, blocks, cap(_variant(opt, mom, sched)), mistakes=False)
    finally:
        L.close()
    Ck.done(f'impala_{name}')


def _variant(opt, mom, sched):
    return next(k for k, v in VARIANTS.items() if v == (opt, mom, sched))


def _apex_heads():
    from tests import apex_cases as AC
    return list(AC.HEADS)


@pytest.mark.parametrize('head', _apex_heads())
def test_apex_learner_step_is_the_hook(head):
    from tests import apex_cases as AC
    h = AC.HEADS[head]
    B, A = 8, 4
    on, tg = AC.nets(h, A, seed=1)
    clip = 10.0 if len(head) % 2 else None
    Ck = E.Checker(RESULTS, R)
    (obs, act, rew, nobs, done), w = AC.batch(B, A, seed=4)
    xs = tuple(t.cuda() for t in (obs, act, h.scale_reward(rew), nobs, done))
    L = AC.learner(h, B, A, on, tg, seed=1, max_grad_norm=clip)
    hb = _as_bufs(L.flat_params, L.flat_grads, L.exp_avg, L.exp_avg_sq, None, 'adam', False)
    L.learn(xs, weights=w.cuda(), use_graph=False)
    before = hb.state()
    torch.cuda.synchronize()
    hb.g.copy_(L.flat_grads)
    cfg = L._cfg
    mn = cfg.max_grad_norm
    blocks = hook('adam', False, 'constant', hb, mn, lr=cfg.learning_rate, a=cfg.adam_beta1, bb=cfg.adam_beta2, eps=cfg.adam_eps)
    Ck.exact('p_is_hook', _host(L.flat_params), _host(hb.p))
    Ck.exact('exp_avg_is_hook', _host(L.exp_avg), _host(hb.s0))
    Ck.exact('exp_avg_sq_is_hook', _host(L.exp_avg_sq), _host(hb.s1))
    st = L.stats()
    Ck.exact('norm_and_coef_are_hook', np.array([st['grad_norm'], st['clip_coef']], np.float32), _host(hb.coef)[:2])
    g = _host(hb.g)
    hpa = R.HP['adam']
    assert (np.float32(cfg.learning_rate), np.float32(cfg.adam_beta1), np.float32(cfg.adam_beta2), np.float32(cfg.adam_eps)) == \
        tuple(np.float32(hpa[k]) for k in ('lr', 'a', 'b', 'eps')), 'the Ape-X defaults are the reference hyperparameters'
    check_step(Ck, 'step1', 'adam', False, 'constant', hb, before, g, mn, 1, blocks, cap('adam_const'), mistakes=False)
    L.close()
    Ck.done(f'apex_{head}')
