"""The harness the fp64 exact-check suites share (tests/test_gpu_*_exact.py): the error metric of a per-element rounding bound, one
Checker, the results writer and the end-of-module summary.

A suite's reference module (tests/tail_ref.py, optim_ref.py, apex_head_ref.py) binds its own ETA and NaN rule into `ratio` /
`sensitivity` and keeps its SENS and MISTAKES; a Checker given that module uses them for its bounds and witness requirements.

Results go to $SRL_RESULTS_DIR/<results file> when SRL_RESULTS_DIR is set: one entry per case ({check: its measurements}), and from
the suites that install `summary` one 'summary' entry per kind of check, which takes the smallest value over every case of each margin
and sensitivity (keys margin, *_margin, sensitivity, sens_*) above 0 -- a sensitivity of 0 is a case where no mistake moves the
check -- and the largest of every other number."""
import json
import math
import os

import numpy as np
import pytest
import torch

from tests import layer_ref as LR

U = 2.0 ** -24                  # fp32's unit roundoff
# an fp32 result of one accumulation (test_gpu_layer_exact / lstm_exact): rel-L2 and normalised max error, and the multiple of RTOL
# by which leaving out one unit of the work must move its reference
RTOL, NTOL, SENS = 2e-5, 1e-4, 20


# ------------------------------------------------------------------------------------------------ results
def _path(results_file):
    d = os.environ.get('SRL_RESULTS_DIR')
    return os.path.join(d, results_file) if d else None


def _write(p, cur):
    os.makedirs(os.path.dirname(p), exist_ok=True)
    json.dump(cur, open(p, 'w'), indent=1, sort_keys=True)


def record(results_file, case, obj):
    """store obj under case in $SRL_RESULTS_DIR/results_file (merged into what the file holds); nothing when SRL_RESULTS_DIR is unset"""
    p = _path(results_file)
    if not p:
        return
    cur = json.load(open(p)) if os.path.exists(p) else {}
    cur[case] = obj
    _write(p, cur)


def _weakest_first(key):
    return key == 'margin' or key.endswith('_margin') or key == 'sensitivity' or key.startswith('sens_')


def summarize(results_file, kind=lambda name: name):
    """add the 'summary' entry to the results file: per kind(check name), the smallest margin / sensitivity above 0 and the largest
    of every other number, over every case"""
    p = _path(results_file)
    if not p or not os.path.exists(p):
        return
    cur = json.load(open(p))
    table = {}
    for case, res in cur.items():
        if case == 'summary' or not isinstance(res, dict):
            continue
        for name, e in res.items():
            if not isinstance(e, dict):
                continue
            t = table.setdefault(kind(name), {})
            for k, v in e.items():
                if not isinstance(v, (int, float)):
                    continue
                if _weakest_first(k):
                    if v > 0:
                        t[k] = min(t.get(k, v), v)
                else:
                    t[k] = max(t.get(k, v), v)
    cur['summary'] = table
    _write(p, cur)


def summary(results_file, kind=lambda name: name):
    """an autouse module fixture that summarizes the results file after the module: `_summary = exact.summary(...)` in the suite"""
    @pytest.fixture(scope='module', autouse=True)
    def _summary():
        yield
        summarize(results_file, kind)
    return _summary


# ------------------------------------------------------------------------------------------------ metrics
def _t64(x, device):
    if isinstance(x, torch.Tensor):
        return x.detach().to(device, torch.float64)
    return torch.from_numpy(np.asarray(x, dtype=np.float64)).to(device)


def ratio(got, ref, S, c, eta, nan_equal):
    """max |got - ref| / (c (U S + eta)) over every element, in float64 on the device of the first tensor among got, ref, S (numpy
    arrays and numbers are converted exactly; nothing is copied to the host).  0 where both agree exactly and for empty inputs,
    inf where only one side is NaN; where both are NaN, 0 when nan_equal, else NaN, which fails every check"""
    dev = next((x.device for x in (got, ref, S) if isinstance(x, torch.Tensor)), 'cpu')
    got, ref, S = (_t64(x, dev) for x in (got, ref, S))
    diff = (got - ref).abs()
    q = torch.where(diff == 0, torch.zeros_like(diff), diff / (c * (U * S + eta)))
    q = torch.where(got.isnan() != ref.isnan(), math.inf, q)
    if nan_equal:
        q = torch.where(got.isnan() & ref.isnan(), 0.0, q)
    return float(q.max()) if q.numel() else 0.0


# how far a mistake moves the reference, in bounds: the ratio of the mistake's reference to the true one
sensitivity = ratio


def left_out(part, ref):
    """how far leaving the part of a sum out moves it, relative: |part| / |ref| in L2"""
    return float(part.norm() / max(float(ref.norm()), 1e-300))


def _margin(bound, err):
    return bound / err if err > 0 else math.inf


def _bits(x):
    return x.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[x.element_size()])


# ------------------------------------------------------------------------------------------------ the checks of one case
class Checker:
    """Each check records its measurements under its name in `res` and adds a line to `fails` when it fails; done(case) writes res
    to the results file, then asserts.  ref: the suite's reference module, whose ratio / sensitivity, SENS and MISTAKES bound() and
    require() use.  `sens` collects the strongest sensitivity of every mistake over the case's bound() calls."""

    def __init__(self, results_file, ref=None):
        self.results_file, self.ref = results_file, ref
        self.res, self.fails, self.sens = {}, [], {}

    def bound(self, name, got, ref, S, c, sens=None, mistakes=None):
        """got within c (U S + ETA) of ref, element by element.  sens: the check's sensitivity, a number or {mistake: sensitivity}
        (recorded as the strongest, its mistake and each one); mistakes: {mistake: its reference}, whose sensitivities are taken
        here"""
        q = self.ref.ratio(got, ref, S, c)
        e = {'err_over_bound': q, 'margin': 1.0 / q if q > 0 else math.inf}
        if mistakes:
            sens = {m: self.ref.sensitivity(pert, ref, S, c) for m, pert in mistakes.items()}
        if isinstance(sens, dict):
            for m, s in sens.items():
                e[f'sens_{m}'] = min(s, 1e30)
                self.sens[m] = max(self.sens.get(m, 0.0), s)
            if sens:
                e['sensitivity'] = max(sens.values())
                e['mistake'] = max(sens, key=sens.get)
        elif sens is not None:
            e['sensitivity'] = sens
        self.res[name] = e
        if not q <= 1.0:
            self.fails.append(f'{name}: {q:.3f} x the bound')

    def require(self, name, sens, mistakes):
        """each of `mistakes` moves `name` (a check or the case) by at least SENS x the bound, as sens = {mistake: sensitivity} says"""
        for m in mistakes:
            s = sens.get(m, 0.0)
            if not s >= self.ref.SENS:
                self.fails.append(f'{name}: {m} ({self.ref.MISTAKES[m]}) moves it by only {s:.1f} x the bound')

    def exact(self, name, got, want):
        """bit for bit.  Tensors compare by their own element size, and a shape or dtype mismatch fails; numpy arrays and numbers
        are rounded to fp32 and flattened first"""
        got, want = (x.contiguous() if isinstance(x, torch.Tensor) else torch.from_numpy(np.array(x, np.float32).reshape(-1))
                     for x in (got, want))
        same = got.shape == want.shape and got.dtype == want.dtype
        n = int((_bits(got) != _bits(want)).sum()) if same else -1
        self.res[name] = {'bits_differ': n, 'n': want.numel()}
        if not same:
            self.fails.append(f'{name}: {tuple(got.shape)} {got.dtype} vs {tuple(want.shape)} {want.dtype}')
        elif n:
            self.fails.append(f'{name}: {n} of {want.numel()} elements differ in their bits (got {got.reshape(-1)[:4].tolist()}, '
                              f'want {want.reshape(-1)[:4].tolist()})')

    def zero(self, name, x):
        """every element is +0.0 (its bits are 0, so -0.0 fails), at any element size"""
        n = int((_bits(x.contiguous()) != 0).sum())
        self.res[name] = {'nonzero': n, 'n': x.numel()}
        if n:
            self.fails.append(f'{name}: {n} of {x.numel()} elements are not +0.0')

    def fp32(self, name, got, ref, sens=None):
        """an fp32 result of one accumulation: rel-L2 <= RTOL and normalised max error <= NTOL.  sens: how far leaving one unit of
        the work out moves the reference (left_out), which must be at least SENS x RTOL"""
        got = got.reshape(ref.shape)
        e = {'rel_l2': LR.rel_l2(got, ref), 'nerr': LR.nerr(got, ref)}
        e['rel_l2_margin'], e['nerr_margin'] = _margin(RTOL, e['rel_l2']), _margin(NTOL, e['nerr'])
        if sens is not None:
            e['sensitivity'] = sens
            e['sensitivity_margin'] = sens / (SENS * RTOL)
            if sens < SENS * RTOL:
                self.fails.append(f'{name}: one left-out unit of work moves the reference by {sens:.2e} < {SENS} x {RTOL:.0e}')
        self.res[name] = e
        if not (e['rel_l2'] <= RTOL and e['nerr'] <= NTOL):
            self.fails.append(f'{name}: {e}')

    def stored(self, name, hi, lo, ref, pre=None, split=False, terms=None):
        """a bf16-stored output (lo: the fp32-split mode's low twin) by layer_ref.compare_stored / stored_ok"""
        st = LR.compare_stored(hi, lo, ref, pre, terms)
        if 'mismatch_frac' in st:
            st['mismatch_margin'] = _margin(LR.MISMATCH, st['mismatch_frac'])
        self.res[name] = st
        if not LR.stored_ok(st, split):
            self.fails.append(f'{name}: {st}')

    def equal(self, name, got, want):
        self.res[name] = {'got': got, 'want': want}
        if got != want:
            self.fails.append(f'{name}: {got} != {want}')

    def count(self, name, **kv):
        self.res[name] = kv

    def done(self, case):
        """record the case, then assert that no check failed"""
        record(self.results_file, case, self.res)
        assert not self.fails, f'{len(self.fails)} failed:\n' + '\n'.join(self.fails[:20])
