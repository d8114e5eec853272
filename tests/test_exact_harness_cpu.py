"""CPU: the shared harness of the fp64 exact-check suites (tests/exact.py) on small hand-made inputs: the error metric with each
suite's ETA and NaN rule, the Checker's bit comparisons and witness requirement, the results writer and the summary."""
import json
import math
import types

import numpy as np
import pytest
import torch

from tests import apex_head_ref, optim_ref, tail_ref
from tests import exact as E

NAN = float('nan')
REF = types.SimpleNamespace(ratio=optim_ref.ratio, sensitivity=optim_ref.sensitivity, SENS=20.0, MISTAKES={'m': 'a mistake'})


def test_nan_on_one_side_fails():
    for R in (tail_ref, optim_ref, apex_head_ref):
        assert R.ratio(np.array([1.0, NAN]), np.array([1.0, 2.0]), np.ones(2), 1) == math.inf
        assert R.ratio(np.array([1.0, 2.0]), np.array([1.0, NAN]), np.ones(2), 1) == math.inf
    Ck = E.Checker('x.json', REF)
    Ck.bound('b', np.array([NAN]), np.array([0.0]), np.ones(1), 1)
    assert Ck.res['b']['err_over_bound'] == math.inf and Ck.fails


def test_nan_on_both_sides_follows_the_suites_rule():
    got, ref = np.array([1.0, NAN]), np.array([1.0, NAN])
    assert math.isnan(tail_ref.ratio(got, ref, np.ones(2), 1))          # the tail's check on such an output fails
    assert optim_ref.ratio(got, ref, np.ones(2), 1) == 0.0              # the optimizer's and the heads' agree
    assert apex_head_ref.ratio(torch.tensor(got), torch.tensor(ref), torch.ones(2), 1) == 0.0
    for R, fails in ((tail_ref, True), (optim_ref, False)):
        Ck = E.Checker('x.json', types.SimpleNamespace(ratio=R.ratio))
        Ck.bound('b', got, ref, np.ones(2), 1)
        assert bool(Ck.fails) == fails


def test_eta():
    assert tail_ref.ETA == apex_head_ref.ETA == 2.0 ** -126 and optim_ref.ETA == 2.0 ** -149
    for R in (tail_ref, optim_ref, apex_head_ref):
        assert R.ratio(np.array([R.ETA]), np.array([0.0]), np.array([0.0]), 1) == 1.0
        assert R.ratio(np.array([2 * R.ETA]), np.array([0.0]), np.array([0.0]), 2) == 1.0
        assert R.ratio(np.array([1.0 + 2 * E.U]), np.array([1.0]), np.array([1.0]), 1) == 2 * E.U / (E.U + R.ETA)


def test_empty_inputs_give_zero():
    for R in (tail_ref, optim_ref):
        assert R.ratio(np.zeros(0), np.zeros(0), np.zeros(0), 1) == 0.0
    assert apex_head_ref.ratio(torch.zeros(0), torch.zeros(0), torch.zeros(0), 1) == 0.0


def test_ratio_takes_numpy_and_numbers_exactly():
    x = np.float32(1.0) + np.float32(2.0 ** -23)
    assert optim_ref.ratio(x, 1.0, 1.0, 1) == E.ratio(torch.tensor([float(x)], dtype=torch.float64), 1.0, 1.0, 1, optim_ref.ETA, True)
    assert E.ratio(float(x), 1.0, 1.0, 1, 0.0, True) == 2.0


def test_sign_of_zero_is_a_bit_difference():
    Ck = E.Checker('x.json')
    Ck.exact('e', torch.tensor([0.0, -0.0]), torch.tensor([0.0, 0.0]))
    assert Ck.res['e'] == {'bits_differ': 1, 'n': 2} and Ck.fails
    for dtype in (torch.float32, torch.bfloat16, torch.float64, torch.uint8):
        Ck = E.Checker('x.json')
        Ck.zero('z', torch.zeros(5, dtype=dtype))
        assert Ck.res['z'] == {'nonzero': 0, 'n': 5} and not Ck.fails
    Ck.zero('z', torch.tensor([0.0, -0.0, 0.0], dtype=torch.bfloat16))
    assert Ck.res['z'] == {'nonzero': 1, 'n': 3} and Ck.fails


def test_exact_fails_on_a_shape_or_dtype_mismatch():
    Ck = E.Checker('x.json')
    Ck.exact('same', torch.ones(3, dtype=torch.bfloat16), torch.ones(3, dtype=torch.bfloat16))
    assert Ck.res['same'] == {'bits_differ': 0, 'n': 3} and not Ck.fails
    Ck.exact('shape', torch.ones(3), torch.ones(4))
    assert Ck.res['shape']['bits_differ'] == -1 and len(Ck.fails) == 1
    Ck.exact('dtype', torch.ones(3), torch.ones(3, dtype=torch.bfloat16))
    assert Ck.res['dtype']['bits_differ'] == -1 and len(Ck.fails) == 2
    Ck.exact('numpy_shape', np.ones(3, np.float32), np.ones(2, np.float32))
    assert Ck.res['numpy_shape']['bits_differ'] == -1 and len(Ck.fails) == 3


def test_exact_rounds_numpy_to_fp32_first():
    Ck = E.Checker('x.json')
    Ck.exact('scalar', np.float32(1.5), np.array([1.5], np.float32))                # a 0-d value against one element
    Ck.exact('nan', np.float32(np.nan), np.float32(np.nan))
    Ck.exact('rounded', np.float64(1.0 + 2.0 ** -30), np.float32(1.0))              # equal once both are fp32
    assert not Ck.fails and Ck.res['scalar'] == {'bits_differ': 0, 'n': 1}
    Ck.exact('differ', np.array([1.0, 2.0], np.float32), np.array([1.0, np.nextafter(np.float32(2), np.float32(3))], np.float32))
    assert Ck.res['differ'] == {'bits_differ': 1, 'n': 2} and Ck.fails


def test_witness_below_sens_fails_and_at_sens_passes():
    Ck = E.Checker('x.json', REF)
    Ck.require('at', {'m': 20.0}, ['m'])
    assert not Ck.fails
    Ck.require('below', {'m': np.nextafter(20.0, 0.0)}, ['m'])
    Ck.require('missing', {}, ['m'])
    Ck.require('nan', {'m': NAN}, ['m'])
    assert len(Ck.fails) == 3 and all('a mistake' in f for f in Ck.fails)


def test_bound_records_the_mistakes_it_is_given():
    Ck = E.Checker('x.json', REF)
    ref, S = np.array([1.0, 2.0]), np.array([1.0, 1.0])
    Ck.bound('b', ref, ref, S, 1, mistakes={'m': ref + 100 * E.U, 'k': ref})
    e = Ck.res['b']
    assert e['err_over_bound'] == 0.0 and e['margin'] == math.inf and e['mistake'] == 'm' and e['sens_k'] == 0.0
    assert e['sensitivity'] == e['sens_m'] == Ck.sens['m'] > 20
    Ck.bound('n', ref, ref, S, 1, sens=3.0)
    assert Ck.res['n']['sensitivity'] == 3.0 and 'mistake' not in Ck.res['n']


def test_done_records_the_case_then_raises(tmp_path, monkeypatch):
    monkeypatch.setenv('SRL_RESULTS_DIR', str(tmp_path))
    Ck = E.Checker('x.json', REF)
    Ck.bound('b', np.array([1.0]), np.array([2.0]), np.ones(1), 1)
    with pytest.raises(AssertionError, match='b: '):
        Ck.done('case')
    assert json.load(open(tmp_path / 'x.json'))['case']['b']['err_over_bound'] > 1


def test_record_merges_into_the_file(tmp_path, monkeypatch):
    monkeypatch.delenv('SRL_RESULTS_DIR', raising=False)
    E.record('r.json', 'a', {'v': 1})                                  # unset: nothing written
    assert not list(tmp_path.iterdir())
    d = tmp_path / 'out'
    monkeypatch.setenv('SRL_RESULTS_DIR', str(d))
    E.record('r.json', 'a', {'v': 1})
    E.record('r.json', 'b', {'v': 2})
    E.record('r.json', 'a', {'v': 3})
    assert json.load(open(d / 'r.json')) == {'a': {'v': 3}, 'b': {'v': 2}}


def test_summary_takes_the_weakest_margin_and_sensitivity_and_the_worst_of_the_rest(tmp_path, monkeypatch):
    monkeypatch.setenv('SRL_RESULTS_DIR', str(tmp_path))
    E.record('s.json', 'c1', {'x@t1': {'err_over_bound': 0.5, 'margin': 2.0, 'sensitivity': 0.0, 'sens_m': 30.0, 'rel_l2_margin': 9.0,
                                       'mistake': 'm'}})
    E.record('s.json', 'c2', {'x@t2': {'err_over_bound': 0.25, 'margin': 4.0, 'sensitivity': 50.0, 'sens_m': 25.0, 'rel_l2_margin': 3.0},
                              'partition': 7})
    E.summarize('s.json', kind=lambda name: name.split('@')[0])
    assert json.load(open(tmp_path / 's.json'))['summary'] == {
        'x': {'err_over_bound': 0.5, 'margin': 2.0, 'sensitivity': 50.0, 'sens_m': 25.0, 'rel_l2_margin': 3.0}}
