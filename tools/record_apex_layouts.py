"""Record tests/golden/apex_layouts.json: what every Ape-X layout entry point of the C ABI returns (python tools/record_apex_layouts.py
[--out PATH]).

For every A in 1..31, each entry point and each valid head it takes (plain; dueling; num_atoms 2, 51 and 64; each with noisy 0 and 1
through srl_apex_param_layout_noisy), the return value and all 18 offset and count slots (slots an entry point leaves alone keep
the fill value -7).  For the bad arguments below, the return value, the slots and the srl_last_error text: A 0 and 32, dueling 2,
num_atoms 1 and 65, noisy -1 and 2, dueling with num_atoms, and srl_apex_param_layout(40), which checks nothing and returns a layout.

tests/test_apex_layouts_cpu.py recomputes all of it: the flat buffer's offsets, padding included, are part of the bits the
learner computes (its gradient norm runs over the whole buffer), so the layout code may change how it is written, not what it
returns.  Host code only: no CUDA device needed."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

OUT = os.path.join(ROOT, 'tests', 'golden', 'apex_layouts.json')
HEADS = ((0, 0), (1, 0), (0, 2), (0, 51), (0, 64))      # (dueling, num_atoms)


def _calls():
    """(entry point, args) of every recorded call"""
    calls = []
    for A in range(1, 32):
        calls.append(('srl_apex_param_layout', (A,)))
        calls += [('srl_apex_param_layout_ex', (A, d)) for d in (0, 1)]
        calls += [('srl_apex_param_layout_cat', (A, K)) for K in (0, 2, 51, 64)]
        calls += [('srl_apex_param_layout_noisy', (A, d, K, n)) for d, K in HEADS for n in (0, 1)]
    calls += [('srl_apex_param_layout', (A,)) for A in (0, 32, 40)]
    calls += [('srl_apex_param_layout_ex', args) for args in ((0, 0), (32, 0), (6, 2))]
    calls += [('srl_apex_param_layout_cat', args) for args in ((0, 0), (32, 0), (6, 1), (6, 65))]
    calls += [('srl_apex_param_layout_noisy', args) for args in ((0, 0, 0, 0), (32, 0, 0, 1), (6, 2, 0, 0), (6, 0, 1, 0), (6, 0, 65, 1),
                                                                (6, 0, 0, -1), (6, 0, 0, 2), (6, 1, 51, 0), (6, 1, 51, 1))]
    return calls


def record():
    """{"entry(args)": {ret, off, cnt[, error]}} of every call of _calls()"""
    from scalerl_b200 import _lib
    L = _lib.lib()
    rec = {}
    for fn, args in _calls():
        off, cnt = (C.c_int64 * 18)(*[-7] * 18), (C.c_int64 * 18)(*[-7] * 18)
        ret = getattr(L, fn)(*args, off, cnt)
        r = {'ret': int(ret), 'off': list(off), 'cnt': list(cnt)}
        if ret < 0:
            r['error'] = L.srl_last_error().decode()
        rec[f'{fn}{args}'.replace(' ', '')] = r
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=OUT)
    a = ap.parse_args()
    rec = record()
    with open(a.out, 'w') as f:
        f.write('{\n' + ',\n'.join(f'{json.dumps(k)}: {json.dumps(v)}' for k, v in rec.items()) + '\n}\n')
    print(f'{len(rec)} calls -> {a.out}')


if __name__ == '__main__':
    main()
