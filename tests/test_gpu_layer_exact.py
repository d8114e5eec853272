"""Every encoder and head kernel of the learner step against an fp64 evaluation of that one operation on the operands the GPU
itself read (tests/layer_ref.py).  No rounding of an earlier layer carries over, so the bounds are those of one fp32 accumulation:

  * fp32 outputs that are sums of exact bf16 products (conv / fc / head weight and bias gradients, h): rel-L2 <= 2e-5 and
    normalised max error <= 1e-4 per tensor.  Each check also measures its own SENSITIVITY -- the reference with one
    128-position chunk of a middle wgrad CTA (one 64-frame k-block for fc, one 16-frame slab for the heads, one 64-channel
    k-block for h) left out -- and requires it to be at least 20x the rel-L2 bound: a bound that could not see a missing chunk
    fails instead of passing quietly.
  * bf16-stored outputs (a1, a2, a3, dh, da3, da2, da1): every element is the bf16 rounding of the fp64 result or one ulp from
    it, at most 0.5 % differ, and a ReLU mask may disagree only at a tie (|pre-activation| < 1e-5 rms).  In the fp32-split mode
    hi + lo is within 2^-16 relative of the fp64 result.  Both allow for the fp32 accumulation error where a sum cancels:
    max(1e-5 rms, 2^-18 sum|products|) (layer_ref.compare_stored).
  * the zero padding of the dgrad grids (da3g outside 7x7, da2g outside 9x9, da1g outside 20x20) is bit-exactly zero.

The partition sweep re-runs the benchmark shape in child processes with other wgrad / backward / persistent CTA counts and with
programmatic dependent launch off: activations must be bit-identical everywhere, gradients within the fp32 bounds of the same
fp64 reference (scaled by chunks per CTA / 16 beyond 16: the tensor cores' accumulation error grows with the length of a CTA's
sum), and bit-identical between PDL on and off.  Measured errors, sensitivities and the partition table go to
$SRL_RESULTS_DIR/layer_exact.json when SRL_RESULTS_DIR is set."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import exact as E
from tests import layer_ref as R
from tests.layer_exact_worker import digest, run_step

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESULTS = 'layer_exact.json'

# each shape sits on an edge of the kernels
SHAPES = {
    (20, 32, 6): 'the benchmark: every conv wgrad ring wraps many times (conv1: 19 chunks per CTA, last CTA 1 chunk)',
    (20, 64, 4): "one GPU's shard of config 3",
    (1, 1, 6): 'one partial tile everywhere; one-CTA conv3 / conv2 wgrads with fewer chunks than ring stages',
    (4, 8, 6): "conv2's 3200 wgrad positions are a multiple of 128",
    (16, 8, 6): 'conv1 and conv3 wgrad positions and the fc M = 128 are exact multiples of their tiles',
    (7, 19, 18): 'ragged everywhere, and the 32-action head instantiation',
}
# (precision, column kernel, fused front, replayed learn(), poisoned shared memory)
MODES = {
    'bf16': ('bf16', True, False, False, False),
    'bf16_three_kernels': ('bf16', False, False, False, False),
    'bf16_fused_front': ('bf16', True, True, False, False),
    'bf16_replay': ('bf16', True, False, True, False),
    'split': ('fp32_split', True, False, False, False),
    'split_three_kernels': ('fp32_split', False, False, False, False),
}


def check_layers(T, B, A, bufs, grads, params, batch, split, ctas):
    """all per-layer comparisons of one step; returns (Checker, fp64 reference gradients)"""
    NF, NB = (T + 1) * B, T * B
    W = R.weights(params, split)
    C = E.Checker(RESULTS)
    lo = lambda n: bufs[n + '_lo'] if split else None
    sl = lambda p, a, b: (p[0][a:b], None if p[1] is None else p[1][a:b])
    frames = batch['obs'].reshape(NF, 4, 84, 84)
    reward, action = batch['reward'].reshape(-1), batch['action'].reshape(-1)
    # ---- forward
    if not torch.equal(bufs['xs'].reshape(NF, 21, 21, 64), R.s2d(frames).to(torch.bfloat16)):
        C.fails.append('xs is not the space-to-depth copy of the frames')
    a1 = (R.a1_planes_to_nchw(bufs['a1'], NF), None if not split else R.a1_planes_to_nchw(bufs['a1_lo'], NF))
    z1 = R.conv1_fwd(frames, W['conv1.weight'], params['conv1.bias'])
    C.stored('a1', a1[0], a1[1], z1.clamp_min(0), pre=z1, split=split)
    a1p = R.pair(*a1)
    z2 = R.conv_fwd(a1p, W['conv2.weight'], params['conv2.bias'], 2)
    a2 = (R.nhwc_to_nchw(bufs['a2'], NF, 9), None if not split else R.nhwc_to_nchw(bufs['a2_lo'], NF, 9))
    C.stored('a2', a2[0], a2[1], z2.clamp_min(0), pre=z2, split=split)
    a2p = R.pair(*a2)
    z3 = R.conv_fwd(a2p, W['conv3.weight'], params['conv3.bias'], 1)
    a3 = (R.nhwc_to_nchw(bufs['a3'], NF, 7), None if not split else R.nhwc_to_nchw(bufs['a3_lo'], NF, 7))
    C.stored('a3', a3[0], a3[1], z3.clamp_min(0), pre=z3, split=split)
    a3p = R.pair(*a3)
    zh = R.fc_fwd(a3p, W['fc.weight'], params['fc.bias'])
    idx = torch.arange(64) * 49 + 24                                    # one 64-channel k-block (pixel hw = 24)
    kblk = R.sp(lambda a, w: a.reshape(NF, -1)[:, idx] @ w[:, idx].t(), a3p, W['fc.weight'])
    C.fp32('h', bufs['h'], zh.clamp_min(0), E.left_out((zh - kblk).clamp_min(0) - zh.clamp_min(0), zh.clamp_min(0)))
    h = bufs['h'].reshape(NF, 512).to(R.F64)
    lg, bs = R.heads_fwd(R.core(h, reward, action, A), params)
    C.fp32('logits', bufs['logits'], lg)
    C.fp32('baseline', bufs['baseline'], bs)
    # ---- heads backward
    dl, dv = bufs['dlogits'].reshape(NB, A), bufs['dbaseline'].reshape(NB)
    C.stored('dh', bufs['dh'].reshape(NB, 512), None if not split else lo('dh').reshape(NB, 512), R.dh_ref(dl, dv, h[:NB], params), split=split)
    c_nb = R.core(h[:NB], reward[:NB], action[:NB], A)
    ref = R.head_grads(dl, dv, c_nb)
    nslab = (NB + 15) // 16
    spg = (nslab + 31) // 32
    s0 = ((nslab + spg - 1) // spg // 2) * spg                           # first slab of the middle slab group
    part = R.head_grads(dl[16 * s0:16 * s0 + 16], dv[16 * s0:16 * s0 + 16], c_nb[16 * s0:16 * s0 + 16])
    for k in ref:
        C.fp32(k, grads[k], ref[k], E.left_out(part[k], ref[k]))
    # ---- fc
    dhp = R.pair(bufs['dh'].reshape(NB, 512), None if not split else lo('dh').reshape(NB, 512))
    mask3 = (a3[0][:NB] > 0).to(R.F64)
    dWf, dbf, da3 = R.fc_bwd(dhp, sl(a3p, 0, NB), W['fc.weight'], mask3)
    dterms = R.abs_terms(lambda d, w: d @ w, dhp, W['fc.weight']).reshape(-1, 64, 7, 7) * mask3
    kb = ((NB + 63) // 64 // 2) * 64                                     # middle 64-frame k-block
    ke = min(NB, kb + 64)
    pWf, pbf, _ = R.fc_bwd(sl(dhp, kb, ke), sl(a3p, kb, ke), W['fc.weight'], mask3[kb:ke])
    C.fp32('fc.weight', grads['fc.weight'], dWf, E.left_out(pWf, dWf))
    C.fp32('fc.bias', grads['fc.bias'], dbf, E.left_out(pbf, dbf))
    ref.update({'fc.weight': dWf, 'fc.bias': dbf})
    # ---- conv3 / conv2 / conv1: dgrad on the grid, wgrad + bias from the GPU's own dY
    layers = (('conv3', 'da3', 9, 7, 64, a2p, a2, 1, 1.0), ('conv2', 'da2', 10, 9, 64, a1p, a1, 2, 1.0),
              ('conv1', 'da1', 21, 20, 32, (frames.to(R.F64), None), None, 4, 1.0 / 255.0))
    dref = da3
    parts = R.wgrad_partitions(NB, ctas, split)
    for name, dname, G, V, Cch, xp, xs, stride, scale in layers:
        dy_hi, pad = R.grid_to_nchw(bufs[dname], NB, G, V, Cch)
        C.zero(f'{dname}_padding', pad)
        dy_lo = None
        if split:
            dy_lo, pad_lo = R.grid_to_nchw(lo(dname), NB, G, V, Cch)
            C.zero(f'{dname}_lo_padding', pad_lo)
        C.stored(dname, dy_hi, dy_lo, dref, split=split, terms=dterms)
        dyp = R.pair(dy_hi, dy_lo)
        mask = None if xs is None else (xs[0][:NB] > 0).to(R.F64)
        dW, db, dx = R.conv_bwd(sl(xp, 0, NB), dyp, W[f'{name}.weight'], stride, mask, scale)
        n0, n1, m = R.mid_chunk_frames(NB, G, parts[name])
        m = m[:, :, :V, :V]
        pW, pb, _ = R.conv_bwd(sl(xp, n0, n1), (dyp[0][n0:n1] * m, None if dy_lo is None else dyp[1][n0:n1] * m), W[f'{name}.weight'], stride, None, scale)
        C.fp32(f'{name}.weight', grads[f'{name}.weight'], dW, E.left_out(pW, dW))
        C.fp32(f'{name}.bias', grads[f'{name}.bias'], db, E.left_out(pb, db))
        ref.update({f'{name}.weight': dW, f'{name}.bias': db})
        dref = dx
        if mask is not None:
            dterms = R.abs_terms(lambda d, w: torch.nn.grad.conv2d_input(xp[0][:NB].shape, w, d, stride=stride), dyp, W[f'{name}.weight']) * mask
    C.res['partition'] = parts
    return C, ref


@pytest.mark.parametrize('mode', list(MODES))
@pytest.mark.parametrize('T,B,A', list(SHAPES))
def test_layers_exact(T, B, A, mode, monkeypatch):
    precision, column, fused, replay, poison = MODES[mode]
    monkeypatch.setenv('SRL_NO_COLUMN_FUSION', '0' if column else '1')      # read when the learner is created
    bufs, grads, batch, params = run_step(T, B, A, precision, fused=fused, replay=replay, poison=poison)
    C, _ = check_layers(T, B, A, bufs, grads, params, batch, precision == 'fp32_split', R.cta_counts(R.sm_count(), os.environ))
    C.done(f'T{T}_B{B}_A{A}_{mode}')


def test_layers_exact_after_poisoned_shared_memory():
    """every SM's shared memory filled with NaN patterns before each of three replayed steps (ragged shape): same checks"""
    T, B, A = 7, 19, 18
    bufs, grads, batch, params = run_step(T, B, A, 'bf16', replay=True, poison=True)
    C, _ = check_layers(T, B, A, bufs, grads, params, batch, False, R.cta_counts(R.sm_count(), os.environ))
    C.done(f'T{T}_B{B}_A{A}_bf16_poisoned')


# ------------------------------------------------------------------------------------------------ partition sweep
SWEEP = [  # SRL_WGRAD_CTAS, SRL_BWD_CTAS, SRL_PERSISTENT_CTAS ('' = default; 'sm' = the device's SM count)
    ('8', '16', '16'), ('8', '', ''), ('64', '16', ''), ('64', '', '16'), ('sm', '16', '16'), ('sm', '', ''),
]


def _worker(T, B, A, env_over, out):
    env = dict(os.environ)
    for k in ('SRL_WGRAD_CTAS', 'SRL_BWD_CTAS', 'SRL_PERSISTENT_CTAS', 'SRL_PDL'):
        env.pop(k, None)
    env.update({k: v for k, v in env_over.items() if v != ''})
    os.makedirs(out, exist_ok=True)
    r = subprocess.run([sys.executable, os.path.join(ROOT, 'tests', 'layer_exact_worker.py'), str(T), str(B), str(A), out],
                       cwd=ROOT, env=env, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and 'RESULT ' in r.stdout, (env_over, (r.stdout + r.stderr)[-4000:])
    return {p: torch.load(os.path.join(out, f'{p}.pt')) for p in ('bf16', 'fp32_split')}


def test_partition_sweep(tmp_path):
    """T=20, B=32 with other CTA counts: the partition decides which CTA sums which chunks, so only the fp32 summation order of
    the weight gradients may change -- activations and dY bit-identical, gradients within the fp32 bounds of the fp64 reference;
    with SRL_PDL=0 (no programmatic dependent launch) everything bit-identical to the same partition with it"""
    T, B, A = 20, 32, 6
    NB, sm = T * B, R.sm_count()
    base = {}
    for precision in ('bf16', 'fp32_split'):
        bufs, grads, batch, params = run_step(T, B, A, precision)
        C, ref = check_layers(T, B, A, bufs, grads, params, batch, precision == 'fp32_split', R.cta_counts(sm, {}))
        assert not C.fails, '\n'.join(C.fails)
        base[precision] = ({n: digest(b) for n, b in bufs.items()}, ref)
    table, rec, seen = [], {}, set()
    # the in-process runs of test_layers_exact (default CTA counts) at every shape
    for (t, b, _) in SHAPES:
        for split in (False, True):
            for name, p in R.wgrad_partitions(t * b, R.cta_counts(sm, os.environ), split).items():
                table.append({'T': t, 'B': b, 'env': 'default', 'split': split, 'layer': name, **p})
    runs = [dict(zip(('SRL_WGRAD_CTAS', 'SRL_BWD_CTAS', 'SRL_PERSISTENT_CTAS'), (str(sm) if v == 'sm' else v for v in s))) for s in SWEEP]
    runs.append({'SRL_PDL': '0'})
    runs.append({'SRL_WGRAD_CTAS': '8', 'SRL_BWD_CTAS': '16', 'SRL_PERSISTENT_CTAS': '16', 'SRL_PDL': '0'})
    outs = {}
    for i, env_over in enumerate(runs):
        key = json.dumps(env_over, sort_keys=True)
        got = _worker(T, B, A, env_over, str(tmp_path / f'run{i}'))
        outs[key] = got
        ctas = R.cta_counts(sm, env_over)
        for precision, (hashes, ref) in base.items():
            g = got[precision]
            diff = [n for n in hashes if g['hashes'][n] != hashes[n]]
            assert not diff, (env_over, precision, 'activations / dY differ from the default partition', diff)
            errs = {k: (R.rel_l2(g['grads'][k].reshape(ref[k].shape), ref[k]), R.nerr(g['grads'][k].reshape(ref[k].shape), ref[k])) for k in ref}
            parts = R.wgrad_partitions(NB, ctas, precision == 'fp32_split')
            rec[f'{key} {precision}'] = {'ctas': ctas, 'grad_errors': errs}
            for k, (e, n) in errs.items():
                # the tensor cores' fp32 accumulation error grows linearly with the chunks one CTA sums into its registers
                # (measured, fp32-split conv2: rel-L2 3.6e-6 at 8 chunks per CTA, 2.2e-5 at 63): the bounds scale beyond 16
                grow = max(1.0, parts[k.split('.')[0]]['chunks_per_cta'] / 16) if k.split('.')[0] in parts else 1.0
                assert e <= E.RTOL * grow and n <= E.NTOL * grow, (env_over, precision, k, e, n, grow)
            for name, p in parts.items():
                table.append({'T': T, 'B': B, 'env': key, 'split': precision == 'fp32_split', 'layer': name, **p})
    # PDL off == PDL on, bit for bit, in the same partition
    for pdl_off, twin in ((json.dumps({'SRL_PDL': '0'}), None),
                          (json.dumps(runs[-1], sort_keys=True), json.dumps(dict(zip(('SRL_WGRAD_CTAS', 'SRL_BWD_CTAS', 'SRL_PERSISTENT_CTAS'), SWEEP[0])), sort_keys=True))):
        for precision in ('bf16', 'fp32_split'):
            a = outs[pdl_off][precision]
            if twin is None:        # default partition: the in-process run
                bufs, grads, _, _ = run_step(T, B, A, precision)
                b = {'grads': grads, 'hashes': {n: digest(x) for n, x in bufs.items()}}
            else:
                b = outs[twin][precision]
            assert a['hashes'] == b['hashes'], (pdl_off, precision)
            for k in a['grads']:
                assert torch.equal(a['grads'][k], b['grads'][k]), (pdl_off, precision, k, 'SRL_PDL=0 changed the bits')
    for row in table:
        seen.update(k for k, v in R.regimes(row).items() if v)
    E.record(RESULTS, 'partition_sweep_T20_B32', {'runs': rec, 'partition_table': table, 'regimes_reached': sorted(seen)})
    assert seen == {'one_chunk_per_cta', 'within_ring', 'ring_wraps_twice', 'last_cta_single_chunk'}, sorted(seen)
