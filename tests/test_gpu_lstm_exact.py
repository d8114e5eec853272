"""Every kernel of the LSTM training core (csrc/lstm.cu) against an fp64 evaluation of its own operation on the operands the GPU itself
read (tests/lstm_ref.py), step by step and layer by layer, for the stand-alone core (srl_lstm_core_*, backward over all T1*B rows, with
dhT / dcT / dh0 / dc0) and the learner's context (B200LstmCore, backward over the first (T1-1)*B rows).  Both caller-owned blocks (the
context's arena) start as 0xFF bytes (NaN), and the rows are read back by name (srl_lstm_core_debug_buffer / srl_lstm_debug_buffer).

  * bit-exact: the packed weights (bf16, [4][Hp][Hp], zero padded) and their transposes, xin0 = bf16(core), c_init = c0,
    hm[l][0] = bf16(m_0 h0[l]), hbf = bf16(hseq), hm[l][t+1] = bf16(m_{t+1} hseq[t]), out / hT / cT, db_ih == db_hh, and +0.0 in every
    padding column [H, Hp) of xin0, hm, hbf, gates, cseq, hseq and dgates (a NaN there would enter the next GEMM as 0 * NaN).
  * fp32 results (gate activations, c, h, dWih, dWhh, the bias gradients, dcore, dh0, dc0): rel-L2 <= 2e-5 and normalised max error
    <= 1e-4, the bounds of tests/test_gpu_layer_exact.py.  The gates check the input-projection and recurrent GEMMs plus the cell; c
    and h use the GPU's own gates and c_{t-1}; the gradients use the GPU's own bf16 dgates.  Each GEMM-backed check also measures its
    SENSITIVITY -- how far its reference moves when one unit of work is left out (a 64-row k-block / bias chunk in the middle of the
    rows for the weight and bias gradients, one 64-wide k-block for dcore and the gates) -- and requires at least 20x the rel-L2 bound.
  * dgates (stored bf16): the backward reference carries its own fp64 dc, takes dhm_{t+1} from the GPU's bf16 dgates_{t+1} and Whh,
    and layer 0's dh_out from the GPU's dgates of layer 1 and Wih_1.  Every element is the bf16 rounding of the fp64 value or one ulp
    from it, at most 0.5 % differ, with the cancellation allowance of the sum of |terms| of dh (layer_ref.compare_stored).

Measured on an H100 80GB HBM3 at 700 W: the fp32 results within 2.3e-6 rel-L2 (dWhh over 101 steps; gates 1.5e-7, c 3.3e-8), at
least 8.8x under the bound; the smallest sensitivity 1.8e-2 (gates), 45x the 20x requirement; dgates at most 1 ulp, 0.060 % of elements.
Measured errors, sensitivities and the margin under every bound go to $SRL_RESULTS_DIR/lstm_exact.json when SRL_RESULTS_DIR is set."""
import ctypes as C

import pytest
import torch

from oracle import impala_oracle as O
from scalerl_b200 import _lib
from scalerl_b200.algorithms.utils.atari_model import lstm_block_sizes
from scalerl_b200.lstm import LSTM_PARAM_NAMES, B200LstmCore
from tests import exact as E
from tests import lstm_ref as R

pytestmark = pytest.mark.gpu

F64, BF16 = torch.float64, torch.bfloat16
RESULTS = 'lstm_exact.json'

# (T1, B, A): the edge of the kernels each shape sits on
SHAPES = {
    (5, 3, 6): 'a partial 128-row tile everywhere; NB = 15: one partial k-block and one bias chunk',
    (4, 16, 6): 'NB = 64: exactly one k-block and one bias chunk',
    (1, 7, 6): 'stand-alone only: no recurrence, dhT / dcT seed the only step',
    (2, 130, 31): 'the step GEMMs run two M tiles, the second with 2 rows; H = 544',
    (9, 128, 1): 'B is exactly one tile; H = 514, the widest padding (62 columns)',
    (21, 32, 6): 'the shape of the fp32-torch tests',
    (101, 16, 6): "config 4's rollout: 101 sequential steps, the longest carry; NB is ragged",
}
# stand-alone cases: (T1, B, A, done pattern, nonzero dhT / dcT)
CORE_CASES = [(5, 3, 6, 'edges', True), (4, 16, 6, 'edges', False), (1, 7, 6, 'edges', True), (2, 130, 31, 'edges', False),
              (9, 128, 1, 'edges', True), (21, 32, 6, 'none', False), (101, 16, 6, 'edges', True)]
LEARNER_SHAPES = [s for s in SHAPES if s[0] >= 2]


def _stream():
    return torch.cuda.current_stream().cuda_stream


_summary = E.summary(RESULTS, kind=lambda name: name.rstrip('01'))      # per check kind: the two layers together


# ------------------------------------------------------------------------------------------------ inputs and runs
def _done(T1, B, kind, g):
    """done_p 0.1 plus a done at row 0, two consecutive dones, a column done at every step and a done at the last row"""
    if kind == 'none':
        return torch.zeros(T1, B, dtype=torch.bool)
    d = torch.rand(T1, B, generator=g) < 0.1
    d[0, 0] = True
    if T1 >= 2:
        t0 = max(0, T1 // 2 - 1)
        d[t0, 1] = d[t0 + 1, 1] = True
    d[:, B - 1] = True
    d[T1 - 1, 0] = True
    return d


def _inputs(T1, B, A, seed, dones, seeded):
    H = R.hidden(A)
    g = torch.Generator().manual_seed(1000 + seed)
    x = {'lp': {k: v.cuda() for k, v in O.init_lstm_params(A, seed=seed).items()},
         'core': torch.randn(T1, B, H, generator=g) * 0.5, 'h0': torch.randn(2, B, H, generator=g) * 0.3,
         'c0': torch.randn(2, B, H, generator=g) * 0.3, 'done': _done(T1, B, dones, g), 'dout': torch.randn(T1, B, H, generator=g),
         'dhT': torch.randn(2, B, H, generator=g) if seeded else None, 'dcT': torch.randn(2, B, H, generator=g) if seeded else None}
    return {k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in x.items()}


def _read(ptr, count, dtype):
    out = torch.empty(count, dtype=dtype, device='cuda')
    _lib.check(_lib.lib().srl_memcpy_d2d(out.data_ptr(), ptr, count * out.element_size(), _stream()), 'srl_memcpy_d2d')
    return out


def _core_lookup(T1, B, A, saved, scratch):
    def where(name, layer):
        p, n = C.c_void_p(), C.c_int64()
        _lib.check(_lib.lib().srl_lstm_core_debug_buffer(T1, B, A, saved.data_ptr(), scratch.data_ptr(), name.encode(), layer, C.byref(p),
                                                          C.byref(n)), 'srl_lstm_core_debug_buffer')
        return p.value, n.value
    return where


def _learner_lookup(net):
    def where(name, layer):
        p, n = C.c_void_p(), C.c_int64()
        _lib.check(_lib.lib().srl_lstm_debug_buffer(net._h, name.encode(), layer, C.byref(p), C.byref(n)), 'srl_lstm_debug_buffer')
        return p.value, n.value
    return where


def _rows(where, names):
    """{name: [layer 0, layer 1] or the one row} read back from the device"""
    out = {}
    for name in names:
        got = [_read(*where(name, l), R.row_dtype(name)) for l in ((0, 1) if name in R.LAYER_ROWS else (0,))]
        out[name] = got if name in R.LAYER_ROWS else got[0]
    return out


FWD_ROWS = ('xin0', 'hm', 'hbf', 'Wih', 'WihT', 'Whh', 'WhhT', 'gates', 'cseq', 'hseq', 'c_init')


def _w8(lp):
    return (C.c_void_p * 8)(*[lp[n].data_ptr() for n in LSTM_PARAM_NAMES])


def run_core(T1, B, A, x, blocks=None):
    """one srl_lstm_core_forward + srl_lstm_core_backward on `blocks` (fresh ones filled with 0xFF when None) -> results and rows"""
    H = R.hidden(A)
    if blocks is None:
        sb, kb = lstm_block_sizes(T1, B, A)
        blocks = (torch.full((sb,), 255, dtype=torch.uint8, device='cuda'), torch.full((kb,), 255, dtype=torch.uint8, device='cuda'))
    saved, scratch = blocks
    nan = lambda *s: torch.full(s, float('nan'), device='cuda')
    out, hT, cT = nan(T1, B, H), nan(2, B, H), nan(2, B, H)
    done = x['done'].to(torch.uint8)
    L = _lib.lib()
    _lib.check(L.srl_lstm_core_forward(x['core'].data_ptr(), done.data_ptr(), x['h0'].data_ptr(), x['c0'].data_ptr(), A, T1, B, _w8(x['lp']),
                                       saved.data_ptr(), scratch.data_ptr(), out.data_ptr(), hT.data_ptr(), cT.data_ptr(), _stream()),
               'srl_lstm_core_forward')
    where = _core_lookup(T1, B, A, saved, scratch)
    fw = _rows(where, FWD_ROWS)                   # hseq lives in the scratch block: read before the backward reuses it
    grads = {n: torch.full_like(v, float('nan')) for n, v in x['lp'].items()}
    dcore, dh0, dc0 = nan(T1, B, H), nan(2, B, H), nan(2, B, H)
    opt = lambda t: None if t is None else t.data_ptr()
    _lib.check(L.srl_lstm_core_backward(x['dout'].data_ptr(), opt(x['dhT']), opt(x['dcT']), A, T1, B, saved.data_ptr(), scratch.data_ptr(),
                                        (C.c_void_p * 8)(*[grads[n].data_ptr() for n in LSTM_PARAM_NAMES]), dcore.data_ptr(), dh0.data_ptr(),
                                        dc0.data_ptr(), _stream()), 'srl_lstm_core_backward')
    dgates = _rows(where, ('dgates',))['dgates']
    torch.cuda.synchronize()
    return {'out': out, 'hT': hT, 'cT': cT, 'fw': fw, 'dgates': dgates, 'grads': grads, 'dcore': dcore, 'dh0': dh0, 'dc0': dc0,
            'steps': T1, 'blocks': blocks}


def run_learner(T1, B, A, x):
    """B200LstmCore (srl_lstm_*): forward over T1 steps, backward over the first T1 - 1, its arena filled with 0xFF first"""
    H = R.hidden(A)
    net = B200LstmCore(T1, B, H, state_dict=x['lp'])
    where = _learner_lookup(net)
    ff = torch.full((1 << 20,), 255, dtype=torch.uint8, device='cuda')
    for name in R.LAYER_ROWS + R.SHARED_ROWS:
        for l in ((0, 1) if name in R.LAYER_ROWS else (0,)):
            p, n = where(name, l)
            nbytes = n * R.row_dtype(name).itemsize
            for o in range(0, nbytes, ff.numel()):
                _lib.check(_lib.lib().srl_memcpy_d2d(p + o, ff.data_ptr(), min(ff.numel(), nbytes - o), _stream()), 'srl_memcpy_d2d')
    net.zero_grad()
    out, (hT, cT) = net.forward(x['core'], x['done'], (x['h0'], x['c0']))
    fw = _rows(where, FWD_ROWS)
    dcore = net.backward(x['dout'][:T1 - 1])
    dgates = _rows(where, ('dgates',))['dgates']
    torch.cuda.synchronize()
    res = {'out': out, 'hT': hT, 'cT': cT, 'fw': fw, 'dgates': dgates, 'grads': {n: g.clone() for n, g in net.grads.items()},
           'dcore': dcore, 'dh0': None, 'dc0': None, 'steps': T1 - 1}
    net.close()
    return res


# ------------------------------------------------------------------------------------------------ checks
def check_forward(Ck, T1, B, A, x, r):
    H = R.hidden(A)
    Hp, N1 = R.padded(H), T1 * B
    G = 4 * Hp
    fw, lp, done = r['fw'], x['lp'], x['done']
    m = (~done).to(F64).view(T1, B, 1)
    mf = (~done).float().view(T1, B, 1)
    # packing: the operands the GEMMs read
    for l in (0, 1):
        for nm, key in (('Wih', 'weight_ih'), ('Whh', 'weight_hh')):
            got = fw[nm][l].view(G, Hp)
            Ck.exact(f'{nm}{l}', got, R.pad_weight(lp[f'rnn_layer.{key}_l{l}'].to(BF16), Hp))
            Ck.exact(f'{nm}T{l}', fw[nm + 'T'][l].view(Hp, G), got.t())
        Ck.exact(f'hm_row0_{l}', fw['hm'][l].view(T1, B, Hp)[0], R.pad_cols((mf[0] * x['h0'][l]).to(BF16), Hp))
    xin0 = fw['xin0'].view(T1, B, Hp)
    Ck.exact('xin0', xin0, R.pad_cols(x['core'].to(BF16), Hp))
    Ck.zero('xin0_padding', xin0[..., H:])
    c_init = fw['c_init'].view(2, B, Hp)
    Ck.exact('c_init', c_init[..., :H], x['c0'])             # its padding is never written and never read
    for l in (0, 1):
        xin = (xin0 if l == 0 else fw['hbf'][0].view(T1, B, Hp)).reshape(N1, Hp)
        hm = fw['hm'][l].view(T1, B, Hp)
        Wih, Whh = fw['Wih'][l].view(G, Hp).to(F64), fw['Whh'][l].view(G, Hp).to(F64)
        bias = R.pad_gates(lp[f'rnn_layer.bias_ih_l{l}'].to(F64) + lp[f'rnn_layer.bias_hh_l{l}'].to(F64), H, Hp)
        pre = R.preact(xin, hm.reshape(N1, Hp), Wih, Whh, bias)
        ref = R.activate(pre, H)
        k0, k1 = R.mid_block(Hp)
        part = xin[:, k0:k1].to(F64) @ Wih[:, k0:k1].t()         # one 64-wide k-block of the input projection
        gates = fw['gates'][l].view(N1, G)
        Ck.fp32(f'gates{l}', R.unpad_gates(gates, H), R.unpad_gates(ref, H), E.left_out(R.activate(pre - part, H) - ref, ref))
        Ck.zero(f'gates_padding{l}', R.gate_padding(gates, H))
        gates = gates.view(T1, B, G)
        cseq, hseq = fw['cseq'][l].view(T1, B, Hp), fw['hseq'][l].view(T1, B, Hp)
        c_prev = torch.cat([R.pad_cols(c_init[l, :, :H], Hp)[None], cseq[:-1]])
        c_ref, _ = R.cell(gates, c_prev, m)
        Ck.fp32(f'cseq{l}', cseq[..., :H], c_ref[..., :H])
        o = gates[..., 3 * Hp:].to(F64)
        Ck.fp32(f'hseq{l}', hseq[..., :H], (o * torch.tanh(cseq.to(F64)))[..., :H])
        hbf = fw['hbf'][l].view(T1, B, Hp)
        Ck.exact(f'hbf{l}', hbf, hseq.to(BF16))
        if T1 > 1:
            Ck.exact(f'hm_next{l}', hm[1:], torch.where(done[1:, :, None], 0.0, hseq[:-1]).to(BF16))
        for nm, v in (('hm', hm), ('hbf', hbf), ('cseq', cseq), ('hseq', hseq)):
            Ck.zero(f'{nm}_padding{l}', v[..., H:])
        Ck.exact(f'hT{l}', r['hT'][l], hseq[T1 - 1, :, :H])
        Ck.exact(f'cT{l}', r['cT'][l], cseq[T1 - 1, :, :H])
    Ck.exact('out', r['out'], fw['hseq'][1].view(T1, B, Hp)[..., :H])


def check_backward(Ck, T1, B, A, x, r):
    H = R.hidden(A)
    Hp, steps = R.padded(H), r['steps']
    G, NB = 4 * Hp, steps * B
    fw, lp, done = r['fw'], x['lp'], x['done']
    m = (~done).to(F64).view(T1, B, 1)
    dh_out, dh_terms = R.pad_cols(x['dout'][:steps].to(F64), Hp), None
    for l in (1, 0):
        dg = r['dgates'][l].view(steps, B, G)
        gates, cseq = fw['gates'][l].view(T1, B, G), fw['cseq'][l].view(T1, B, Hp)
        c_init = R.pad_cols(fw['c_init'].view(2, B, Hp)[l, :, :H], Hp)
        Wih, Whh = fw['Wih'][l].view(G, Hp).to(F64), fw['Whh'][l].view(G, Hp).to(F64)
        seed = lambda v: None if v is None else R.pad_cols(v[l], Hp)
        ref = R.bptt_layer(gates, cseq, c_init, m, dh_out, Whh, steps, seed(x['dhT']), seed(x['dcT']), dgates_next=dg, dh_out_terms=dh_terms)
        Ck.stored(f'dgates{l}', R.unpad_gates(dg, H), None, R.unpad_gates(ref['dgates'], H), terms=R.unpad_gates(ref['terms'], H))
        Ck.zero(f'dgates_padding{l}', R.gate_padding(dg, H))
        # weight and bias gradients over rows [0, NB) (the learner's bootstrap row T1-1 must not reach them)
        dgr = dg.reshape(NB, G)
        xin = (fw['xin0'] if l == 0 else fw['hbf'][0]).view(T1 * B, Hp)[:NB]
        hm = fw['hm'][l].view(T1 * B, Hp)[:NB]
        dWih, dWhh, db = R.weight_grads(dgr, xin, hm, 0, NB)
        k0, k1 = R.mid_block(NB)
        pWih, pWhh, pdb = R.weight_grads(dgr, xin, hm, k0, k1)
        g = lambda n: r['grads'][f'rnn_layer.{n}_l{l}']
        Ck.fp32(f'dWih{l}', g('weight_ih'), R.unpad_weight(dWih, H), E.left_out(pWih, dWih))
        Ck.fp32(f'dWhh{l}', g('weight_hh'), R.unpad_weight(dWhh, H), E.left_out(pWhh, dWhh))
        Ck.fp32(f'db{l}', g('bias_ih'), R.unpad_gates(db, H), E.left_out(pdb, db))
        Ck.exact(f'db_hh_equals_db_ih{l}', g('bias_hh'), g('bias_ih'))
        if r['dh0'] is not None:
            Ck.fp32(f'dh0_{l}', r['dh0'][l], ref['dh0'][:, :H])
            Ck.fp32(f'dc0_{l}', r['dc0'][l], ref['dc0'][:, :H])
            Ck.zero(f'dh0_done_rows{l}', r['dh0'][l][done[0]])
            Ck.zero(f'dc0_done_rows{l}', r['dc0'][l][done[0]])
        dx = R.input_grad(dg, Wih)
        if l == 1:
            dh_out, dh_terms = dx, R.input_grad(dg.abs(), Wih.abs())
        else:
            k0, k1 = R.mid_block(G)
            part = dgr[:, k0:k1].to(F64) @ Wih[k0:k1]                # one 64-wide k-block of K = 4Hp
            Ck.fp32('dcore', r['dcore'][:steps], dx[..., :H], E.left_out(part, dx.reshape(NB, Hp)))


def _check(name, T1, B, A, x, r):
    Ck = E.Checker(RESULTS)
    check_forward(Ck, T1, B, A, x, r)
    check_backward(Ck, T1, B, A, x, r)
    Ck.done(name)


# ------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize('T1,B,A,dones,seeded', CORE_CASES)
def test_core_exact(T1, B, A, dones, seeded):
    x = _inputs(T1, B, A, T1 + B + A, dones, seeded)
    _check(f'core_T1{T1}_B{B}_A{A}_{dones}{"_seeded" if seeded else ""}', T1, B, A, x, run_core(T1, B, A, x))


@pytest.mark.parametrize('T1,B,A', LEARNER_SHAPES)
def test_learner_core_exact(T1, B, A):
    x = _inputs(T1, B, A, 7 * T1 + B + A, 'edges', False)
    _check(f'learner_T1{T1}_B{B}_A{A}', T1, B, A, x, run_learner(T1, B, A, x))


@pytest.mark.parametrize('T1,B,A', [(5, 3, 6), (2, 130, 31)])
def test_core_exact_on_reused_blocks(T1, B, A):
    """a second call on the first call's blocks (not refilled) with other inputs, dones and seeds passes the same checks: a read of a
    row the first call left behind would be a mismatch"""
    x1 = _inputs(T1, B, A, 1, 'edges', True)
    first = run_core(T1, B, A, x1)
    x2 = _inputs(T1, B, A, 2, 'edges', False)
    _check(f'core_T1{T1}_B{B}_A{A}_reused_blocks', T1, B, A, x2, run_core(T1, B, A, x2, first['blocks']))
