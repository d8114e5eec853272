"""CPU: the fp64 per-step LSTM references of tests/lstm_ref.py, chained over T1 steps in the kernels' padded layouts, equal torch
autograd through oracle.impala_oracle.lstm_core_forward in float64 -- outputs, state, dcore, dh0 / dc0 and all 8 parameter gradients
-- over both row ranges the kernels run (NB = T1*B: the stand-alone core; NB = (T1-1)*B: the learner).  The GPU check
(tests/test_gpu_lstm_exact.py) relies on these functions, so they are proven here first."""
import pytest
import torch

from oracle import impala_oracle as O
from tests import layer_ref as LR
from tests import lstm_ref as R

F64 = torch.float64
TOL = 1e-12


def test_layout_helpers():
    for A in range(1, 32):
        assert R.padded(R.hidden(A)) == 576, A
    H, Hp = 7, 64
    w = torch.arange(4 * H * H, dtype=F64).reshape(4 * H, H) + 1
    wp = R.pad_weight(w, Hp)
    assert wp.shape == (4 * Hp, Hp)
    for q in range(4):
        assert torch.equal(wp[q * Hp:q * Hp + H, :H], w[q * H:(q + 1) * H])
    assert int((wp != 0).sum()) == w.numel()
    assert torch.equal(R.unpad_weight(wp, H), w)
    v = torch.arange(2 * 4 * H, dtype=F64).reshape(2, 4 * H) + 1
    vp = R.pad_gates(v, H, Hp)
    assert vp.shape == (2, 4 * Hp) and torch.equal(R.unpad_gates(vp, H), v)
    assert torch.equal(vp.reshape(2, 4, Hp)[:, 2, :H], v[:, 2 * H:3 * H])
    assert not R.gate_padding(vp, H).any()
    assert R.mid_block(15) == (0, 15) and R.mid_block(64) == (0, 64) and R.mid_block(1616) == (832, 896)
    assert R.mid_block(4 * 576) == (1152, 1216) and R.mid_block(576) == (256, 320)


def _done(T1, B, g):
    """done_p 0.1 with a done at row 0, two consecutive dones, an always-done column and a done at the last row"""
    d = torch.rand(T1, B, generator=g) < 0.1
    d[0, 0] = True
    d[2, 1] = d[3, 1] = True
    d[:, B - 1] = True
    d[T1 - 1, 2] = True
    return d


def _chain(lp, core, done, h0, c0, dout, dhT, dcT, steps):
    """the per-step references chained over the sequence (padded layouts, no rounding anywhere)"""
    T1, B, H = core.shape
    Hp = R.padded(H)
    NB = steps * B
    m = (~done).to(F64)[..., None]
    pw = lambda l, n: lp[f'rnn_layer.{n}_l{l}']
    W = [(R.pad_weight(pw(l, 'weight_ih'), Hp), R.pad_weight(pw(l, 'weight_hh'), Hp), R.pad_gates(pw(l, 'bias_ih') + pw(l, 'bias_hh'), H, Hp))
         for l in (0, 1)]
    xin, fw = R.pad_cols(core, Hp), []
    for l in (0, 1):
        hm, gates, cs, hs = R.forward_layer(xin, W[l][0], W[l][1], W[l][2], R.pad_cols(h0[l], Hp), R.pad_cols(c0[l], Hp), m, H)
        assert not R.gate_padding(gates, H).any() and not cs[..., H:].any() and not hs[..., H:].any()
        fw.append((xin, hm, gates, cs, hs))
        xin = hs
    res = {'out': fw[1][4][..., :H], 'hT': torch.stack([fw[l][4][-1, :, :H] for l in (0, 1)]),
           'cT': torch.stack([fw[l][3][-1, :, :H] for l in (0, 1)])}
    dh_out = R.pad_cols(dout[:steps], Hp)
    dh0, dc0 = [None, None], [None, None]
    for l in (1, 0):
        x, hm, gates, cs, _ = fw[l]
        pad = lambda v: None if v is None else R.pad_cols(v[l], Hp)
        r = R.bptt_layer(gates, cs, R.pad_cols(c0[l], Hp), m, dh_out, W[l][1], steps, pad(dhT), pad(dcT))
        assert bool((r['terms'] >= r['dgates'].abs() * (1 - 1e-12)).all())
        assert not R.gate_padding(r['dgates'], H).any()
        dg = r['dgates'].reshape(NB, 4 * Hp)
        dWih, dWhh, db = R.weight_grads(dg, x.reshape(-1, Hp), hm.reshape(-1, Hp), 0, NB)
        res[f'rnn_layer.weight_ih_l{l}'] = R.unpad_weight(dWih, H)
        res[f'rnn_layer.weight_hh_l{l}'] = R.unpad_weight(dWhh, H)
        res[f'rnn_layer.bias_ih_l{l}'] = res[f'rnn_layer.bias_hh_l{l}'] = R.unpad_gates(db, H)
        dh0[l], dc0[l] = r['dh0'][:, :H], r['dc0'][:, :H]
        dh_out = R.input_grad(r['dgates'], W[l][0])
    res.update(dcore=dh_out[..., :H], dh0=torch.stack(dh0), dc0=torch.stack(dc0))
    return res


@pytest.mark.parametrize('rows,seeds,dones', [('core', True, 'pattern'), ('core', False, 'pattern'), ('learner', False, 'pattern'),
                                              ('core', True, 'none'), ('learner', False, 'none')])
def test_chained_steps_equal_autograd(rows, seeds, dones):
    T1, B, A = 6, 5, 3
    H = R.hidden(A)
    g = torch.Generator().manual_seed(11)
    lp = {k: v.to(F64).requires_grad_(True) for k, v in O.init_lstm_params(A, seed=2).items()}
    core = (torch.randn(T1, B, H, generator=g, dtype=F64) * 0.5).requires_grad_(True)
    h0 = (torch.randn(2, B, H, generator=g, dtype=F64) * 0.3).requires_grad_(True)
    c0 = (torch.randn(2, B, H, generator=g, dtype=F64) * 0.3).requires_grad_(True)
    done = _done(T1, B, g) if dones == 'pattern' else torch.zeros(T1, B, dtype=torch.bool)
    dout = torch.randn(T1, B, H, generator=g, dtype=F64)
    dhT = torch.randn(2, B, H, generator=g, dtype=F64) if seeds else None
    dcT = torch.randn(2, B, H, generator=g, dtype=F64) if seeds else None
    steps = T1 if rows == 'core' else T1 - 1
    out, (hT, cT) = O.lstm_core_forward(lp, core, done, (h0, c0))
    loss = (out[:steps] * dout[:steps]).sum()
    if seeds:
        loss = loss + (hT * dhT).sum() + (cT * dcT).sum()
    loss.backward()
    want = {'out': out, 'hT': hT, 'cT': cT, 'dcore': core.grad[:steps], 'dh0': h0.grad, 'dc0': c0.grad,
            **{k: v.grad for k, v in lp.items()}}
    with torch.no_grad():
        got = _chain({k: v.detach() for k, v in lp.items()}, core.detach(), done, h0.detach(), c0.detach(), dout, dhT, dcT, steps)
    assert set(got) == set(want)
    for k in want:
        assert got[k].shape == want[k].shape, k
        e = LR.nerr(got[k], want[k].detach())
        assert e <= TOL, (k, e)
    # the dones reach the gradients they must: a column done at every step has no gradient into the initial state
    if dones == 'pattern':
        assert not got['dh0'][:, done[0]].any() and not got['dc0'][:, done[0]].any()
        assert bool(got['dh0'][:, ~done[0]].abs().sum() > 0)
