"""The fp32-accurate operand mode (ImpalaHParams(precision='fp32_split'), srl_config_t.precision = 1; SURVEY.md §7.9):
whole-step parity against the REFERENCE-generated goldens and the fp32 oracle at tolerances two to four orders tighter than
the bf16 mode's (VERDICT r1 item 1b).

What is measured ($SRL_RESULTS_DIR/parity_fullsize.json, keys split_*): every forward quantity (activations, logits, baseline, vs)
agrees to 2e-6 .. 1e-5 rel-L2, and so does every gradient -- EXCEPT when a ReLU unit's pre-activation lies within ~1e-5 of zero, so
that 16-bit operands put it on the other side than fp32 does.  Such a tie flips one mask bit and moves the conv gradients by
1e-3 .. 8e-3 on a 20-frame batch (the fp32 reference against its own fp64 evaluation shows the same effect one decade lower).  The
tests therefore (a) count the mask disagreements against fp32 pre-activations computed on the CPU, (b) require every disagreeing
unit to be a genuine tie (|z| < 1e-4 rms), (c) hold the gradients to 1e-4 when no unit flipped and to 2e-2 otherwise, and at
BASELINE's T=20,B=32 to the 2e-3 the round-1 verdict asked for (measured 1.2-1.7e-3; the CPU emulation of 16-bit operands predicts
1.0-1.5e-3)."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import impala_oracle as O
from tests import layer_ref as R
from tests.conftest import GOLDEN
from tests.exact import record
from tests.helpers import assert_close, rel_l2, strided_sample

pytestmark = pytest.mark.gpu


def _learner(T, B, A, seed, **kw):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, precision='fp32_split', **kw)
    params = O.init_params(A, seed=seed)
    return B200ImpalaLearner(hp, init_state_dict=params, process_group=False), params


def _mask_flips(L, params, batch, T, B):
    """ReLU masks of the learner (hi tensors > 0) vs fp32 pre-activations on the CPU -> (flipped units, units, worst |z|/rms of a flipped unit)"""
    import torch.nn.functional as F
    NF = (T + 1) * B
    x = batch['obs'].reshape(NF, 4, 84, 84).float() / 255.0
    z1 = F.conv2d(x, params['conv1.weight'], params['conv1.bias'], stride=4)
    z2 = F.conv2d(F.relu(z1), params['conv2.weight'], params['conv2.bias'], stride=2)
    z3 = F.conv2d(F.relu(z2), params['conv3.weight'], params['conv3.bias'], stride=1)
    zh = F.linear(F.relu(z3).reshape(NF, -1), params['fc.weight'], params['fc.bias'])
    g1 = R.a1_planes_to_nchw(L.debug_buffer('a1').float().cpu(), NF)
    g2 = R.nhwc_to_nchw(L.debug_buffer('a2').float().cpu(), NF, 9)
    g3 = R.nhwc_to_nchw(L.debug_buffer('a3').float().cpu(), NF, 7)
    gh = L.debug_buffer('h').view(NF, 512).cpu()
    flips, units, worst = 0, 0, 0.0
    for z, g in ((z1, g1), (z2, g2), (z3, g3), (zh, gh)):
        bad = (z > 0) != (g > 0)
        flips += int(bad.sum())
        units += z.numel()
        if bad.any():
            worst = max(worst, float(z[bad].abs().max() / z.pow(2).mean().sqrt()))
    return flips, units, worst


def _grad_tol(flips):
    return 1e-4 if flips == 0 else 2e-2


@pytest.mark.parametrize('fusion', ['column_kernel', 'three_kernels'])
@pytest.mark.parametrize('name', ['t5b4a6', 't3b5a4'])
def test_split_mode_vs_reference_goldens(name, fusion, monkeypatch):
    """goldens written by oracle/make_golden.py from the reference's own modules (fp32 torch autograd)"""
    monkeypatch.setenv('SRL_NO_COLUMN_FUSION', '0' if fusion == 'column_kernel' else '1')
    g = np.load(os.path.join(GOLDEN, f'learn_{name}.npz'))
    T, B, A, seed, steps, clip = [int(v) for v in g['meta']]
    L, params = _learner(T, B, A, seed, reward_clipping='abs_one' if clip else 'none')
    batch = O.synthetic_batch(T, B, A, seed=seed * 10)
    stats = L.learn({k: v.cuda() for k, v in batch.items()})
    lg = L.debug_buffer('logits').view(T + 1, B, A).cpu()
    errs = {'logits': rel_l2(lg, g['s0_policy_logits']), 'baseline': rel_l2(L.debug_buffer('baseline').view(T + 1, B).cpu(), g['s0_baseline']),
            'vs': rel_l2(L._vs.cpu(), g['s0_vs'])}
    for k in O.PARAM_ORDER:
        errs['grad_' + k] = rel_l2(strided_sample(L.grads[k].reshape(-1).cpu()), g['s0_gradsamp_' + k])
    flips, units, worst = _mask_flips(L, params, batch, T, B)
    errs.update(relu_mask_flips=flips, relu_units=units, worst_flipped_margin=worst)
    record('parity_fullsize.json', f'split_golden_{name}_{fusion}', errs)
    assert errs['logits'] < 1e-5 and errs['baseline'] < 1e-5 and errs['vs'] < 1e-5, errs
    assert abs(stats['total_loss'] - g['s0_losses'][3]) <= 1e-5 * max(1.0, abs(g['s0_losses'][3]))
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)       # only genuine ties may flip
    tol = _grad_tol(flips)
    for k in O.PARAM_ORDER:
        assert errs['grad_' + k] < tol, (k, flips, errs)
        gn = float(L.grads[k].double().norm())
        assert abs(gn - g['s0_gradnorm_' + k][0]) <= tol * g['s0_gradnorm_' + k][0] + 1e-7, k


@pytest.mark.parametrize('T,B,A', [(20, 32, 6), (7, 19, 4)])
def test_split_mode_vs_fp32_oracle(T, B, A):
    L, params = _learner(T, B, A, 3)
    batch = O.synthetic_batch(T, B, A, seed=7, done_p=0.05)
    p0 = {k: v.clone() for k, v in params.items()}
    opt = O.new_opt_state(params)
    ref = O.learn_step(p0, opt, batch, use_autograd=True)                      # fp32 reference arithmetic incl. the RMSprop update
    stats = L.learn({k: v.cuda() for k, v in batch.items()})
    lg = L.debug_buffer('logits').view(T + 1, B, A).cpu()
    errs = {k: rel_l2(L.grads[k].cpu(), ref['grads'][k]) for k in O.PARAM_ORDER}
    errs['logits'] = rel_l2(lg, ref['policy_logits'])
    errs['vs'] = rel_l2(L._vs.cpu(), ref['vs'])
    flips, units, worst = _mask_flips(L, params, batch, T, B)
    errs.update(relu_mask_flips=flips, relu_units=units, worst_flipped_margin=worst)
    record('parity_fullsize.json', f'split_vs_fp32_T{T}_B{B}_A{A}', errs)
    assert errs['logits'] < 1e-5 and errs['vs'] < 1e-5, errs
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)
    tol = 2e-3 if (T, B) == (20, 32) else _grad_tol(flips)          # BASELINE size: the round-1 verdict's bound, ties included
    for k in O.PARAM_ORDER:
        assert errs[k] < tol, (k, flips, errs)
    for k in ('pg_loss', 'baseline_loss', 'entropy_loss', 'total_loss'):
        assert abs(stats[k] - ref[k]) <= 1e-4 * max(1.0, abs(ref[k])), k
    assert abs(stats['grad_norm'] - ref['grad_norm']) <= 1e-4 * ref['grad_norm']
    # post-step weights: RMSprop normalises the step, so compare through the oracle's own update on the DEVICE gradients
    g_dev = {k: L.grads[k].cpu().clone() for k in O.PARAM_ORDER}
    O.clip_grad_norm(g_dev, 40.0)
    before = {k: v.clone() for k, v in params.items()}
    O.rmsprop_step(before, g_dev, O.new_opt_state(params)['square_avg'], 1e-4, 0.99, 1e-5)
    for k in O.PARAM_ORDER:
        assert_close(L.params[k], before[k], 2e-6, f'post-step {k}')


def test_split_mode_rejects_lstm():
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    with pytest.raises(ValueError):
        B200ImpalaLearner(ImpalaHParams(rollout_length=3, batch_size=2, use_lstm=True, precision='fp32_split'), process_group=False)
