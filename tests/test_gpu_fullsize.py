"""Whole-learn-step parity at BASELINE.json's sizes (VERDICT r1, item 1a): T=20,B=32,A=6 (configs[1]), T=20,B=64,A=4 (one GPU's
shard of configs[2]) and the LSTM core at T=100 (configs[4]; B=16 keeps the CPU oracle at seconds), against the oracle in BOTH
modes -- bf16-operand emulation (isolates kernel bugs from operand rounding) and plain fp32 (the reference's arithmetic).
Against the emulation the per-tensor gradient rel-L2 is 2-4e-3 (tolerance 5e-3, tighter than test_gpu_parity.py's tiny-batch 2e-2).
Against fp32 the conv/fc gradients differ by 3-7e-2 -- and test_bf16_gap_is_operand_rounding_only shows this is the price of bf16
OPERANDS, not of the kernels: the oracle's own bf16 emulation is as far from its fp32 mode, at every batch size (round 1's
"shrinks with the batch" claim was measured here and is false: 0.076 / 0.044 / 0.094 at B = 2 / 8 / 32).  Parity against the
fp32 reference proper is the job of the fp32-accurate operand mode (tests/test_gpu_precision.py, <= 2e-3).
The measured errors are written to $SRL_RESULTS_DIR/parity_fullsize.json when SRL_RESULTS_DIR is set."""
import os

import numpy as np
import pytest
import torch

from oracle import impala_oracle as O
from tests.exact import record
from tests.helpers import assert_close, rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESULTS = 'parity_fullsize.json'


def _learner(T, B, A, seed, **kw):
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, **kw)
    params = O.init_params(A, seed=seed)
    return B200ImpalaLearner(hp, init_state_dict=params, process_group=False), params


def _errors(L, ref):
    return {k: rel_l2(L.grads[k].cpu(), ref['grads'][k]) for k in O.PARAM_ORDER}


# tolerances: (vs bf16-emulating oracle, vs fp32 oracle) -- gradients per tensor, and logits / vs / losses.
# The fp32 bound is set by the bf16 operands themselves, not by the kernels: the ORACLE's own bf16 emulation differs from its fp32
# mode by 2.7-4.4e-2 rel-L2 on the conv/fc gradients at T=20,B=32 and 3-7e-2 at B=64,A=4 (ReLU-mask flips of near-zero
# pre-activations).  The fp32-accurate operand mode (precision='fp32_split', test_gpu_precision.py) is held to 2e-3 against fp32.
TOL_GRAD_BF16, TOL_GRAD_FP32 = 5e-3, 0.1
TOL_OUT_BF16, TOL_OUT_FP32 = 2e-3, 1e-2


@pytest.mark.parametrize('T,B,A', [(20, 32, 6), (20, 64, 4)])
def test_learn_step_at_baseline_sizes(T, B, A):
    L, params = _learner(T, B, A, 3)
    batch = O.synthetic_batch(T, B, A, seed=7)
    ref_bf = O.learn_step({k: v.clone() for k, v in params.items()}, O.new_opt_state(params), batch, emulate_bf16=True, update=False)
    ref_32 = O.learn_step({k: v.clone() for k, v in params.items()}, O.new_opt_state(params), batch, use_autograd=True, update=False)
    stats = L.learn({k: v.cuda() for k, v in batch.items()})
    lg = L.debug_buffer('logits').view(T + 1, B, A).cpu()
    rec = {'grad_vs_bf16_oracle': _errors(L, ref_bf), 'grad_vs_fp32_oracle': _errors(L, ref_32),
           'logits_vs_bf16': rel_l2(lg, ref_bf['policy_logits']), 'logits_vs_fp32': rel_l2(lg, ref_32['policy_logits']),
           'vs_vs_bf16': rel_l2(L._vs.cpu(), ref_bf['vs']), 'vs_vs_fp32': rel_l2(L._vs.cpu(), ref_32['vs']),
           'total_loss': [stats['total_loss'], ref_bf['total_loss'], ref_32['total_loss']],
           'grad_norm': [stats['grad_norm'], ref_bf['grad_norm'], ref_32['grad_norm']]}
    record(RESULTS, f'learn_T{T}_B{B}_A{A}', rec)
    assert rec['logits_vs_bf16'] < TOL_OUT_BF16 and rec['logits_vs_fp32'] < TOL_OUT_FP32, rec
    assert rec['vs_vs_bf16'] < TOL_OUT_BF16 and rec['vs_vs_fp32'] < TOL_OUT_FP32, rec
    for k in ('pg_loss', 'baseline_loss', 'entropy_loss', 'total_loss'):
        assert abs(stats[k] - ref_bf[k]) <= TOL_OUT_BF16 * max(1.0, abs(ref_bf[k])), (k, stats[k], ref_bf[k])
        assert abs(stats[k] - ref_32[k]) <= TOL_OUT_FP32 * max(1.0, abs(ref_32[k])), (k, stats[k], ref_32[k])
    for k in O.PARAM_ORDER:
        assert rec['grad_vs_bf16_oracle'][k] < TOL_GRAD_BF16, (k, rec['grad_vs_bf16_oracle'])
        assert rec['grad_vs_fp32_oracle'][k] < TOL_GRAD_FP32, (k, rec['grad_vs_fp32_oracle'])
    assert abs(stats['grad_norm'] - ref_32['grad_norm']) <= 5e-3 * ref_32['grad_norm']
    assert np.allclose(stats['episode_returns'], ref_32['episode_returns'])
    # V-trace on IDENTICAL inputs (the learner's own logits / baseline): north_star's 1e-4
    bs = L.debug_buffer('baseline').view(T + 1, B).cpu()
    rewards = torch.clamp(batch['reward'][1:], -1, 1)
    discounts = (~batch['done'][1:]).float() * 0.99
    vs, pg, *_ = O.vtrace_from_logits(batch['policy_logits'][1:], lg[:-1], batch['action'][1:], discounts, rewards, bs[:-1], bs[-1])
    assert_close(L._vs, vs, 1e-4, 'vs'); assert_close(L._pg_adv, pg, 1e-4, 'pg_adv')


def test_bf16_gap_is_operand_rounding_only():
    """the distance of the bf16 kernels from fp32 arithmetic == the distance of the oracle's bf16-operand EMULATION from its own
    fp32 mode, tensor by tensor and at every batch size: the kernels add nothing beyond the rounding of their operands"""
    T, A = 20, 6
    rec = {}
    for B in (2, 8, 32):
        L, params = _learner(T, B, A, 3)
        batch = O.synthetic_batch(T, B, A, seed=11)
        cp = lambda: {k: v.clone() for k, v in params.items()}
        ref32 = O.learn_step(cp(), O.new_opt_state(params), batch, use_autograd=True, update=False)
        refbf = O.learn_step(cp(), O.new_opt_state(params), batch, emulate_bf16=True, update=False)
        L.learn({k: v.cuda() for k, v in batch.items()})
        kern = _errors(L, ref32)
        emul = {k: rel_l2(refbf['grads'][k], ref32['grads'][k]) for k in O.PARAM_ORDER}
        rec[str(B)] = {'kernel_vs_fp32_max': max(kern.values()), 'emulation_vs_fp32_max': max(emul.values())}
        for k in O.PARAM_ORDER:
            assert kern[k] <= 1.3 * emul[k] + 2e-3, (B, k, kern[k], emul[k])
        L.close()
    record(RESULTS, 'bf16_gap_kernel_vs_emulation_T20', rec)


def test_lstm_learn_step_T100():
    """configs[4]'s rollout length through encoder -> LSTM -> heads -> BPTT (atari_model.py:109-120), fp32 oracle"""
    T, B, A = 100, 16, 6
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    params, lp = O.init_params(A, seed=5), O.init_lstm_params(A, seed=5)
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, use_lstm=True), init_state_dict={**params, **lp}, process_group=False)
    batch = O.synthetic_batch(T, B, A, seed=13, done_p=0.02)
    rng = np.random.RandomState(2)
    state = tuple(torch.from_numpy(rng.randn(2, B, 513 + A).astype(np.float32) * 0.3) for _ in range(2))
    ref = O.learn_step_lstm(params, lp, batch, state)
    stats = L.learn({k: v.cuda() for k, v in batch.items()}, (state[0].cuda(), state[1].cuda()))
    allg = {**ref['grads'], **ref['lstm_grads']}
    errs = {k: rel_l2(L.grads[k].cpu(), v) for k, v in allg.items()}
    rec = {'grad_vs_fp32_oracle': errs, 'vs': rel_l2(L._vs.cpu(), ref['vs']), 'total_loss': [stats['total_loss'], ref['total_loss']]}
    record(RESULTS, f'lstm_learn_T{T}_B{B}', rec)
    assert abs(stats['total_loss'] - ref['total_loss']) <= 1e-2 * max(1.0, abs(ref['total_loss'])), rec['total_loss']
    assert rec['vs'] < 1e-2
    for k, e in errs.items():       # encoder tensors: bf16 operand bound (no LSTM emulation oracle); LSTM / head tensors far tighter
        assert e < (0.1 if k.startswith(('conv', 'fc')) else 1e-2), (k, e)
