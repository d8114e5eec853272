"""The stand-alone optimizer ops of the C ABI and the learner's fused clip + optimizer step share their arithmetic: from the same
parameters, state, gradients and clip coefficient, srl_rmsprop_step / srl_adam_step give the fused step's bits, and
srl_grad_norm_clip_coef gives its norm and clip coefficient (to rounding: the block partials are grouped differently)."""
import pytest
import torch

from oracle import impala_oracle as O
from scalerl_b200 import _lib
from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams

pytestmark = pytest.mark.gpu
T, B, A = 5, 4, 6
MAX_NORMS = [40.0, 1e-3]          # the default, and one every gradient here exceeds (clip coefficient < 1)


def _learner(**kw):
    return B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, **kw), seed=3, process_group=False)


def _batch(seed):
    return {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=seed, done_p=0.1).items()}


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _fused_step(L, seed):
    """forward_backward + apply_gradients; returns the parameters, optimizer state and gradients the step started from"""
    L.forward_backward(_batch(seed))
    state = [s.clone() for s in (L.flat_params, L.opt_state0, L.opt_state1) if s is not None]
    grads = L.flat_grads.clone()
    L.apply_gradients()
    torch.cuda.synchronize()
    return state, grads


@pytest.mark.parametrize('max_grad_norm', MAX_NORMS)
def test_rmsprop_op_matches_fused_step(max_grad_norm):
    L = _learner(max_grad_norm=max_grad_norm)
    (p, v), g = _fused_step(L, seed=11)
    coef = L._coef.clone()
    hp = L.hp
    _lib.check(L._L.srl_rmsprop_step(p.data_ptr(), g.data_ptr(), v.data_ptr(), L.numel, coef.data_ptr(), hp.learning_rate, hp.alpha,
                                     hp.epsilon, _stream()), 'srl_rmsprop_step')
    torch.cuda.synchronize()
    assert torch.equal(p, L.flat_params) and torch.equal(v, L.opt_state0)
    assert (coef[1].item() < 1.0) == (max_grad_norm < 1.0)


@pytest.mark.parametrize('max_grad_norm', MAX_NORMS)
def test_adam_op_matches_fused_step(max_grad_norm):
    L = _learner(optimizer='adam', max_grad_norm=max_grad_norm)
    hp = L.hp
    for step in (1, 2, 3):                      # checked at step 1 and again after two more learner steps
        (p, m, v), g = _fused_step(L, seed=20 + step)
        if step == 2:
            continue
        assert L.device_opt_step() == step
        coef = L._coef.clone()
        _lib.check(L._L.srl_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), L.numel, coef.data_ptr(), hp.learning_rate,
                                      hp.adam_beta1, hp.adam_beta2, hp.adam_eps, step, _stream()), 'srl_adam_step')
        torch.cuda.synchronize()
        assert torch.equal(p, L.flat_params), step
        assert torch.equal(m, L.opt_state0) and torch.equal(v, L.opt_state1), step


@pytest.mark.parametrize('optimizer', ['rmsprop', 'adam'])
@pytest.mark.parametrize('max_grad_norm', MAX_NORMS)
def test_grad_norm_op_matches_fused_step(optimizer, max_grad_norm):
    L = _learner(optimizer=optimizer, max_grad_norm=max_grad_norm)
    _, g = _fused_step(L, seed=7)
    out = torch.zeros(2, device='cuda')
    scratch = torch.zeros(2048, device='cuda')
    _lib.check(L._L.srl_grad_norm_clip_coef(g.data_ptr(), L.numel, max_grad_norm, out.data_ptr(), scratch.data_ptr(), _stream()),
               'srl_grad_norm_clip_coef')
    torch.cuda.synchronize()
    norm, c = L._coef[0].item(), L._coef[1].item()
    assert norm > 0 and abs(out[0].item() - norm) <= 1e-6 * norm, (out[0].item(), norm)
    assert abs(out[1].item() - c) <= 1e-6 * c, (out[1].item(), c)
