"""Torch-tensor front end of the C ABI (device memory + streams are torch's; the math is ours).

Mirrors the reference's operator surface for the hot path:
  from_importance_weights / from_logits  <->  scalerl/algorithms/impala/vtrace.py:43-172
  impala_loss_and_head_grads            <->  scalerl/algorithms/impala/loss_fn.py:5-23 + impala_atari.py:293-330
Errors follow the reference's Python behaviour: ValueError for bad arguments, RuntimeError for CUDA failures.
"""
import collections

import torch

from . import _lib

VTraceFromLogitsReturns = collections.namedtuple(
    'VTraceFromLogitsReturns',
    ['vs', 'pg_advantages', 'log_rhos', 'behavior_action_log_probs', 'target_action_log_probs'])
VTraceReturns = collections.namedtuple('VTraceReturns', 'vs pg_advantages')


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _f32(t, name):
    if not t.is_cuda:
        raise ValueError(f'{name} must be a CUDA tensor (scalerl_b200 has no CPU path)')
    if t.dtype != torch.float32:
        raise ValueError(f'{name} must be float32, got {t.dtype}')
    return t.contiguous()


def _clip(v):
    """a clip threshold for the C ABI: None (no clipping) is -1; a number must be >= 0 (a negative or NaN one is refused, not read as
    None)"""
    if v is None:
        return -1.0
    v = float(v)
    if not v >= 0.0:
        raise ValueError(f'clip thresholds must be >= 0 or None, got {v}')
    return v


@torch.no_grad()
def from_importance_weights(log_rhos, discounts, rewards, values, bootstrap_value,
                            clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0, variant=0):
    """vtrace.from_importance_weights (vtrace.py:78-172) for [T,B] inputs -> VTraceReturns(vs, pg_advantages)."""
    log_rhos, discounts, rewards, values = [_f32(t, n) for t, n in
                                            ((log_rhos, 'log_rhos'), (discounts, 'discounts'), (rewards, 'rewards'), (values, 'values'))]
    bootstrap_value = _f32(bootstrap_value, 'bootstrap_value')
    if log_rhos.dim() != 2:
        raise ValueError('log_rhos must be [T, B]')
    T, B = log_rhos.shape
    for t, n in ((discounts, 'discounts'), (rewards, 'rewards'), (values, 'values')):
        if tuple(t.shape) != (T, B):
            raise ValueError(f'{n} has shape {tuple(t.shape)}, expected {(T, B)}')
    if tuple(bootstrap_value.shape) != (B,):
        raise ValueError(f'bootstrap_value has shape {tuple(bootstrap_value.shape)}, expected {(B,)}')
    vs = torch.empty_like(log_rhos)
    pg = torch.empty_like(log_rhos)
    _lib.check(_lib.lib().srl_vtrace_from_importance_weights(
        log_rhos.data_ptr(), discounts.data_ptr(), rewards.data_ptr(), values.data_ptr(), bootstrap_value.data_ptr(),
        T, B, _clip(clip_rho_threshold), _clip(clip_pg_rho_threshold), vs.data_ptr(), pg.data_ptr(), int(variant), _stream()),
        'vtrace_from_importance_weights')
    return VTraceReturns(vs=vs, pg_advantages=pg)


@torch.no_grad()
def _from_logits_raw(behavior_policy_logits, target_policy_logits, actions, discounts, rewards, values, bootstrap_value,
                     clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0):
    """vtrace.from_logits (vtrace.py:43-75): logits [T,B,A], actions int64 [T,B]; no autograd (see from_logits)."""
    bl = _f32(behavior_policy_logits, 'behavior_policy_logits')
    tl = _f32(target_policy_logits, 'target_policy_logits')
    discounts, rewards, values = _f32(discounts, 'discounts'), _f32(rewards, 'rewards'), _f32(values, 'values')
    bootstrap_value = _f32(bootstrap_value, 'bootstrap_value')
    if actions.dtype != torch.int64:
        raise ValueError('actions must be int64')
    actions = actions.contiguous()
    if tl.dim() != 3 or bl.shape != tl.shape:
        raise ValueError('policy logits must both be [T, B, A]')
    T, B, A = tl.shape
    outs = [torch.empty(T, B, device=tl.device, dtype=torch.float32) for _ in range(5)]
    _lib.check(_lib.lib().srl_vtrace_from_logits(
        bl.data_ptr(), tl.data_ptr(), actions.data_ptr(), discounts.data_ptr(), rewards.data_ptr(), values.data_ptr(),
        bootstrap_value.data_ptr(), T, B, A, _clip(clip_rho_threshold), _clip(clip_pg_rho_threshold),
        *[o.data_ptr() for o in outs], _stream()), 'vtrace_from_logits')
    return VTraceFromLogitsReturns(vs=outs[0], pg_advantages=outs[1], log_rhos=outs[2],
                                   behavior_action_log_probs=outs[3], target_action_log_probs=outs[4])


# ------------------------------------------------------------------------------------------------------------------
# differentiable row ops (srl_policy_rows_forward / _backward, srl_reduce_sum) and the autograd functions built on them
# ------------------------------------------------------------------------------------------------------------------
def _rows(logits, actions):
    lg = _f32(logits.detach(), 'logits')
    A = lg.shape[-1]
    lg2 = lg.reshape(-1, A)
    act = None
    if actions is not None:
        if actions.dtype != torch.int64:
            raise ValueError('actions must be int64')
        act = actions.detach().reshape(-1).contiguous()
        if act.numel() != lg2.shape[0]:
            raise ValueError(f'actions has {act.numel()} elements for {lg2.shape[0]} logit rows')
    return lg2, act, A


@torch.no_grad()
def policy_rows_forward(logits, actions=None, want_logp=True, want_entropy=False):
    """-> (logp [rows] | None, ent [rows] | None): log pi(a) and sum_a p log p per row of [..., A] logits"""
    lg2, act, A = _rows(logits, actions)
    N = lg2.shape[0]
    logp = torch.empty(N, device=lg2.device) if want_logp else None
    ent = torch.empty(N, device=lg2.device) if want_entropy else None
    _lib.check(_lib.lib().srl_policy_rows_forward(lg2.data_ptr(), act.data_ptr() if act is not None else None, N, A,
                                                  logp.data_ptr() if want_logp else None, ent.data_ptr() if want_entropy else None, _stream()),
               'policy_rows_forward')
    return logp, ent


@torch.no_grad()
def policy_rows_backward(logits, actions=None, w_logp=None, w_entropy=None):
    """d/dlogits of sum_n w_logp[n] * logp[n] + w_entropy[n] * ent[n]  -> tensor shaped like logits"""
    lg2, act, A = _rows(logits, actions)
    N = lg2.shape[0]
    wl = _f32(w_logp.detach().reshape(-1), 'w_logp') if w_logp is not None else None
    we = _f32(w_entropy.detach().reshape(-1), 'w_entropy') if w_entropy is not None else None
    for w in (wl, we):
        if w is not None and w.numel() != N:
            raise ValueError('weight arrays need one entry per logit row')
    d = torch.empty_like(lg2)
    _lib.check(_lib.lib().srl_policy_rows_backward(lg2.data_ptr(), act.data_ptr() if act is not None else None,
                                                   wl.data_ptr() if wl is not None else None, we.data_ptr() if we is not None else None,
                                                   N, A, d.data_ptr(), _stream()), 'policy_rows_backward')
    return d.view(logits.shape)


@torch.no_grad()
def reduce_sum(x, square=False, scale=1.0):
    x = _f32(x.detach(), 'x').reshape(-1)
    out = torch.empty((), device=x.device)
    _lib.check(_lib.lib().srl_reduce_sum(x.data_ptr(), x.numel(), 1 if square else 0, float(scale), out.data_ptr(), _stream()), 'reduce_sum')
    return out


class _ActionLogProbs(torch.autograd.Function):
    """vtrace.action_log_probs (vtrace.py:31-40) with its gradient g * (onehot(a) - softmax)"""

    @staticmethod
    def forward(ctx, logits, actions):
        ctx.save_for_backward(logits, actions)
        return policy_rows_forward(logits, actions)[0].view(actions.shape)

    @staticmethod
    def backward(ctx, g):
        logits, actions = ctx.saved_tensors
        return policy_rows_backward(logits, actions, w_logp=g.contiguous()), None


class _PolicyGradientLoss(torch.autograd.Function):
    """loss_fn.compute_policy_gradient_loss (loss_fn.py:16-23): sum(-log pi(a) * adv), advantages detached"""

    @staticmethod
    def forward(ctx, logits, actions, advantages):
        adv = _f32(advantages.detach(), 'advantages')
        ctx.save_for_backward(logits, actions, adv)
        logp = policy_rows_forward(logits, actions)[0]
        return reduce_sum(logp * adv.reshape(-1), scale=-1.0)

    @staticmethod
    def backward(ctx, g):
        logits, actions, adv = ctx.saved_tensors
        return policy_rows_backward(logits, actions, w_logp=(-g) * adv.reshape(-1)), None, None


class _EntropyLoss(torch.autograd.Function):
    """loss_fn.compute_entropy_loss (loss_fn.py:9-13): sum p log p, gradient p (log p - sum p log p)"""

    @staticmethod
    def forward(ctx, logits):
        ctx.save_for_backward(logits)
        return reduce_sum(policy_rows_forward(logits, None, want_logp=False, want_entropy=True)[1])

    @staticmethod
    def backward(ctx, g):
        (logits,) = ctx.saved_tensors
        n = logits.numel() // logits.shape[-1]
        return policy_rows_backward(logits, None, w_entropy=g.expand(n).contiguous())


class _BaselineLoss(torch.autograd.Function):
    """loss_fn.compute_baseline_loss (loss_fn.py:5-6): 0.5 * sum(adv^2), gradient adv"""

    @staticmethod
    def forward(ctx, advantages):
        ctx.save_for_backward(advantages)
        return reduce_sum(advantages, square=True, scale=0.5)

    @staticmethod
    def backward(ctx, g):
        (adv,) = ctx.saved_tensors
        return g * adv


class _FromLogits(torch.autograd.Function):
    """vtrace.from_logits (vtrace.py:43-75).  As in the reference, vs / pg_advantages carry no graph (from_importance_weights
    is @torch.no_grad, vtrace.py:78) while log_rhos / *_action_log_probs are differentiable w.r.t. the logits."""

    @staticmethod
    def forward(ctx, bl, tl, actions, discounts, rewards, values, bootstrap_value, clip_rho, clip_pg):
        r = _from_logits_raw(bl, tl, actions, discounts, rewards, values, bootstrap_value, clip_rho, clip_pg)
        ctx.save_for_backward(bl, tl, actions)
        ctx.mark_non_differentiable(r.vs, r.pg_advantages)
        return tuple(r)

    @staticmethod
    def backward(ctx, g_vs, g_pg, g_lr, g_balp, g_talp):
        bl, tl, actions = ctx.saved_tensors
        zero = torch.zeros(actions.shape, device=tl.device)
        g_lr = zero if g_lr is None else g_lr
        d_tl = d_bl = None
        if ctx.needs_input_grad[1]:
            d_tl = policy_rows_backward(tl, actions, w_logp=(g_lr + (zero if g_talp is None else g_talp)).contiguous())
        if ctx.needs_input_grad[0]:
            d_bl = policy_rows_backward(bl, actions, w_logp=((zero if g_balp is None else g_balp) - g_lr).contiguous())
        return d_bl, d_tl, None, None, None, None, None, None, None


def action_log_probs(policy_logits, actions):
    """vtrace.action_log_probs (vtrace.py:31-40), differentiable w.r.t. policy_logits"""
    return _ActionLogProbs.apply(policy_logits, actions)


def from_logits(behavior_policy_logits, target_policy_logits, actions, discounts, rewards, values, bootstrap_value,
                clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0):
    """vtrace.from_logits (vtrace.py:43-75): logits [T,B,A], actions int64 [T,B] -> VTraceFromLogitsReturns."""
    return VTraceFromLogitsReturns(*_FromLogits.apply(behavior_policy_logits, target_policy_logits, actions, discounts, rewards, values,
                                                      bootstrap_value, clip_rho_threshold, clip_pg_rho_threshold))


def compute_policy_gradient_loss(logits, actions, advantages):
    return _PolicyGradientLoss.apply(logits, actions, advantages)


def compute_entropy_loss(logits):
    return _EntropyLoss.apply(logits)


def compute_baseline_loss(advantages):
    return _BaselineLoss.apply(advantages)


@torch.no_grad()
def impala_loss_and_head_grads(behavior_logits, target_logits, baseline, action, reward, done, discounting=0.99,
                               reward_clipping='abs_one', clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0,
                               baseline_cost=0.5, entropy_cost=0.0006):
    """Fused learner tail on [T+1,B] batch rows -> dict(vs, pg_advantages, dlogits, dbaseline, losses[4])."""
    bl, tl, baseline, reward = [_f32(t, n) for t, n in ((behavior_logits, 'behavior_logits'), (target_logits, 'target_logits'),
                                                         (baseline, 'baseline'), (reward, 'reward'))]
    T1, B, A = tl.shape
    T = T1 - 1
    if T < 1:
        raise ValueError('need at least 2 rows (T >= 1)')
    if reward_clipping not in ('abs_one', 'none'):
        raise ValueError("reward_clipping must be 'abs_one' or 'none'")
    action = action.contiguous()
    done_u8 = done.contiguous().view(torch.uint8) if done.dtype == torch.bool else done.contiguous()
    dev = tl.device
    vs = torch.empty(T, B, device=dev)
    pg = torch.empty(T, B, device=dev)
    dlogits = torch.empty(T, B, A, device=dev)
    dbaseline = torch.empty(T, B, device=dev)
    losses = torch.empty(4, device=dev)
    scratch = torch.zeros(3 * ((B + 3) // 4) + 8, device=dev)
    _lib.check(_lib.lib().srl_impala_loss_and_head_grads(
        bl.data_ptr(), tl.data_ptr(), baseline.data_ptr(), action.data_ptr(), reward.data_ptr(), done_u8.data_ptr(), T, B, A,
        float(discounting), 1 if reward_clipping == 'abs_one' else 0, _clip(clip_rho_threshold), _clip(clip_pg_rho_threshold),
        float(baseline_cost), float(entropy_cost), vs.data_ptr(), pg.data_ptr(), dlogits.data_ptr(), dbaseline.data_ptr(),
        losses.data_ptr(), scratch.data_ptr(), _stream()), 'impala_loss_and_head_grads')
    return dict(vs=vs, pg_advantages=pg, dlogits=dlogits, dbaseline=dbaseline, losses=losses)
