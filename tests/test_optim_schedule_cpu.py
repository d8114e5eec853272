"""The learning-rate schedule and RMSprop momentum on the host side (no GPU): the closed form the optimizer kernels evaluate
against torchbeast's LambdaLR and ScaleRL's LinearDecayScheduler, the torch.optim checkpoint layout with momentum, and the
argument checks of ImpalaHParams."""
import types

import pytest
import torch

from scalerl_b200 import _lib
from scalerl_b200.learner import (ImpalaHParams, from_torch_optimizer_state, param_shapes, reference_param_order, scheduled_lr,
                                  to_torch_optimizer_state)

T, B = 5, 4
F = T * B
LR = 2.0 ** -10          # exact in float32: the float32 closed form is then the rounded torch value


class _LinearDecay:
    """ScaleRL's LinearDecayScheduler(start_value, end_value, max_steps) stepping rule (scalerl/utils/lr_scheduler.py:50-88):
    a step counter advanced by step(n) and clamped at max_steps; the value is the linear interpolation to 0, floored at end_value"""

    def __init__(self, start, end, max_steps):
        self.start, self.end, self.max_steps, self.count = start, end, max_steps, 0

    def step(self, n):
        self.count = min(self.count + n, self.max_steps)
        return max(self.start * (1.0 - (self.count * 1.0) / self.max_steps), self.end)


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def test_closed_form_equals_torchbeast_lambda_lr():
    """torchbeast: LambdaLR(lambda epoch: 1 - min(epoch * T * B, total) / total), scheduler.step() after optimizer.step(): the lr
    step t runs at is the scheduler's value after t - 1 steps.  K crosses the frame budget."""
    total = 6 * F + 7                               # reached between steps 7 and 8
    p = torch.nn.Parameter(torch.zeros(3))
    opt = torch.optim.RMSprop([p], lr=LR)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda epoch: 1 - min(epoch * T * B, total) / total)
    seen = []
    for t in range(1, 12):
        lr_torch = opt.param_groups[0]['lr']
        mine = scheduled_lr(LR, 'linear', t, F, total, 0.0)
        assert mine == lr_torch, (t, mine, lr_torch)                       # same double arithmetic
        assert _f32(scheduled_lr(_f32(LR), 'linear', t, F, total, _f32(0.0))) == _f32(lr_torch), t     # what the kernel computes
        seen.append(mine)
        p.grad = torch.ones_like(p)
        opt.step()
        sched.step()
    assert seen[0] == LR and seen[-1] == 0.0 and seen[7] == 0.0 and seen[6] > 0.0
    assert scheduled_lr(LR, 'constant', 99, F, None) == LR


def test_closed_form_equals_linear_decay_scheduler_with_floor():
    """the reference's LinearDecayScheduler stepped by the F frames of every optimizer step, with a floor; K crosses the floor
    (step 6) and the frame budget (step 9)"""
    total, end = 8 * F, LR / 4
    ref = _LinearDecay(LR, end, total)
    value = LR                                       # before the first step() the scheduler holds its start value
    for t in range(1, 14):
        mine = scheduled_lr(LR, 'linear', t, F, total, end)
        assert mine == value, (t, mine, value)
        assert _f32(scheduled_lr(_f32(LR), 'linear', t, F, total, _f32(end))) == _f32(value), t
        value = ref.step(F)
    assert scheduled_lr(LR, 'linear', 6, F, total, end) > end == scheduled_lr(LR, 'linear', 7, F, total, end)
    assert scheduled_lr(LR, 'linear', 13, F, total, end) == end


def _params(use_lstm, A):
    shapes = param_shapes(A, use_lstm)
    return [torch.nn.Parameter(torch.zeros(shapes[n])) for n in reference_param_order(use_lstm)]


@pytest.mark.parametrize('use_lstm', [False, True])
def test_momentum_checkpoint_round_trip_through_torch(use_lstm):
    """optimizer_state_dict's layout with momentum and the linear schedule: torch.optim.RMSprop(momentum=mu) loads it (state and
    param_groups, lr as a LambdaLR leaves it after `step` steps), takes a step, and the parser reads the result back"""
    A, mu, step, total = 6, 0.9, 7, 20 * F
    hp = ImpalaHParams(num_actions=A, use_lstm=use_lstm, momentum=mu, learning_rate=LR, lr_schedule='linear', total_frames=total)
    order = reference_param_order(use_lstm)
    shapes = param_shapes(A, use_lstm)
    g = torch.Generator().manual_seed(3)
    tensors = {k: {n: torch.rand(shapes[n], generator=g) for n in order} for k in ('square_avg', 'momentum_buffer')}
    sd = to_torch_optimizer_state(hp, tensors, step=step, frames_per_step=F)
    params = _params(use_lstm, A)
    opt = torch.optim.RMSprop(params, lr=LR, momentum=mu, eps=hp.epsilon, alpha=hp.alpha)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 1 - min(e * F, total) / total)
    for _ in range(step):
        opt.step()                                   # no gradients: only the schedule moves
        sched.step()
    want_lr = opt.param_groups[0]['lr']
    opt2 = torch.optim.RMSprop(_params(use_lstm, A), lr=LR, momentum=mu, eps=hp.epsilon, alpha=hp.alpha)
    opt2.load_state_dict(sd)
    grp = opt2.param_groups[0]
    assert grp['momentum'] == mu and grp['lr'] == want_lr and grp['initial_lr'] == LR
    for i, p in enumerate(opt2.param_groups[0]['params']):
        st = opt2.state[p]
        assert float(st['step']) == step
        for k in ('square_avg', 'momentum_buffer'):
            assert torch.equal(st[k], tensors[k][order[i]]), (k, order[i])
    for p in opt2.param_groups[0]['params']:
        p.grad = torch.ones_like(p)
    opt2.step()
    back_step, back = from_torch_optimizer_state(opt2.state_dict(), use_lstm, momentum=True)
    assert back_step == step + 1 and set(back) == {'square_avg', 'momentum_buffer'} and set(back['momentum_buffer']) == set(order)
    p0 = opt2.param_groups[0]['params'][0]
    assert torch.equal(back['momentum_buffer'][order[0]], opt2.state[p0]['momentum_buffer'])
    # a momentum-0 learner's parser path refuses the buffer, as before
    with pytest.raises(ValueError, match='momentum_buffer'):
        from_torch_optimizer_state(opt2.state_dict(), use_lstm)
    with pytest.raises(ValueError, match='momentum_buffer'):
        from_torch_optimizer_state(opt2.state_dict(), use_lstm, momentum=False)


def test_constant_schedule_param_groups_unchanged():
    """the default learner writes the param_groups torch writes for the reference's optimizer: no scheduler keys"""
    hp = ImpalaHParams()
    sd = to_torch_optimizer_state(hp, {'square_avg': {}}, step=0)
    ref = torch.optim.RMSprop([torch.nn.Parameter(torch.zeros(1)) for _ in range(12)], lr=hp.learning_rate, momentum=0.0,
                              eps=hp.epsilon, alpha=hp.alpha).state_dict()['param_groups']
    assert sd['param_groups'] == ref


def test_hparams_validation():
    ImpalaHParams().to_c()
    ImpalaHParams(momentum=0.9).to_c()
    ImpalaHParams(lr_schedule='linear', total_frames=1000, min_learning_rate=1e-6).to_c()
    ImpalaHParams(optimizer='adam', lr_schedule='linear', total_frames=1000).to_c()
    with pytest.raises(ValueError, match='total_frames'):
        ImpalaHParams(lr_schedule='linear').to_c()
    with pytest.raises(ValueError, match='total_frames'):
        ImpalaHParams(lr_schedule='linear', total_frames=0).to_c()
    with pytest.raises(ValueError, match='momentum'):
        ImpalaHParams(optimizer='adam', momentum=0.9).to_c()
    with pytest.raises(ValueError, match='momentum'):
        ImpalaHParams(momentum=-0.1).to_c()
    with pytest.raises(ValueError, match='lr_schedule'):
        ImpalaHParams(lr_schedule='cosine', total_frames=1000).to_c()
    with pytest.raises(ValueError, match='min_learning_rate'):
        ImpalaHParams(lr_schedule='linear', total_frames=1000, min_learning_rate=-1.0).to_c()


def test_trainer_forwards_the_schedule():
    """ImpalaArguments.total_steps counts frames (the reference adds T * B per learner step): it is the schedule's frame budget"""
    from scalerl_b200.algorithms.impala.impala_atari import ImpalaArguments, ImpalaTrainer
    a = ImpalaArguments(lr_schedule='linear', min_learning_rate=1e-6, momentum=0.5, total_steps=12345)
    hp = ImpalaTrainer.hparams(types.SimpleNamespace(args=a))
    assert (hp.lr_schedule, hp.min_learning_rate, hp.momentum, hp.total_frames) == ('linear', 1e-6, 0.5, 12345)
    d = ImpalaTrainer.hparams(types.SimpleNamespace(args=ImpalaArguments()))
    assert (d.lr_schedule, d.momentum) == ('constant', 0.0)


def test_c_entry_points_reject_a_null_learner():
    L = _lib.lib()
    assert L.srl_learner_set_lr_schedule(None, 0, 0.0, 1.0, 1.0) == -1
    assert b'NULL' in L.srl_last_error()
    assert L.srl_learner_set_momentum(None, 0.0, None) == -1
    assert b'NULL' in L.srl_last_error()
