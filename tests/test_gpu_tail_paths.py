"""GPU: the V-trace and loss paths share one implementation, so they agree bit for bit on the same operands.
  * The fused column kernel of a learner step and the stand-alone tail (`impala_loss_and_head_grads`, the warp-per-column kernel at these
    sizes) run the same column tail: fed the learner's own logits and baselines, the stand-alone tail gives the learner's vs, pg_advantages,
    dlogits and dbaseline exactly.  The losses are summed in a different tree (per column vs per block of four columns): 1e-6 relative.
  * `from_logits` and `from_importance_weights(variant=0)` run the same sequential V-trace step: fed the log_rhos that from_logits returns,
    the latter gives the same vs and pg_advantages."""
import numpy as np
import pytest
import torch

from oracle import impala_oracle as O

pytestmark = pytest.mark.gpu


def _mismatch(got, want):
    return f'{int((got != want).sum())} of {want.numel()} elements differ, max |diff| {float((got - want).abs().max()):.3e}'


@pytest.mark.parametrize('T,B,A', [(20, 32, 6), (33, 5, 18), (7, 19, 4)])
def test_column_kernel_matches_standalone_tail(T, B, A):
    from scalerl_b200 import ops
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    hp = ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A)
    L = B200ImpalaLearner(hp, init_state_dict=O.init_params(A, seed=7), process_group=False)
    try:
        batch = {k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=T + B, done_p=0.1).items()}
        L.set_option('column_fusion', 1)           # explicit: SRL_NO_COLUMN_FUSION in the environment would turn it off
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            L.forward_backward(batch)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events()]
        assert any('column_step_kernel' in n for n in names), 'the learner step did not run the column kernel'
        assert not any('impala_tail' in n for n in names)
        logits = L.debug_buffer('logits').view(T + 1, B, A)
        baseline = L.debug_buffer('baseline').view(T + 1, B)
        out = ops.impala_loss_and_head_grads(batch['policy_logits'], logits, baseline, batch['action'], batch['reward'], batch['done'])
        want = {'vs': L._vs, 'pg_advantages': L._pg_adv, 'dlogits': L.debug_buffer('dlogits').view(T, B, A),
                'dbaseline': L.debug_buffer('dbaseline').view(T, B)}
        for k, w in want.items():
            assert torch.equal(out[k], w), f'{k}: {_mismatch(out[k], w)}'
        got, ref = out['losses'].cpu().double(), L._losses.cpu().double()
        assert torch.all((got - ref).abs() <= 1e-6 * ref.abs()), (got, ref)
    finally:
        L.close()


@pytest.mark.parametrize('T,B,A', [(20, 32, 6), (33, 5, 18), (7, 19, 4)])
def test_from_logits_matches_from_importance_weights(T, B, A):
    from scalerl_b200 import ops
    rng = np.random.RandomState(T * B + A)
    f = lambda *s: torch.from_numpy(rng.randn(*s).astype(np.float32)).cuda()
    bl, tl, rewards, values, boot = f(T, B, A), f(T, B, A), f(T, B), f(T, B), f(B)
    actions = torch.from_numpy(rng.randint(0, A, size=(T, B)).astype(np.int64)).cuda()
    discounts = torch.from_numpy(((rng.rand(T, B) > 0.05) * 0.99).astype(np.float32)).cuda()
    a = ops.from_logits(bl, tl, actions, discounts, rewards, values, boot)
    b = ops.from_importance_weights(a.log_rhos, discounts, rewards, values, boot, variant=0)
    assert torch.equal(a.vs, b.vs), f'vs: {_mismatch(a.vs, b.vs)}'
    assert torch.equal(a.pg_advantages, b.pg_advantages), f'pg_advantages: {_mismatch(a.pg_advantages, b.pg_advantages)}'
