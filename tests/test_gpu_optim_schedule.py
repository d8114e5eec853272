"""The learning-rate schedule and RMSprop momentum of the fused clip + optimizer step on the GPU, under CUDA-graph replay:
momentum against torch.optim.RMSprop(momentum=0.9), the 'linear' schedule against the host closed form (bit for bit) and
against torch's LambdaLR, the default path unchanged, determinism and checkpoint resume, the C ABI's argument errors, and the
data-parallel step (tests/dp_schedule_check.py under torchrun; skipped below 2 GPUs)."""
import os
import subprocess
import sys

import pytest
import torch

from oracle import impala_oracle as O
from scalerl_b200 import _lib
from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams, scheduled_lr
from tests.helpers import assert_close
from tests.test_gpu_multi import _counts, _free_port

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T, B, A = 5, 4, 6
F = T * B
LR = 2.0 ** -10            # exact in float32


def _f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


def _batches(n, seed=100):
    return [{k: v.cuda() for k, v in O.synthetic_batch(T, B, A, seed=seed + i, done_p=0.1).items()} for i in range(n)]


class _Run:
    """a learner fed through ONE set of batch buffers: step 1 runs eagerly, step 2 captures the CUDA graph, later steps replay it"""

    def __init__(self, use_lstm=False, seed=1, **kw):
        self.L = B200ImpalaLearner(ImpalaHParams(rollout_length=T, batch_size=B, num_actions=A, use_lstm=use_lstm, **kw), seed=seed,
                                   process_group=False)
        self.buf = None

    def step(self, batch):
        if self.buf is None:
            self.buf = {k: v.clone() for k, v in batch.items()}
        for k, v in batch.items():
            self.buf[k].copy_(v)
        return self.L.learn(self.buf)


def _cpu_mirror(L):
    return [torch.nn.Parameter(L.params[n].detach().cpu().clone()) for n in L.names]


def _cpu_step(L, cpu, opt, sched=None):
    """clip_grad_norm_(40) + the torch optimizer step on the CPU in fp32, from the gradients the device step used"""
    for n, p in zip(L.names, cpu):
        p.grad = L.grads[n].detach().cpu().clone()
    torch.nn.utils.clip_grad_norm_(cpu, L.hp.max_grad_norm)
    opt.step()
    if sched is not None:
        sched.step()


@pytest.mark.parametrize('use_lstm', [False, True])
def test_momentum_matches_torch_rmsprop(use_lstm):
    run = _Run(use_lstm=use_lstm, momentum=0.9)
    L = run.L
    cpu = _cpu_mirror(L)
    opt = torch.optim.RMSprop(cpu, lr=L.hp.learning_rate, momentum=0.9, eps=L.hp.epsilon, alpha=L.hp.alpha)
    mom = {n: v for n, v in L._opt_tensors()['momentum_buffer'].items()}
    for step, batch in enumerate(_batches(6)):
        run.step(batch)
        _cpu_step(L, cpu, opt)
        for n, p in zip(L.names, cpu):
            assert_close(L.params[n], p.detach(), 2e-6, f'step {step + 1} {n}')
            assert_close(mom[n], opt.state[p]['momentum_buffer'], 2e-6, f'step {step + 1} momentum_buffer {n}')
        assert L.learning_rate() == _f32(L.hp.learning_rate)
    assert len(L._graphs) == 1 and L.global_opt_step == 6 and L.device_opt_step() == 6


@pytest.mark.parametrize('optimizer,momentum', [('rmsprop', 0.0), ('rmsprop', 0.9), ('adam', 0.0)])
def test_linear_schedule_under_replay(optimizer, momentum):
    """F = 20 frames per step, Ftot = 60: the decay reaches 0 at step 4, so steps 4..8 run at the floor lr_end = LR / 5.
    Every step after the first replays the one captured graph; the lr it used is read back with the step's stats."""
    total, end = 3 * F, LR / 5
    run = _Run(optimizer=optimizer, momentum=momentum, learning_rate=LR, lr_schedule='linear', total_frames=total, min_learning_rate=end)
    L = run.L
    cpu = _cpu_mirror(L)
    if optimizer == 'adam':
        opt = torch.optim.Adam(cpu, lr=LR, betas=(L.hp.adam_beta1, L.hp.adam_beta2), eps=L.hp.adam_eps)
    else:
        opt = torch.optim.RMSprop(cpu, lr=LR, momentum=momentum, eps=L.hp.epsilon, alpha=L.hp.alpha)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: max(1 - min(e * F, total) / total, end / LR))
    assert L.learning_rate() == _f32(LR)                    # before the first step: the lr step 1 will use
    lrs = []
    for step, batch in enumerate(_batches(8), start=1):
        run.step(batch)
        want = _f32(scheduled_lr(_f32(LR), 'linear', step, F, total, _f32(end)))
        assert L.learning_rate() == want, (step, L.learning_rate(), want)
        lrs.append(want)
        _cpu_step(L, cpu, opt, sched)
        for n, p in zip(L.names, cpu):
            assert_close(L.params[n], p.detach(), 2e-6, f'step {step} {n}')
    assert lrs[0] == _f32(LR) and lrs[1] < lrs[0] and lrs[2] < lrs[1] and lrs[3:] == [_f32(end)] * 5
    assert len(L._graphs) == 1 and L.device_opt_step() == 8


def test_default_path_unchanged():
    """lr_schedule='constant', momentum=0 spelled out is the default learner: same kernels, same bits"""
    a = _Run()
    b = _Run(lr_schedule='constant', momentum=0.0, min_learning_rate=0.0)
    for batch in _batches(5):
        a.step(batch)
        b.step(batch)
    assert torch.equal(a.L.flat_params, b.L.flat_params) and torch.equal(a.L.opt_state0, b.L.opt_state0)
    assert a.L.opt_state2 is None and b.L.opt_state2 is None
    assert a.L.learning_rate() == b.L.learning_rate() == _f32(a.L.hp.learning_rate)


_KW = dict(momentum=0.9, learning_rate=LR, lr_schedule='linear', total_frames=4 * F + 3, min_learning_rate=LR / 50)


def test_momentum_schedule_deterministic_and_resumable(tmp_path):
    batches = _batches(6)
    a, b = _Run(**_KW), _Run(**_KW)
    for batch in batches:
        a.step(batch)
        b.step(batch)
    assert torch.equal(a.L.flat_params, b.L.flat_params) and torch.equal(a.L.opt_state2, b.L.opt_state2)
    # 3 steps, checkpoint, a fresh learner resumes: the schedule continues from the restored step count
    c = _Run(**_KW)
    for batch in batches[:3]:
        c.step(batch)
    path = str(tmp_path / 'ck.tar')
    c.L.save_checkpoint(path)
    ck = torch.load(path, weights_only=False)['optimizer_state_dict']
    assert ck['param_groups'][0]['momentum'] == 0.9 and 'momentum_buffer' in ck['state'][0]
    assert ck['param_groups'][0]['lr'] == scheduled_lr(LR, 'linear', 4, F, _KW['total_frames'], LR / 50)
    d = _Run(seed=7, **_KW)
    d.L.load_checkpoint(path)
    assert d.L.learning_rate() == c.L.learning_rate()
    for batch in batches[3:]:
        d.step(batch)
    assert torch.equal(d.L.flat_params, a.L.flat_params)
    assert torch.equal(d.L.opt_state0, a.L.opt_state0) and torch.equal(d.L.opt_state2, a.L.opt_state2)
    assert d.L.learning_rate() == a.L.learning_rate() and d.L.device_opt_step() == 6
    # a momentum checkpoint does not load into a learner without momentum
    e = _Run(learning_rate=LR, lr_schedule='linear', total_frames=4 * F + 3)
    with pytest.raises(ValueError, match='momentum_buffer'):
        e.L.load_checkpoint(path)


def test_c_abi_argument_errors():
    rms, adam = _Run().L, _Run(optimizer='adam').L
    lib, h = rms._L, rms._h
    buf = torch.zeros(rms.numel + 4, device='cuda')
    bad = [
        lambda: lib.srl_learner_set_lr_schedule(h, 2, 0.0, 20.0, 100.0),            # unknown kind
        lambda: lib.srl_learner_set_lr_schedule(h, -1, 0.0, 20.0, 100.0),
        lambda: lib.srl_learner_set_lr_schedule(h, 1, 0.0, 20.0, 0.0),              # total_frames <= 0
        lambda: lib.srl_learner_set_lr_schedule(h, 1, 0.0, 20.0, -5.0),
        lambda: lib.srl_learner_set_lr_schedule(h, 1, 0.0, 0.0, 100.0),             # frames_per_step <= 0
        lambda: lib.srl_learner_set_lr_schedule(h, 1, -1e-6, 20.0, 100.0),          # lr_end < 0
        lambda: lib.srl_learner_set_lr_schedule(h, 0, -1e-6, 20.0, 100.0),
        lambda: lib.srl_learner_set_momentum(h, -0.5, buf.data_ptr()),               # negative momentum
        lambda: lib.srl_learner_set_momentum(h, 0.9, None),                          # momentum without a buffer
        lambda: lib.srl_learner_set_momentum(h, 0.9, buf.data_ptr() + 4),            # misaligned buffer
        lambda: adam._L.srl_learner_set_momentum(adam._h, 0.9, buf.data_ptr()),      # momentum with Adam
    ]
    for i, call in enumerate(bad):
        with pytest.raises(ValueError):
            _lib.check(call(), f'case {i}')
    _lib.check(adam._L.srl_learner_set_momentum(adam._h, 0.0, None), 'momentum off is fine with Adam')
    # a refused call changes nothing: that learner still computes the default step's bits
    batch = _batches(1)[0]
    ref, r = _Run(), _Run()
    assert r.L._L.srl_learner_set_lr_schedule(r.L._h, 1, 0.0, 20.0, 0.0) == -1
    assert r.L._L.srl_learner_set_momentum(r.L._h, 0.9, None) == -1
    ref.step(batch)
    r.step(batch)
    assert torch.equal(ref.L.flat_params, r.L.flat_params) and r.L.learning_rate() == _f32(r.L.hp.learning_rate)


@pytest.mark.parametrize('world', [2, 4, 8])
@pytest.mark.parametrize('fused', ['nvls', 'peer_memory', 'nccl'])
def test_dp_schedule_and_momentum(world, fused):
    """sharded learners == full-batch learner with momentum and the linear schedule; replicas bit-identical (torchrun)"""
    if world not in _counts():
        pytest.skip(f'{world} GPUs not visible')
    env = dict(os.environ, SRL_DP_FUSED='0' if fused == 'nccl' else '1', SRL_DP_NVLS='1' if fused == 'nvls' else '0', MASTER_ADDR='127.0.0.1')
    cmd = [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', f'--nproc-per-node={world}', '--master-addr', '127.0.0.1',
           '--master-port', str(_free_port()), os.path.join(ROOT, 'tests', 'dp_schedule_check.py')]
    r = subprocess.run(cmd, cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    out = r.stdout + '\n' + r.stderr
    assert r.returncode == 0 and 'DP SCHEDULE CHECK OK' in out, out[-4000:]
    if fused == 'nvls' and 'nvls multimem' not in out:
        pytest.skip('no NVLS multicast mapping on this box: ran on peer loads')
    want = {'nvls': 'nvls multimem', 'peer_memory': 'peer loads', 'nccl': 'NCCL all-reduce'}[fused]
    assert want in out, out[-2000:]
