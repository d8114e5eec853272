"""Batched GPU actor inference (SURVEY.md §8f-4): B200ActorModel behind the reference's actor calling convention."""
import time

import pytest
import torch

from tests.helpers import rel_l2

pytestmark = pytest.mark.gpu


def _env_batch(N, A, seed):
    g = torch.Generator().manual_seed(seed)
    return dict(obs=torch.randint(0, 256, (1, N, 4, 84, 84), dtype=torch.uint8, generator=g), reward=torch.randn(1, N, generator=g),
                done=torch.zeros(1, N, dtype=torch.bool), action=torch.randint(0, A, (1, N), generator=g))


def test_gpu_actor_matches_cpu_actor_and_samples_softmax():
    from scalerl_b200.algorithms.impala.gpu_actor import B200ActorModel
    from scalerl_b200.algorithms.utils.atari_model import ActorNet
    N, A = 48, 6
    cpu = ActorNet((4, 84, 84), A, seed=3)
    gpu = B200ActorModel(N, A, init_state_dict=cpu.state_dict())
    env = _env_batch(N, A, 1)
    cpu.eval()
    ref, _ = cpu(env, ())
    gpu.eval()
    out, state = gpu(env, gpu.initial_hidden_state(N))
    assert state == tuple() and set(out) == {'policy_logits', 'baseline', 'action'}
    assert tuple(out['policy_logits'].shape) == (1, N, A) and out['action'].dtype == torch.int64
    assert rel_l2(out['policy_logits'], ref['policy_logits']) < 2e-2 and rel_l2(out['baseline'], ref['baseline']) < 2e-2
    assert torch.equal(out['action'], out['policy_logits'].argmax(-1))              # eval mode: argmax (atari_model.py:133-134)
    # training mode: actions ~ softmax(logits).  N identical frames -> N draws from one distribution, repeated
    gpu.train()
    same = {k: v[:, :1].expand(-1, N, *v.shape[2:]).contiguous() for k, v in env.items()}
    counts = torch.zeros(A)
    draws = 0
    for _ in range(60):
        o, _ = gpu(same, ())
        counts += torch.bincount(o['action'].view(-1), minlength=A).float()
        draws += N
    p = torch.softmax(o['policy_logits'][0, 0], -1)
    sigma = torch.sqrt(p * (1 - p) / draws)
    assert torch.all((counts / draws - p).abs() < 5 * sigma + 1e-3), (counts / draws, p)
    gpu.close()


def test_gpu_actor_weight_refresh_paths():
    from scalerl_b200.algorithms.impala.gpu_actor import B200ActorModel
    from scalerl_b200.algorithms.utils.atari_model import ActorNet
    from scalerl_b200.learner import B200ImpalaLearner, ImpalaHParams
    N, A = 8, 6
    gpu = B200ActorModel(N, A, seed=1)
    env = _env_batch(N, A, 2)
    gpu.eval()
    a0, _ = gpu(env, ())
    shared = ActorNet((4, 84, 84), A, seed=9).share_memory()           # what ImpalaTrainer.publish_weights writes (flat, learner layout)
    assert gpu.refresh(shared.flat_params, version=5) and gpu.weights_version == 5
    assert not gpu.refresh(shared.flat_params, version=5)              # same version: nothing to do
    a1, _ = gpu(env, ())
    ref, _ = shared.eval()(env, ())
    assert rel_l2(a1['policy_logits'], ref['policy_logits']) < 2e-2 and rel_l2(a1['policy_logits'], a0['policy_logits']) > 0.1
    L = B200ImpalaLearner(ImpalaHParams(rollout_length=2, batch_size=2, num_actions=A), process_group=False, seed=4)
    gpu.sync_from(L, version=6)
    assert torch.equal(gpu._ctx.flat_params, L.flat_params) and gpu.weights_version == 6
    gpu.close(); L.close()


def test_gpu_actor_throughput_is_recorded():
    """actor steps per second at N = 256 environments per call (host tensors in and out, as the actor loop uses it)"""
    from scalerl_b200.algorithms.impala.gpu_actor import B200ActorModel
    from tests.exact import record
    N, A = 256, 6
    gpu = B200ActorModel(N, A)
    env = _env_batch(N, A, 3)
    for _ in range(5):
        gpu(env, ())
    t0 = time.perf_counter()
    n = 50
    for _ in range(n):
        gpu(env, ())
    dt = time.perf_counter() - t0
    record('parity_fullsize.json', 'gpu_actor_N256', {'calls_per_sec': n / dt, 'env_steps_per_sec': n * N / dt, 'ms_per_call': dt / n * 1e3})
    assert n * N / dt > 2e4
    gpu.close()
