"""The GPU prioritized replay memory on the H100 (GpuPrioritizedReplayBuffer / srl_replay_*) and B200ApexLearner.learn_from:
  1. every reference-pinned case (tests/golden/replay_cases.npz): the ring holds exactly the expected frames, actions, reward bits and dones;
  2. sample with given uniforms: idxs identical to PerOracle on the same trees, weights within f32 rounding, rows equal to the storage;
  3. wrap-around with M = 10, E = 4;
  4. learn_from equals an explicit sample (same uniforms) + learn, bit for bit, eager, captured and replayed;
  5. a captured learn_from (and a captured learn with a sampler) replayed after further adds samples the new slots, and their
     priorities reach the trees, as PerOracle fed the learner's priorities says;
  6. two seeded runs with the same adds give the same parameters bit for bit;
  7. a beta change between replays gives the oracle's weights without a recapture;
  8. bad calls raise before anything is enqueued."""
import os

import numpy as np
import pytest
import torch

from oracle import replay_oracle as O
from oracle.per_oracle import PerOracle
from scalerl_b200.algorithms.apex import ApexHParams, B200ApexLearner
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
from tests.conftest import GOLDEN

pytestmark = pytest.mark.gpu
NPIX = 4 * 84 * 84


def frame(step, env, salt):
    """the seeded frame stack of raw step `step`, env `env` (salt 0: its state, 1: its next_state)"""
    x = (np.arange(NPIX, dtype=np.int64) * (2 * step + 1) + 31 * env + 97 * salt + 3 * step) % 251
    return x.astype(np.uint8).reshape(4, 84, 84)


def _frames(steps, E, salt):
    return np.stack([np.stack([frame(t, e, salt) for e in range(E)]) for t in range(steps)])


def _fill(mem, steps, action, reward, done, on_device):
    E = mem.num_envs
    st, nst = _frames(steps, E, 0), _frames(steps, E, 1)
    for t in range(steps):
        args = (st[t], action[t], reward[t], nst[t], done[t])
        if on_device:
            args = tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in args)
        if E == 1:
            mem.save_to_memory(*(a[0] for a in args))
        else:
            mem.save_to_memory(*args, is_vectorised=True)
    return st, nst


def test_ring_matches_reference_cases():
    z = np.load(os.path.join(GOLDEN, 'replay_cases.npz'))
    for ci, (M, E, n, dr, steps, seed) in enumerate(O.CASES):
        mem = GpuPrioritizedReplayBuffer(M, E, n_step=n, gamma=O.GAMMA)
        action, reward, done = O.case_inputs(E, steps, dr, seed)
        st, nst = _fill(mem, steps, action, reward, done, on_device=ci % 2 == 1)
        size = int(z[f'c{ci}_meta'][6])
        assert len(mem) == size
        s, a, r, ns, d = (t.cpu().numpy() for t in mem.gather(torch.arange(size)))
        assert np.array_equal(a, z[f'c{ci}_action']), ci
        assert np.array_equal(r.view(np.uint32), z[f'c{ci}_reward_bits']), ci
        assert np.array_equal(d, z[f'c{ci}_done']), ci
        assert np.array_equal(s, st[z[f'c{ci}_s_step'], z[f'c{ci}_s_env']]), ci
        assert np.array_equal(ns, nst[z[f'c{ci}_ns_step'], z[f'c{ci}_s_env']]), ci
        mem.close()


def _oracle_from(mem):
    """PerOracle holding the memory's current trees (the GPU's own leaf values, so sampled indices compare exactly)"""
    st, mt, mp = mem.sampler.trees()
    o = PerOracle(mem.memory_size, mem.alpha)
    o.sum_tree.tree[:], o.min_tree.tree[:] = st.cpu().numpy(), mt.cpu().numpy()
    o.max_priority, o.size = mp, len(mem)
    return o


def test_sample_matches_oracle_and_storage():
    M, E, B = 300, 8, 64
    rng = np.random.RandomState(3)
    mem = GpuPrioritizedReplayBuffer(M, E, n_step=3, gamma=0.97)
    action, reward, done = O.case_inputs(E, 30, 0.2, 7)
    _fill(mem, 30, action, reward, done, on_device=True)
    assert len(mem) == 224
    mem.update_priorities(torch.from_numpy(rng.randint(0, 224, 500)), torch.from_numpy(rng.rand(500) * 4 + 1e-3))
    o = _oracle_from(mem)
    u = rng.rand(B)
    s, a, r, ns, d, w, idxs = mem.sample(B, beta=0.6, uniforms=torch.from_numpy(u))
    ri, rw = o.sample(u, 0.6)
    assert np.array_equal(idxs.cpu().numpy(), ri)
    assert np.allclose(w.cpu().numpy(), rw, rtol=2e-7, atol=0)
    gs, ga, gr, gns, gd = mem.gather(idxs)
    for x, y in ((s, gs), (a, ga), (r, gr), (ns, gns), (d, gd)):
        assert torch.equal(x, y)
    assert s.dtype == torch.uint8 and a.dtype == torch.int64 and r.dtype == torch.float32 and d.dtype == torch.uint8 and a.shape == (B,)


def test_wraparound_m10_e4():
    mem = GpuPrioritizedReplayBuffer(10, 4)
    action = np.arange(12, dtype=np.int64).reshape(3, 4)
    _fill(mem, 3, action, np.zeros((3, 4), np.float32), np.zeros((3, 4), np.uint8), on_device=False)
    assert len(mem) == 10
    # transitions 0..11 in env order: 10 and 11 (step 2, envs 2 and 3) overwrite slots 0 and 1
    assert mem.gather(torch.arange(10))[1].tolist() == [10, 11, 2, 3, 4, 5, 6, 7, 8, 9]
    mem.save_to_memory(np.stack([frame(9, e, 0) for e in range(4)]), np.full(4, 40), np.zeros(4, np.float32),
                       np.stack([frame(9, e, 1) for e in range(4)]), np.zeros(4, bool), is_vectorised=True)
    assert mem.gather(torch.arange(10))[1].tolist() == [10, 11, 40, 40, 40, 40, 6, 7, 8, 9]
    assert np.array_equal(mem.gather(torch.tensor([5]))[0][0].cpu().numpy(), frame(9, 3, 0))


def _memory(M=256, E=8, steps=10, seed=0, n_step=1):
    mem = GpuPrioritizedReplayBuffer(M, E, n_step=n_step, gamma=0.99)
    add_steps(mem, steps, seed)
    return mem


def add_steps(mem, steps, seed):
    g = torch.Generator().manual_seed(seed)
    E = mem.num_envs
    for _ in range(steps):
        mem.save_to_memory(torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(),
                           torch.randint(0, 6, (E,), generator=g).cuda(), torch.randn(E, generator=g).cuda(),
                           torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(),
                           (torch.rand(E, generator=g) < 0.1).cuda(), is_vectorised=True)


def _hp(B=32):
    return ApexHParams(batch_size=B, num_actions=6, gamma=0.99 ** 3, double_dqn=True, target_update_frequency=2)


def test_learn_from_equals_sample_and_learn():
    B = 32
    La, Lb = B200ApexLearner(_hp(B)), B200ApexLearner(_hp(B))
    ma, mb = _memory(n_step=3), _memory(n_step=3)
    for k in range(5):
        La.learn_from(ma, beta=0.5, sync_stats=False)
        u = La._from['u'].clone()
        s, a, r, ns, d, w, idxs = mb.sample(B, beta=0.5, uniforms=u)
        assert torch.equal(idxs, La._from['idxs']) and torch.equal(w, La._from['weights'])
        Lb.learn((s, a, r, ns, d), w, idxs, mb.sampler, sync_stats=False, use_graph=False)
        assert torch.equal(La.flat_params, Lb.flat_params), k
        assert torch.equal(La.flat_target, Lb.flat_target), k
        assert torch.equal(ma.sampler.trees()[0], mb.sampler.trees()[0]), k
        if k == 2:
            add_steps(ma, 2, seed=5)
            add_steps(mb, 2, seed=5)
    assert len(La._graphs) == 1 and La.learner_update_step == 5 and La.target_model_update_step == 3


def _leaf_check(sampler, oracle):
    st, _, mp = sampler.trees()
    cap = sampler.capacity
    leaves = st[cap:cap + sampler.memory_size].cpu().numpy()
    assert np.allclose(leaves, oracle.sum_tree.tree[cap:cap + sampler.memory_size], rtol=1e-14, atol=0)
    assert mp == oracle.max_priority
    assert sampler._L.srl_per_invalid_updates(sampler._h, sampler._stream()) == 0


def test_captured_learn_from_sees_later_adds():
    B, E = 32, 8
    L = B200ApexLearner(_hp(B))
    mem = _memory(M=64, E=E, steps=2)                      # 16 stored when the graph is captured
    o = PerOracle(64, mem.alpha)
    o.add(16)
    seen_new = 0
    for k in range(5):
        if k == 2:
            add_steps(mem, 4, seed=9)                      # 48 stored: the captured graph must see them
            o.add(32)
        L.learn_from(mem)
        idxs = L._from['idxs'].cpu().numpy()
        o.update_priorities(idxs, L.debug_buffer('priorities').cpu().numpy())
        seen_new += int((idxs >= 16).sum()) if k >= 2 else 0
    assert len(L._graphs) == 1 and seen_new > 0
    _leaf_check(mem.sampler, o)


def test_captured_learn_with_sampler_sees_later_adds():
    """learn(..., idxs, sampler) captured while the sampler held 16 transitions, replayed with idxs at or above 16"""
    B = 32
    L = B200ApexLearner(_hp(B))
    s = GpuPrioritizedSampler(64)
    s.add(16)
    o = PerOracle(64, s.alpha)
    o.add(16)
    g = torch.Generator().manual_seed(1)
    bufs = (torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(), torch.randint(0, 6, (B,), generator=g).cuda(),
            torch.randn(B, generator=g).cuda(), torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(),
            torch.zeros(B, dtype=torch.uint8, device='cuda'))
    idxs = torch.arange(B, device='cuda') % 16
    w = torch.ones(B, device='cuda')
    for k in range(4):
        if k == 2:
            s.add(32)
            o.add(32)
            idxs.copy_(torch.arange(16, 16 + B, device='cuda'))
        L.learn(bufs, w, idxs, s)
        o.update_priorities(idxs.cpu().numpy(), L.debug_buffer('priorities').cpu().numpy())
    assert len(L._graphs) == 1
    _leaf_check(s, o)


def _seeded_run(seed):
    torch.manual_seed(seed)
    L = B200ApexLearner(_hp(32))
    mem = _memory(steps=6, seed=4, n_step=3)
    for k in range(4):
        L.learn_from(mem, sync_stats=False)
        if k == 1:
            add_steps(mem, 3, seed=8)
    return L.flat_params.clone(), mem.sampler.trees()[0]


def test_seeded_runs_are_bit_identical():
    p1, t1 = _seeded_run(11)
    p2, t2 = _seeded_run(11)
    assert torch.equal(p1, p2) and torch.equal(t1, t2)


def test_beta_change_between_replays():
    L = B200ApexLearner(_hp(32))
    mem = _memory(steps=12)
    for _ in range(3):
        L.learn_from(mem, beta=0.4)                        # eager, capture, replay
    for beta in (0.9, 0.4, 1.0):
        o = _oracle_from(mem)
        L.learn_from(mem, beta=beta)
        ri, rw = o.sample(L._from['u'].cpu().numpy(), beta)
        assert np.array_equal(L._from['idxs'].cpu().numpy(), ri)
        assert np.allclose(L._from['weights'].cpu().numpy(), rw, rtol=2e-7, atol=0), beta
    assert len(L._graphs) == 1


def test_bad_calls_raise_before_enqueue():
    L = B200ApexLearner(_hp(32))
    mem = GpuPrioritizedReplayBuffer(16, 1)
    mem.save_to_memory(np.zeros((4, 84, 84), np.uint8), 1, 0.5, np.zeros((4, 84, 84), np.uint8), False)
    before = L.flat_params.clone()
    with pytest.raises(ValueError, match='at least 2'):
        L.learn_from(mem)
    with pytest.raises(ValueError, match='GpuPrioritizedReplayBuffer'):
        L.learn_from(GpuPrioritizedSampler(16))
    with pytest.raises(ValueError, match='beta'):
        mem.save_to_memory(np.zeros((4, 84, 84), np.uint8), 1, 0.5, np.zeros((4, 84, 84), np.uint8), False)
        L.learn_from(mem, beta=float('nan'))
    with pytest.raises(ValueError, match='state'):
        mem.save_to_memory(np.zeros((1, 4, 84, 84), np.uint8), 1, 0.5, np.zeros((4, 84, 84), np.uint8), False)
    with pytest.raises(ValueError, match='at least 2'):
        GpuPrioritizedReplayBuffer(16, 1).sample(4)
    dev = mem.device
    mem.device = torch.device('cuda', 1)
    with pytest.raises(ValueError, match='cuda:1'):
        L.learn_from(mem)
    mem.device = dev
    torch.cuda.synchronize()
    assert len(mem) == 2 and L._opt_steps == 0 and L.learner_update_step == 0 and not L._seen
    assert torch.equal(L.flat_params, before) and int(L.debug_buffer('step')[0]) == 0
