"""The frame replay memory on the H100 (GpuFrameReplayBuffer / srl_frame_replay_*) against the stack memory (GpuPrioritizedReplayBuffer)
fed the same adds, and against oracle/frame_replay_oracle.py:
  1. every replay_cases.npz case and an Atari-like stream: gather(arange(len)) bit-identical, frames_allocated() the oracle's count;
  2. sample with given uniforms: identical idxs, weights and rows;
  3. save_to_memory(..., priorities_from=actor): bit-identical trees;
  4. learn_from from the same seed: the same parameters and trees bit for bit, eager, captured and replayed, and a captured learn_from
     replayed after further adds samples the new slots;
  5. forced retirement: the oracle's retired slots and count, never sampled, gather and priority writes leave them as they are;
  6. wrap-around with M = 10, E = 4;
  7. bad calls raise before anything is enqueued."""
import numpy as np
import pytest
import torch

from oracle import frame_replay_oracle as FO
from oracle import replay_oracle as O
from scalerl_b200.algorithms.apex import ApexHParams, B200ApexActor, B200ApexLearner
from scalerl_b200.data.replay_memory import GpuFrameReplayBuffer, GpuPrioritizedReplayBuffer
from tests.test_gpu_replay import frame

pytestmark = pytest.mark.gpu


class Stream:
    """an Atari-like stream (oracle/frame_replay_oracle.py) of E envs: step t's (state, action, reward, next_state, done)"""

    def __init__(self, E, steps, seed, done=None, done_rate=0.05, A=18):
        rng = np.random.RandomState(seed + 1)
        self.action = rng.randint(0, A, size=(steps, E)).astype(np.int64)
        self.reward = rng.randn(steps, E).astype(np.float32)
        self.si, self.ni, self.done, K = FO.atari_stream(E, steps, seed, done=done, done_rate=done_rate)
        self.frames = FO.stream_frames(E, K, seed)

    def __getitem__(self, t):
        return (FO.stream_stacks(self.frames, self.si[t]), self.action[t], self.reward[t], FO.stream_stacks(self.frames, self.ni[t]),
                self.done[t])


def _add(mems, step, on_device, oracle=None, **kw):
    if oracle is not None:
        oracle.add(*step)
    args = tuple(torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in step) if on_device else step
    for m in mems:
        m.save_to_memory(*args, is_vectorised=True, **kw)


def _fill(M, E, n, stream, steps, frame_capacity=None, gamma=O.GAMMA, alpha=0.6):
    sm = GpuPrioritizedReplayBuffer(M, E, alpha=alpha, n_step=n, gamma=gamma)
    fm = GpuFrameReplayBuffer(M, E, alpha=alpha, n_step=n, gamma=gamma, frame_capacity=frame_capacity)
    fo = FO.FrameReplayOracle(M, E, n, gamma, frame_capacity)
    for t in range(steps):
        _add((sm, fm), stream[t], on_device=t % 2 == 1, oracle=fo)
    return sm, fm, fo


def _same_gather(sm, fm, idxs):
    return all(torch.equal(a, b) for a, b in zip(sm.gather(idxs), fm.gather(idxs)))


@pytest.mark.parametrize('ci', range(len(O.CASES)))
def test_cases_gather_as_the_stack_memory(ci):
    M, E, n, dr, steps, seed = O.CASES[ci]
    _, _, done = O.case_inputs(E, steps, dr, seed)
    sm, fm, fo = _fill(M, E, n, Stream(E, steps, seed, done=done), steps)
    assert len(fm) == len(sm) == fo.size
    assert _same_gather(sm, fm, torch.arange(len(sm)))
    assert fm.frames_allocated() == fo.head and fm.retired() == 0


def test_atari_stream_gathers_as_the_stack_memory():
    M, E, n, steps = 512, 8, 3, 100
    st = Stream(E, steps, seed=3, done_rate=0.08)
    sm, fm, fo = _fill(M, E, n, st, steps)
    assert fm.frames_allocated() == fo.head == FO.expected_new_frames(st.si)
    assert _same_gather(sm, fm, torch.arange(len(sm)))
    assert fm.retired() == 0


def test_sample_is_identical():
    M, E, B = 300, 8, 64
    rng = np.random.RandomState(3)
    sm, fm, _ = _fill(M, E, 3, Stream(E, 30, seed=7, done_rate=0.2), 30, gamma=0.97)
    assert len(fm) == 224
    idxs, prios = torch.from_numpy(rng.randint(0, 224, 500)), torch.from_numpy(rng.rand(500) * 4 + 1e-3)
    sm.update_priorities(idxs, prios)
    fm.update_priorities(idxs, prios)
    u = torch.from_numpy(rng.rand(B))
    for a, b in zip(sm.sample(B, beta=0.6, uniforms=u), fm.sample(B, beta=0.6, uniforms=u)):
        assert torch.equal(a, b)


@pytest.mark.parametrize('n', [1, 3])
def test_prioritized_add_trees_are_identical(n):
    E, A = 8, 6
    X = B200ApexActor(E, A, seed=5)
    sm, fm = (cls(256, E, alpha=1.0, n_step=n, gamma=0.99) for cls in (GpuPrioritizedReplayBuffer, GpuFrameReplayBuffer))
    st = Stream(E, 20, seed=4, done_rate=0.2, A=A)
    for t in range(20):
        _add((sm, fm), st[t], on_device=True, priorities_from=X)
    for a, b in zip(sm.sampler.trees()[:2], fm.sampler.trees()[:2]):
        assert torch.equal(a, b)
    assert sm.sampler.trees()[2] == fm.sampler.trees()[2]
    assert _same_gather(sm, fm, torch.arange(len(sm)))


def _hp(B=32):
    return ApexHParams(batch_size=B, num_actions=18, gamma=0.99 ** 3, double_dqn=True, target_update_frequency=2)


def _learn_run(cls, seed):
    torch.manual_seed(seed)
    L = B200ApexLearner(_hp())
    mem = cls(256, 8, n_step=3, gamma=0.99)
    st = Stream(8, 12, seed=2)
    for t in range(6):
        _add((mem,), st[t], on_device=True)
    seen_new, idxs = 0, []
    for k in range(5):                                     # eager, capture, replays
        if k == 3:
            before = len(mem)
            for t in range(6, 12):
                _add((mem,), st[t], on_device=True)
        L.learn_from(mem, sync_stats=False)
        idxs.append(L._from['idxs'].clone())
        if k >= 3:
            seen_new += int((L._from['idxs'] >= before).sum())
    assert len(L._graphs) == 1 and seen_new > 0
    return L.flat_params.clone(), L.flat_target.clone(), mem.sampler.trees()[0], idxs


def test_learn_from_is_bit_identical_on_both_memories():
    ps, ts, trs, ids = _learn_run(GpuPrioritizedReplayBuffer, 11)
    pf, tf, trf, idf = _learn_run(GpuFrameReplayBuffer, 11)
    assert torch.equal(ps, pf) and torch.equal(ts, tf) and torch.equal(trs, trf)
    assert all(torch.equal(a, b) for a, b in zip(ids, idf))


def _retired_leaves(mem):
    s, m, _ = mem.sampler.trees()
    cap = mem.sampler.capacity
    leaves_s, leaves_m = s[cap:cap + len(mem)].cpu().numpy(), m[cap:cap + len(mem)].cpu().numpy()
    return set(np.flatnonzero((leaves_s == 0) & np.isinf(leaves_m)).tolist())


@pytest.mark.parametrize('n', [1, 3])
def test_forced_retirement(n):
    M, E, steps = 128, 2, 120
    F = 8 * E * (n + 1)
    st = Stream(E, steps, seed=9, done_rate=0.2)
    sm, fm, fo = _fill(M, E, n, st, steps, frame_capacity=F)
    assert fo.retired > 0
    assert fm.retired() == fo.retired and fm.frames_allocated() == fo.head
    assert _retired_leaves(fm) == fo.retired_slots
    live = np.array(sorted(set(range(len(fm))) - fo.retired_slots))
    assert _same_gather(sm, fm, torch.from_numpy(live))
    # never sampled: uniforms at 0, just below 1 and in between
    B = 256
    us = [torch.zeros(B, dtype=torch.float64), torch.full((B,), np.nextafter(1.0, 0.0), dtype=torch.float64),
          torch.from_numpy(np.random.RandomState(0).rand(B))]
    for u in us:
        *_, w, idxs = fm.sample(B, beta=0.4, uniforms=u)
        got = set(idxs.cpu().tolist())
        assert not got & fo.retired_slots and max(got) < len(fm) and bool(torch.isfinite(w).all())
    # gather leaves a retired slot's rows as they were
    r = torch.tensor(sorted(fo.retired_slots)[:4], device='cuda')
    out = tuple(torch.full_like(t, 0xAB if t.dtype == torch.uint8 else 7) for t in fm._outputs(len(r)))
    ref = tuple(t.clone() for t in out)
    fm._L.srl_frame_replay_gather(fm._h, r.data_ptr(), len(r), *(t.data_ptr() for t in out), fm._stream())
    assert all(torch.equal(a, b) for a, b in zip(out, ref))
    # a priority write to a retired leaf leaves it retired and is not an invalid update
    fm.update_priorities(r.cpu(), torch.full((len(r),), 3.0, dtype=torch.float64))
    assert fm.sampler._L.srl_per_invalid_updates(fm.sampler._h, fm.sampler._stream()) == 0
    assert _retired_leaves(fm) == fo.retired_slots


def test_wraparound_m10_e4():
    mem = GpuFrameReplayBuffer(10, 4)
    for t in range(3):
        mem.save_to_memory(np.stack([frame(t, e, 0) for e in range(4)]), np.arange(4 * t, 4 * t + 4), np.zeros(4, np.float32),
                           np.stack([frame(t, e, 1) for e in range(4)]), np.zeros(4, bool), is_vectorised=True)
    assert len(mem) == 10
    assert mem.gather(torch.arange(10))[1].tolist() == [10, 11, 2, 3, 4, 5, 6, 7, 8, 9]
    mem.save_to_memory(np.stack([frame(9, e, 0) for e in range(4)]), np.full(4, 40), np.zeros(4, np.float32),
                       np.stack([frame(9, e, 1) for e in range(4)]), np.zeros(4, bool), is_vectorised=True)
    assert mem.gather(torch.arange(10))[1].tolist() == [10, 11, 40, 40, 40, 40, 6, 7, 8, 9]
    assert np.array_equal(mem.gather(torch.tensor([5]))[0][0].cpu().numpy(), frame(9, 3, 0))
    assert np.array_equal(mem.gather(torch.tensor([5]))[3][0].cpu().numpy(), frame(9, 3, 1))


def test_bad_calls_raise_before_enqueue():
    L = B200ApexLearner(_hp())
    with pytest.raises(ValueError, match='frame_capacity'):
        GpuFrameReplayBuffer(16, 2, frame_capacity=31)
    mem = GpuFrameReplayBuffer(16, 1)
    mem.save_to_memory(np.zeros((4, 84, 84), np.uint8), 1, 0.5, np.zeros((4, 84, 84), np.uint8), False)
    before = L.flat_params.clone()
    with pytest.raises(ValueError, match='at least 2'):
        L.learn_from(mem)
    with pytest.raises(ValueError, match='state'):
        mem.save_to_memory(np.zeros((1, 4, 84, 84), np.uint8), 1, 0.5, np.zeros((4, 84, 84), np.uint8), False)
    with pytest.raises(ValueError, match='at least 2'):
        mem.sample(4)
    with pytest.raises(ValueError, match='beta'):
        mem.save_to_memory(np.zeros((4, 84, 84), np.uint8), 1, 0.5, np.zeros((4, 84, 84), np.uint8), False)
        L.learn_from(mem, beta=float('nan'))
    torch.cuda.synchronize()
    assert len(mem) == 2 and mem.frames_allocated() == 1 and L._opt_steps == 0 and not L._seen
    assert torch.equal(L.flat_params, before)
