"""The Ape-X actor on the H100 (B200ApexActor / srl_apex_actor_*, srl_replay_add_prioritized); 1 and 5 are the checks every head
shares (tests/apex_cases.py), here with the plain head:
  1. after sync_from(learner) the actor's Q values equal the learner's bit for bit; with every epsilon 0, act is their first argmax;
  2. epsilon = 1 gives uniform actions, and the apex_epsilons schedule gives each env group its non-greedy rate eps (A - 1) / A;
  3. seeded, eager and captured acting draw the same sequence; each replay draws anew and follows set_epsilons;
  4. fp32-accurate actor: the inserted leaves against compute_prior's p^alpha (oracle/apex_oracle.initial_priorities), the trees against
     PerOracle, the ring against the plain add;
  5. bf16 actor and learner on the same weights: the actor's priorities are the learner's, bit for bit;
  6. a NaN in the snapshot gives finite trees, leaves at max_priority^alpha and E invalid updates;
  7. a 200-step act -> env -> prioritized add -> learn_from loop stays finite and two seeded runs are bit-identical.
The measured errors are written to $SRL_RESULTS_DIR/apex_actor.json when SRL_RESULTS_DIR is set."""
import math

import numpy as np
import pytest
import torch

from oracle import apex_oracle as O
from oracle import replay_oracle as RO
from oracle.per_oracle import PerOracle
from scalerl_b200.algorithms.apex import ApexHParams, B200ApexActor, B200ApexLearner, apex_epsilons, default_q_state_dict
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
from tests import apex_cases as cases
from tests.apex_cases import frames, nmax
from tests.exact import record

pytestmark = pytest.mark.gpu
NPIX = 4 * 84 * 84
PLAIN = cases.HEADS['plain']


def _dominant(sd, a, by=50.0):
    """a copy of sd whose Q head prefers action a at every frame (a unique argmax)"""
    sd = {k: v.clone() for k, v in sd.items()}
    sd['q.bias'][a] += by
    return sd


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('E', [1, 13, 256, 1500])
def test_q_values_equal_the_learners_and_greedy_act(E):
    cases.check_actor_q_values_and_greedy_act(PLAIN, E)


# ---------------------------------------------------------------------------------------------------------------- 2
def test_epsilon_one_is_uniform():
    E, A, T = 1500, 6, 20
    X = B200ApexActor(E, A, epsilons=np.ones(E), seed=7)
    obs = frames(E, 2, 'cuda')
    counts = torch.zeros(A, dtype=torch.int64)
    for _ in range(T):
        counts += torch.bincount(X.act(obs).cpu(), minlength=A)
    n, p = E * T, 1.0 / A
    sigma = math.sqrt(n * p * (1 - p))
    record('apex_actor.json', 'uniform_counts', counts.tolist())
    assert counts.sum() == n and float((counts - n * p).abs().max()) <= 5 * sigma, counts


def test_apex_schedule_rates():
    E, A, T, groups = 256, 6, 300, 8
    eps = apex_epsilons(E)
    X = B200ApexActor(E, A, seed=11, init_state_dict=_dominant(default_q_state_dict(A, 0), 2))
    obs = frames(E, 3, 'cuda')
    assert bool((torch.argmax(X.q_values(obs), 1) == 2).all())
    off = torch.zeros(E, dtype=torch.int64)
    for _ in range(T):
        off += (X.act(obs) != 2).cpu().long()
    p = eps * (A - 1) / A
    dev = []
    for g in np.array_split(np.arange(E), groups):
        want, sigma = T * p[g].sum(), math.sqrt(T * (p[g] * (1 - p[g])).sum())
        dev.append((float(off[g].sum()) - want) / sigma)
    record('apex_actor.json', 'schedule_group_deviation_sigma', dev)
    assert max(abs(d) for d in dev) <= 5, dev


# ---------------------------------------------------------------------------------------------------------------- 3
def test_seeded_eager_and_captured_acting():
    E, A = 256, 6
    obs = frames(E, 4, 'cuda')
    a1, a2 = B200ApexActor(E, A, epsilons=np.full(E, 0.5), seed=5), B200ApexActor(E, A, epsilons=np.full(E, 0.5), seed=5)
    eager = [a1.act(obs) for _ in range(6)]
    assert all(torch.equal(x, a2.act(obs)) for x in eager[:1])          # same seed, same draw
    assert not torch.equal(eager[0], eager[1])                          # a new draw per call
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = a2.act(obs)
    for k in range(1, 6):                                               # each replay is the next eager call
        g.replay()
        assert torch.equal(out, eager[k]), k
    a2.set_epsilons(np.zeros(E))
    g.replay()
    assert torch.equal(out, torch.argmax(a2.q_values(obs), 1))
    a2.set_epsilons(np.ones(E))
    g.replay()
    assert not torch.equal(out, torch.argmax(a2.q_values(obs), 1))


# ---------------------------------------------------------------------------------------------------------------- 4
def _frame(step, env, salt):
    x = (np.arange(NPIX, dtype=np.int64) * (2 * step + 1) + 31 * env + 97 * salt + 3 * step) % 251
    return x.astype(np.uint8).reshape(4, 84, 84)


@pytest.mark.parametrize('M,E,n,steps,alpha', [(10, 4, 3, 7, 1.0), (10, 4, 1, 5, 0.6), (10, 4, 3, 6, 0.6), (2048, 1500, 1, 3, 1.0)])
def test_fp32_actor_against_oracle(M, E, n, steps, alpha):
    A, gamma = 6, 0.99
    sd = default_q_state_dict(A, 4)
    X = B200ApexActor(E, A, precision='fp32_split', priority_eps=1e-6, init_state_dict=sd)
    mem = GpuPrioritizedReplayBuffer(M, E, alpha=alpha, n_step=n, gamma=gamma)
    plain = GpuPrioritizedReplayBuffer(M, E, alpha=alpha, n_step=n, gamma=gamma)
    action, reward, done = RO.case_inputs(E, steps, 0.3, 100 + E)
    action %= A
    st = np.stack([np.stack([_frame(t, e, 0) for e in range(E)]) for t in range(steps)])
    nst = np.stack([np.stack([_frame(t, e, 1) for e in range(E)]) for t in range(steps)])
    ro, po = RO.ReplayOracle(M, E, n, gamma), PerOracle(M, alpha)
    worst = 0.0
    for t in range(steps):
        args = tuple(torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in (st[t], action[t], reward[t], nst[t], done[t]))
        mem.save_to_memory(*args, is_vectorised=True, priorities_from=X)
        plain.save_to_memory(*args, is_vectorised=True)
        ids = [(t, e) for e in range(E)]
        ptr = ro.tree_ptr
        ro.add(ids, action[t], reward[t], ids, done[t])
        if t + 1 < n:
            continue
        slots = [(ptr + e) % M for e in range(E)]
        rows = [ro.slots[i] for i in slots]
        s = torch.from_numpy(np.stack([st[r[0]] for r in rows]))
        ns = torch.from_numpy(np.stack([nst[r[3]] for r in rows]))
        want = O.initial_priorities(sd, s, torch.tensor([r[1] for r in rows]), torch.tensor([r[2] for r in rows]), ns,
                                    torch.tensor([bool(r[4]) for r in rows]), float(np.float32(gamma ** n)), 1e-6)
        sum_t, min_t, mp = mem.sampler.trees()
        cap = mem.sampler.capacity
        leaves = sum_t[cap:cap + M].cpu().numpy()[slots]
        worst = max(worst, nmax(leaves, want.numpy() ** alpha))
        # PerOracle fed the kernel's priorities (alpha = 1: leaf = p) or the kernel's leaves, inserted at tree_ptr
        if alpha == 1.0:
            po.update_priorities(slots, leaves)
        else:
            po.set_leaves(slots, leaves)
            po.max_priority = max(po.max_priority, float(want.max()))
        po.tree_ptr, po.size = (po.tree_ptr + E) % M, min(po.size + E, M)
        assert np.array_equal(sum_t.cpu().numpy(), po.sum_tree.tree) and np.array_equal(min_t.cpu().numpy(), po.min_tree.tree), t
        assert mp == po.max_priority if alpha == 1.0 else mp == pytest.approx(po.max_priority, rel=1e-5)
        assert len(mem) == po.size
    assert mem.sampler._L.srl_per_invalid_updates(mem.sampler._h, mem.sampler._stream()) == 0
    record('apex_actor.json', f'fp32_split_M{M}_E{E}_n{n}_alpha{alpha}', {'leaf_nmax': worst})
    assert worst <= 1e-5, worst
    idx = torch.arange(M)
    for x, y in zip(mem.gather(idx), plain.gather(idx)):
        assert torch.equal(x, y)


# ---------------------------------------------------------------------------------------------------------------- 5
def test_bf16_priorities_are_the_learners():
    cases.check_bf16_actor_priorities(PLAIN)


# ---------------------------------------------------------------------------------------------------------------- 6
def test_nan_snapshot_keeps_the_trees_finite():
    E, A, alpha = 8, 6, 0.6
    X = B200ApexActor(E, A)
    mem = GpuPrioritizedReplayBuffer(32, E, alpha=alpha)
    obs = frames(E, 9, 'cuda')
    z = torch.zeros(E, device='cuda')
    mem.save_to_memory(obs, torch.zeros(E, dtype=torch.int64, device='cuda'), z, obs, z.bool(), is_vectorised=True, priorities_from=X)
    before = mem.sampler._L.srl_per_invalid_updates(mem.sampler._h, mem.sampler._stream())
    X.params['q.bias'].fill_(float('nan'))
    mem.save_to_memory(obs, torch.ones(E, dtype=torch.int64, device='cuda'), z, obs, z.bool(), is_vectorised=True, priorities_from=X)
    after = mem.sampler._L.srl_per_invalid_updates(mem.sampler._h, mem.sampler._stream())
    sum_t, min_t, mp = mem.sampler.trees()
    cap = mem.sampler.capacity
    assert after - before == E
    assert bool(torch.isfinite(sum_t).all()) and not bool(torch.isnan(min_t).any())
    assert torch.allclose(sum_t[cap + E:cap + 2 * E], torch.full((E,), mp ** alpha, dtype=torch.float64, device='cuda'), rtol=1e-15, atol=0)
    assert bool((sum_t[cap + E:cap + 2 * E] == sum_t[cap + E]).all())
    assert len(mem) == 2 * E and math.isfinite(mp)


# ---------------------------------------------------------------------------------------------------------------- 7
class ToyVecEnv:
    """a deterministic vector env on the device: frame stacks from each env's step count, reward 1 when the action matches the count
    mod A (else -0.1), an episode end every 23 steps (offset per env), the finished env restarting at count 0"""

    def __init__(self, E, A):
        self.E, self.A = E, A
        self.t = torch.zeros(E, dtype=torch.int64, device='cuda')
        self.pix = torch.arange(NPIX, device='cuda').view(1, 4, 84, 84)
        self.env = torch.arange(E, device='cuda').view(E, 1, 1, 1)

    def obs(self):
        t = self.t.view(-1, 1, 1, 1)
        return ((self.pix * (t % 5 + 1) + 17 * self.env + 3 * t) % 251).to(torch.uint8)

    def step(self, action):
        self.t += 1
        reward = torch.where(action == self.t % self.A, 1.0, -0.1).float()
        done = (self.t + self.env.view(-1)) % 23 == 0
        next_obs = self.obs()
        self.t = torch.where(done, torch.zeros_like(self.t), self.t)
        return next_obs, reward, done, self.obs()


def _env_loop(seed, steps=200):
    torch.manual_seed(seed)
    E, A, n = 16, 4, 3
    L = B200ApexLearner(ApexHParams(batch_size=32, num_actions=A, gamma=0.99 ** n, target_update_frequency=20), seed=seed)
    X = B200ApexActor(E, A, seed=seed)
    X.sync_from(L)
    mem = GpuPrioritizedReplayBuffer(1024, E, n_step=n, gamma=0.99)
    env = ToyVecEnv(E, A)
    obs, updates, losses = env.obs(), 0, []
    for _ in range(steps):
        action = X.act(obs)
        next_obs, reward, done, obs_after = env.step(action)
        mem.save_to_memory(obs, action, reward, next_obs, done, is_vectorised=True, priorities_from=X)
        obs = obs_after
        if len(mem) >= 64:
            losses.append(L.learn_from(mem)['loss'])
            updates += 1
            if updates % 10 == 0:
                X.sync_from(L)
    return L, mem, losses


def test_one_gpu_apex_loop_is_finite_and_deterministic():
    L1, m1, l1 = _env_loop(21)
    L2, m2, l2 = _env_loop(21)
    assert len(l1) > 150 and len(L1._graphs) == 1 and all(math.isfinite(x) for x in l1)
    assert bool(torch.isfinite(L1.flat_params).all()) and bool(torch.isfinite(m1.sampler.trees()[0]).all())
    assert l1 == l2 and torch.equal(L1.flat_params, L2.flat_params)
    assert torch.equal(m1.sampler.trees()[0], m2.sampler.trees()[0]) and torch.equal(m1.sampler.trees()[1], m2.sampler.trees()[1])
    assert m1.sampler._L.srl_per_invalid_updates(m1.sampler._h, m1.sampler._stream()) == 0
    record('apex_actor.json', 'loop_200', {'updates': len(l1), 'first_loss': l1[0], 'last_loss': l1[-1]})
