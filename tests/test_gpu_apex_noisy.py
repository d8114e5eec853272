"""Noisy networks in the Ape-X learner and actors on the H100 (ApexHParams(noisy_dqn=True), B200ApexActor(..., noisy_dqn=True)); 3 and
5 are the checks every head shares (tests/apex_cases.py):
  1. the composed weights of both networks are torch's mu + sigma * outer(f(eps_out), f(eps_in)) on the device's noise, and the sigma
     gradients are dW * eps, bit for bit, for each head;
  2. with every sigma 0 (and no clipping) one noisy step is the plain learner's on mu, bit for bit: q, y, priorities, loss, the mu
     gradients and the updated mu;
  3. fp32-accurate split operands against the fp32 CPU oracle (oracle/apex_oracle.py) fed the device's noise, with the dueling and
     categorical siblings' tolerances (Q scaled by the size of the terms it sums for every head: it cancels);
  4. the noise: pooled normals of 200 captured replays against N(0, 1) (KS), online != target, new draws per replay, (seed, step)
     determines the draw;
  5. eager = captured, two learners with one seed, a captured learn_from loop with prioritized adds, and a resumed checkpoint;
  6. the learner's q_values use mu; the actor's q_values and priorities are a plain actor's on its composed weights; act at eps 0 is
     the argmax under its own draw, and each act (eager or captured) draws anew.
The measured errors are written to $SRL_RESULTS_DIR/apex_noisy.json when SRL_RESULTS_DIR is set."""
import numpy as np
import pytest
import torch
from scipy import stats

from oracle import apex_oracle as O
from scalerl_b200.algorithms.apex import ApexHParams, B200ApexActor, B200ApexLearner
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer
from tests import apex_cases as cases
from tests.apex_cases import HEADS as ROWS, batch, device_composed, frames, learner, nets
from tests.exact import record

pytestmark = pytest.mark.gpu
HEADS = {h: ROWS[f'noisy_{h}'] for h in ('plain', 'dueling', 'categorical')}


def _dims(head):
    return HEADS[head].kind == 'dueling', HEADS[head].width


def _nets(A, head, seed=0, std=0.5):
    return nets(HEADS[head], A, seed, noisy_std=std)


def _learner(B, A, head, on, tg, seed=0, **kw):
    return learner(HEADS[head], B, A, on, tg, seed=seed, **kw)


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('head', list(HEADS))
def test_composition_and_sigma_grads_are_torchs(head, double):
    B, A = 32, 6
    on, tg = _nets(A, head, seed=1)
    step_batch, w = batch(B, A, seed=2, device='cuda')
    L = _learner(B, A, head, on, tg, double_dqn=double)
    L.learn(step_batch, weights=w, use_graph=False)
    d, K = _dims(head)
    for net, sd in (('online', on), ('target', tg)):
        noise = L.debug_buffer(f'noise_{net}').cpu()
        normals = L.debug_buffer(f'normals_{net}').cpu()
        f = normals.double().sign() * normals.double().abs().sqrt()                 # f(x) = sgn(x) sqrt|x|, rounded once
        assert float((noise.double() - f).abs().max()) <= 2 ** -24 * float(f.abs().max()), net
        dev = device_composed(L, net)
        for name, (Wt, bt) in O.composed(sd, noise, A, d, K).items():
            assert torch.equal(dev[name][0].cpu(), Wt), (net, name)
            assert torch.equal(dev[name][1].cpu(), bt), (net, name)
    noise = O.split_noise(L.debug_buffer('noise_online'), A, d, K)
    for name, (ei, eo) in noise.items():
        gW, gb = L.grads[f'{name}.weight_mu'].cpu(), L.grads[f'{name}.bias_mu'].cpu()
        assert torch.equal(L.grads[f'{name}.weight_sigma'].cpu(), gW * torch.outer(eo, ei)), name
        assert torch.equal(L.grads[f'{name}.bias_sigma'].cpu(), gb * eo), name
    assert bool(L.grads['fc.weight_mu'].any())


# ---------------------------------------------------------------------------------------------------------------- 2
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('head', list(HEADS))
def test_sigma_zero_is_the_plain_learner(head, double):
    B, A = 32, 6
    on, tg = _nets(A, head, seed=3, std=0.0)
    strip = lambda sd: {n.replace('_mu', ''): v for n, v in sd.items() if 'sigma' not in n}
    step_batch, w = batch(B, A, seed=4, device='cuda')
    N = _learner(B, A, head, on, tg, double_dqn=double)
    P = learner(HEADS[head].but(noisy=False), B, A, strip(on), strip(tg), double_dqn=double)
    N.learn(step_batch, weights=w, use_graph=False)
    P.learn(step_batch, weights=w, use_graph=False)
    for k in ('q', 'y', 'priorities', 'loss', 'dcore'):
        assert torch.equal(N.debug_buffer(k), P.debug_buffer(k)), k
    for n, g in P.grads.items():
        m = n.replace('weight', 'weight_mu').replace('bias', 'bias_mu') if not n.startswith('conv') else n
        assert torch.equal(N.grads[m], g), n
        assert torch.equal(N.params[m], P.params[n]), n
    assert bool(N.grads['fc.weight_sigma'].any())          # sigma learns even from 0


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('head', list(HEADS))
@pytest.mark.parametrize('B,A', [(32, 6), (5, 4), (512, 18)])
def test_split_against_noisy_oracle(B, A, head, double, clip):
    cases.check_split_against_oracle(HEADS[head], B, A, double, clip)


# ---------------------------------------------------------------------------------------------------------------- 4
def test_noise_distribution_and_keys():
    B, A = 32, 6
    on, tg = _nets(A, 'plain', seed=5)
    L = _learner(B, A, 'plain', on, tg, seed=11)
    step_batch, w = batch(B, A, seed=6, device='cuda')
    pooled, prev = [], None
    for k in range(202):
        L.learn(step_batch, weights=w, sync_stats=False)               # eager, capture, then 200 replays
        a, b = L.debug_buffer('normals_online'), L.debug_buffer('normals_target')
        assert not torch.equal(a, b)
        if prev is not None:
            assert not torch.equal(a, prev)
        prev = a
        if k >= 2:
            pooled += [a.cpu(), b.cpu()]
    assert len(L._graphs) == 1
    x = torch.cat(pooled).double().numpy()
    ks = stats.kstest(x, 'norm')
    record(HEADS['plain'].results, 'noise_ks', {'n': int(x.size), 'statistic': float(ks.statistic), 'pvalue': float(ks.pvalue), 'mean': float(x.mean()), 'std': float(x.std())})
    assert ks.pvalue > 1e-3, ks
    assert abs(x.mean()) < 5e-3 and abs(x.std() - 1) < 5e-3

    def first_draw(seed, step=0):
        M = _learner(B, A, 'plain', on, tg, seed=seed)
        M.set_step(step)
        M.learn(step_batch, weights=w, use_graph=False)
        return M.debug_buffer('normals_online'), M.debug_buffer('normals_target')

    s0, s0b, s1 = first_draw(11), first_draw(11), first_draw(12)
    assert torch.equal(s0[0], s0b[0]) and torch.equal(s0[1], s0b[1])
    assert not torch.equal(s0[0], s1[0]) and not torch.equal(s0[1], s1[1])
    # (seed, step) determines the draw: update 201 of L is update 201 of a learner set to that step
    assert torch.equal(first_draw(11, 201)[0], prev)


# ---------------------------------------------------------------------------------------------------------------- 5
@pytest.mark.parametrize('head', list(HEADS))
def test_determinism_and_graph_replay(head):
    cases.check_determinism_and_graph_replay(HEADS[head])


def test_captured_learn_from_loop_is_deterministic():
    cases.check_captured_learn_from_loop(HEADS['plain'])


@pytest.mark.parametrize('head', ['plain', 'dueling'])
def test_checkpoint_roundtrip_and_resume(tmp_path, head):
    cases.check_checkpoint_roundtrip_and_resume(HEADS[head], tmp_path)


# ---------------------------------------------------------------------------------------------------------------- 6
def _plain_sd(sd):
    return {n.replace('_mu', ''): v for n, v in sd.items() if 'sigma' not in n}


@pytest.mark.parametrize('head', list(HEADS))
def test_learner_q_values_use_mu(head):
    B, A = 16, 6
    on, _ = _nets(A, head, seed=2)
    L = _learner(B, A, head, on, on)
    P = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, **HEADS[head].but(noisy=False).hp), init_state_dict=_plain_sd(on))
    obs = frames(37, 1, 'cuda')
    assert torch.equal(L.q_values(obs), P.q_values(obs))
    assert torch.equal(L.predict(obs), P.predict(obs))


def _actor_weights(X, sd, head):
    """the plain state dict of the actor's composed weights (its conv tensors from sd)"""
    out = {n: v for n, v in sd.items() if n.startswith('conv')}
    out['fc.weight'], out['fc.bias'] = X.debug_buffer('fc_weight').view(512, 3136), X.debug_buffer('fc_bias')
    W, b = X.debug_buffer('head_weight').view(-1, 512), X.debug_buffer('head_bias')
    if head == 'dueling':
        out.update({'value.weight': W[:1], 'value.bias': b, 'advantage.weight': W[1:], 'advantage.bias': X.debug_buffer('head_adv_bias')})
    else:
        out.update({'q.weight': W, 'q.bias': b})
    return {n: v.clone() for n, v in out.items()}


@pytest.mark.parametrize('head', list(HEADS))
def test_actor_against_a_plain_actor_on_its_composed_weights(head):
    E, A, n, gamma = 32, 6, 3, 0.99
    kw = HEADS[head].but(noisy=False).hp
    d, K = _dims(head)
    sd = HEADS[head].state_dict(A, 4)
    X = B200ApexActor(E, A, seed=9, init_state_dict=sd, noisy_dqn=True, **kw)
    assert bool((X.epsilons == 0).all())
    obs = frames(E, 2, 'cuda')
    # a new actor keeps a first draw: q_values compose it
    n0 = X.debug_buffer('noise')
    q0 = X.q_values(obs)
    ref = O.composed(sd, n0, A, d, K)
    assert torch.equal(X.debug_buffer('fc_weight').view(512, 3136).cpu(), ref['fc'][0])
    P = B200ApexActor(E, A, epsilons=np.zeros(E), init_state_dict=_actor_weights(X, sd, head), **kw)
    assert torch.equal(q0, P.q_values(obs))
    # act draws anew and acts greedily on that draw
    a1 = X.act(obs)
    n1 = X.debug_buffer('noise')
    assert not torch.equal(n0, n1)
    P.load_state_dict(_actor_weights(X, sd, head))
    q1 = P.q_values(obs)
    assert torch.equal(a1, torch.argmax(q1, dim=1)) and torch.equal(X.q_values(obs), q1)
    a2 = X.act(obs)
    assert not torch.equal(X.debug_buffer('noise'), n1)
    P.load_state_dict(_actor_weights(X, sd, head))
    assert torch.equal(a2, torch.argmax(P.q_values(obs), dim=1))
    # the prioritized add on the kept draw is the plain actor's on the composed weights, bit for bit
    mems = [GpuPrioritizedReplayBuffer(256, E, alpha=1.0, n_step=n, gamma=gamma) for _ in range(2)]
    g = torch.Generator().manual_seed(6)
    for t in range(n + 1):
        args = (torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(), torch.randint(0, A, (E,), generator=g).cuda(),
                torch.randn(E, generator=g).cuda(), torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(),
                (torch.rand(E, generator=g) < 0.3).cuda())
        mems[0].save_to_memory(*args, is_vectorised=True, priorities_from=X)
        mems[1].save_to_memory(*args, is_vectorised=True, priorities_from=P)
    for t1, t2 in zip(mems[0].sampler.trees(), mems[1].sampler.trees()):
        assert (t1 == t2) if isinstance(t1, float) else torch.equal(t1, t2)


def test_captured_act_draws_anew():
    E, A = 8, 6
    X = B200ApexActor(E, A, seed=2, noisy_dqn=True)
    obs = frames(E, 3, 'cuda')
    out = torch.empty(E, dtype=torch.int64, device='cuda')
    X.act(obs)                                                 # warm-up
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out.copy_(X.act(obs))
    draws = []
    for _ in range(3):
        g.replay()
        draws.append(X.debug_buffer('noise'))
    assert not torch.equal(draws[0], draws[1]) and not torch.equal(draws[1], draws[2])
    # the same seed gives the same sequence of draws
    Y = B200ApexActor(E, A, seed=2, noisy_dqn=True)
    for _ in range(4):                                         # create's draw, the warm-up's and three replays'
        Y.act(obs)
    assert torch.equal(Y.debug_buffer('noise'), draws[2])
