"""Noisy networks in the Ape-X learner and actors on the H100 (ApexHParams(noisy_dqn=True), B200ApexActor(..., noisy_dqn=True)):
  1. the composed weights of both networks are torch's mu + sigma * outer(f(eps_out), f(eps_in)) on the device's noise, and the sigma
     gradients are dW * eps, bit for bit, for each head;
  2. with every sigma 0 (and no clipping) one noisy step is the plain learner's on mu, bit for bit: q, y, priorities, loss, the mu
     gradients and the updated mu;
  3. fp32-accurate split operands against the noisy oracle (tests/apex_noisy_ref.py) fed the device's noise, with the dueling and
     categorical siblings' tolerances (Q scaled by the size of the terms it sums for every head: it cancels);
  4. the noise: pooled normals of 200 captured replays against N(0, 1) (KS), online != target, new draws per replay, (seed, step)
     determines the draw;
  5. eager = captured, two learners with one seed, a captured learn_from loop with prioritized adds, and a resumed checkpoint;
  6. the learner's q_values use mu; the actor's q_values and priorities are a plain actor's on its composed weights; act at eps 0 is
     the argmax under its own draw, and each act (eager or captured) draws anew.
The measured errors are written to $SRL_RESULTS_DIR/apex_noisy.json when SRL_RESULTS_DIR is set."""
import json
import math
import os

import numpy as np
import pytest
import torch
from scipy import stats

from tests import apex_noisy_ref as NR
from tests.test_gpu_apex import _batch, _mask_flips, nmax, rel_l2
from scalerl_b200.algorithms.apex import ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner, default_q_state_dict
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer

pytestmark = pytest.mark.gpu
F64 = torch.float64
HEADS = {'plain': dict(), 'dueling': dict(dueling_dqn=True), 'categorical': dict(categorical_dqn=True, num_atoms=11, v_min=-10.0, v_max=10.0)}


def _record(name, obj):
    d = os.environ.get('SRL_RESULTS_DIR')
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    p = os.path.join(d, 'apex_noisy.json')
    cur = json.load(open(p)) if os.path.exists(p) else {}
    cur[name] = obj
    json.dump(cur, open(p, 'w'), indent=1)


def _dims(head):
    kw = HEADS[head]
    return kw.get('dueling_dqn', False), (kw['num_atoms'] if kw.get('categorical_dqn') else 0)


def _nets(A, head, seed=0, std=0.5):
    d, K = _dims(head)
    return default_q_state_dict(A, 2 * seed, d, K, noisy=True, noisy_std=std), default_q_state_dict(A, 2 * seed + 1, d, K, noisy=True, noisy_std=std)


def _learner(B, A, head, on, tg, seed=0, **kw):
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, noisy_dqn=True, **HEADS[head], **kw), init_state_dict=on, seed=seed)
    L.load_state_dict(tg, target=True)
    return L


def frames(n, seed):
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).cuda()


def _device_composed(L, net):
    """the learner's composed weights of `net` ('online' / 'target') as {layer: (W, b)}, the head split as the state dict"""
    d = L.hp.dueling_dqn
    W, b = L.debug_buffer(f'head_weight_{net}').view(-1, 512), L.debug_buffer(f'head_bias_{net}')
    out = {'fc': (L.debug_buffer(f'fc_weight_{net}').view(512, 3136), L.debug_buffer(f'fc_bias_{net}'))}
    if d:
        out['value'], out['advantage'] = (W[:1], b), (W[1:], L.debug_buffer(f'head_adv_bias_{net}'))
    else:
        out['q'] = (W, b)
    return out


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('head', list(HEADS))
def test_composition_and_sigma_grads_are_torchs(head, double):
    B, A = 32, 6
    on, tg = _nets(A, head, seed=1)
    batch, w = _batch(B, A, seed=2, device='cuda')
    L = _learner(B, A, head, on, tg, double_dqn=double)
    L.learn(batch, weights=w, use_graph=False)
    d, K = _dims(head)
    for net, sd in (('online', on), ('target', tg)):
        noise = L.debug_buffer(f'noise_{net}').cpu()
        normals = L.debug_buffer(f'normals_{net}').cpu()
        f = normals.double().sign() * normals.double().abs().sqrt()                 # f(x) = sgn(x) sqrt|x|, rounded once
        assert float((noise.double() - f).abs().max()) <= 2 ** -24 * float(f.abs().max()), net
        dev = _device_composed(L, net)
        for name, (Wt, bt) in NR.composed(sd, noise, A, d, K).items():
            assert torch.equal(dev[name][0].cpu(), Wt), (net, name)
            assert torch.equal(dev[name][1].cpu(), bt), (net, name)
    noise = NR.split_noise(L.debug_buffer('noise_online'), A, d, K)
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
    batch, w = _batch(B, A, seed=4, device='cuda')
    N = _learner(B, A, head, on, tg, double_dqn=double)
    P = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, double_dqn=double, **HEADS[head]), init_state_dict=strip(on))
    P.load_state_dict(strip(tg), target=True)
    N.learn(batch, weights=w, use_graph=False)
    P.learn(batch, weights=w, use_graph=False)
    for k in ('q', 'y', 'priorities', 'loss', 'dcore'):
        assert torch.equal(N.debug_buffer(k), P.debug_buffer(k)), k
    for n, g in P.grads.items():
        m = n.replace('weight', 'weight_mu').replace('bias', 'bias_mu') if not n.startswith('conv') else n
        assert torch.equal(N.grads[m], g), n
        assert torch.equal(N.params[m], P.params[n]), n
    assert bool(N.grads['fc.weight_sigma'].any())          # sigma learns even from 0


# ---------------------------------------------------------------------------------------------------------------- 3
def _scaled(a, b, scale):
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    return float((a - b).abs().max() / max(float(scale.abs().max()), 1e-300))


@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('head', list(HEADS))
@pytest.mark.parametrize('B,A', [(32, 6), (5, 4), (512, 18)])
def test_split_against_noisy_oracle(B, A, head, double, clip):
    on, tg = _nets(A, head, seed=B)
    (obs, act, rew, nobs, done), w = _batch(B, A, seed=B + A)
    d, K = _dims(head)
    L = _learner(B, A, head, on, tg, seed=B, precision='fp32_split', double_dqn=double, max_grad_norm=clip, priority_eps=0.0)
    L.learn(tuple(t.cuda() for t in (obs, act, rew, nobs, done)), weights=w.cuda(), use_graph=False)
    n_on, n_tg = L.debug_buffer('noise_online').cpu(), L.debug_buffer('noise_target').cpu()
    ref = NR.learn_step(on, tg, n_on, n_tg, obs, act, rew, nobs, done, dueling=d, num_atoms=K, v_min=-10.0, v_max=10.0, weights=w,
                        gamma=0.99, double_dqn=double, max_grad_norm=clip)
    names = list(L.names)
    assert list(ref['grads']) == names
    q, y, prio, loss = L.debug_buffer('q'), L.debug_buffer('y'), L.debug_buffer('priorities'), float(L.debug_buffer('loss')[0])
    if K:
        err = {'q': _scaled(q, ref['q'], ref['q_scale']), 'y': _scaled(y, ref['y'], ref['y_scale']),
               'priorities': _scaled(prio, ref['priorities'], ref['kl_scale'])}
    else:
        err = {'q': _scaled(q, ref['q'], ref['q_scale']), 'y': nmax(y, ref['y']), 'priorities': nmax(prio, ref['priorities'])}
    err['loss'] = abs(loss - ref['loss']) / max(abs(ref['loss']), 1e-30)
    comp = _device_composed(L, 'online')
    mask_params = dict(on, **{'fc.weight': comp['fc'][0].cpu(), 'fc.bias': comp['fc'][1].cpu()})
    flips, units, worst = _mask_flips(L, mask_params, obs, B)
    gerr = {n: rel_l2(L.grads[n], ref['grads'][n]) for n in names}
    post = NR.adam_on_grads(on, {n: L.grads[n] for n in names}, max_grad_norm=clip)
    perr = max(float((L.params[n].cpu() - post[n]).abs().max()) for n in names)
    _record(f'split_{head}_B{B}_A{A}_double{int(double)}_clip{clip}', dict(err, grads=gerr, relu_mask_flips=flips, relu_units=units,
                                                                           worst_flipped_margin=worst, post_step_max_abs=perr))
    for k, v in err.items():
        assert v <= 1e-5, (k, v)
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)
    gtol = 1e-4 if flips == 0 else 2e-2
    for n, v in gerr.items():
        assert v <= gtol, (n, v, flips)
    assert perr <= 2e-6, perr


# ---------------------------------------------------------------------------------------------------------------- 4
def test_noise_distribution_and_keys():
    B, A = 32, 6
    on, tg = _nets(A, 'plain', seed=5)
    L = _learner(B, A, 'plain', on, tg, seed=11)
    batch, w = _batch(B, A, seed=6, device='cuda')
    pooled, prev = [], None
    for k in range(202):
        L.learn(batch, weights=w, sync_stats=False)               # eager, capture, then 200 replays
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
    _record('noise_ks', {'n': int(x.size), 'statistic': float(ks.statistic), 'pvalue': float(ks.pvalue), 'mean': float(x.mean()), 'std': float(x.std())})
    assert ks.pvalue > 1e-3, ks
    assert abs(x.mean()) < 5e-3 and abs(x.std() - 1) < 5e-3

    def first_draw(seed, step=0):
        M = _learner(B, A, 'plain', on, tg, seed=seed)
        M.set_step(step)
        M.learn(batch, weights=w, use_graph=False)
        return M.debug_buffer('normals_online'), M.debug_buffer('normals_target')

    s0, s0b, s1 = first_draw(11), first_draw(11), first_draw(12)
    assert torch.equal(s0[0], s0b[0]) and torch.equal(s0[1], s0b[1])
    assert not torch.equal(s0[0], s1[0]) and not torch.equal(s0[1], s1[1])
    # (seed, step) determines the draw: update 201 of L is update 201 of a learner set to that step
    assert torch.equal(first_draw(11, 201)[0], prev)


# ---------------------------------------------------------------------------------------------------------------- 5
def _run(A, head, on, tg, batches, use_graph, mem=64, seed=0, **kw):
    B = batches[0][0][0].shape[0]
    L = _learner(B, A, head, on, tg, seed=seed, **kw)
    S = GpuPrioritizedSampler(mem, alpha=0.6)
    S.add(mem)
    bufs = tuple(torch.empty_like(t) for t in batches[0][0])
    wb = torch.empty_like(batches[0][1])
    ib = torch.empty(B, dtype=torch.int64, device='cuda')
    for k, (b, w) in enumerate(batches):
        for d, s in zip(bufs, b):
            d.copy_(s)
        wb.copy_(w)
        ib.copy_(torch.randint(0, mem, (B,), generator=torch.Generator().manual_seed(k)))
        L.learn(bufs, weights=wb, idxs=ib, sampler=S, use_graph=use_graph, sync_stats=False)
    torch.cuda.synchronize()
    return L, S


@pytest.mark.parametrize('head', list(HEADS))
def test_determinism_and_graph_replay(head):
    B, A = 32, 6
    on, tg = _nets(A, head, seed=1)
    batches = [_batch(B, A, seed=s, device='cuda') for s in range(5)]
    kw = dict(double_dqn=True, max_grad_norm=10.0, target_update_frequency=2, soft_update_tau=0.5, seed=3)
    (e1, s1), (e2, s2), (g, sg) = _run(A, head, on, tg, batches, False, **kw), _run(A, head, on, tg, batches, False, **kw), \
        _run(A, head, on, tg, batches, True, **kw)
    assert len(g._graphs) == 1
    for t1, t2, tg_ in zip(s1.trees(), s2.trees(), sg.trees()):
        assert (t1 == t2 == tg_) if isinstance(t1, float) else (torch.equal(t1, t2) and torch.equal(t1, tg_))
    for L in (e2, g):
        assert torch.equal(e1.flat_params, L.flat_params) and torch.equal(e1.flat_target, L.flat_target)
        assert torch.equal(e1.exp_avg, L.exp_avg) and torch.equal(e1.exp_avg_sq, L.exp_avg_sq)
        assert torch.equal(e1.debug_buffer('noise_online'), L.debug_buffer('noise_online'))
    assert not torch.equal(e1.params['fc.weight_sigma'], on['fc.weight_sigma'].cuda())      # sigma trains
    # another noise seed gives another run
    o, _ = _run(A, head, on, tg, batches, False, **dict(kw, seed=4))
    assert not torch.equal(o.flat_params, e1.flat_params)


def _loop(seed, steps=60):
    E, A, n = 16, 4, 3
    L = B200ApexLearner(ApexHParams(batch_size=32, num_actions=A, gamma=0.99 ** n, target_update_frequency=20, noisy_dqn=True), seed=seed)
    X = B200ApexActor(E, A, seed=seed, noisy_dqn=True)
    X.sync_from(L)
    mem = GpuPrioritizedReplayBuffer(1024, E, n_step=n, gamma=0.99)
    torch.manual_seed(seed)
    g = torch.Generator().manual_seed(seed)
    losses = []
    for t in range(steps):
        obs, nobs = frames(E, 1000 * seed + 2 * t), frames(E, 1000 * seed + 2 * t + 1)
        action = X.act(obs)
        reward, done = torch.randn(E, generator=g).cuda(), (torch.rand(E, generator=g) < 0.05).cuda()
        mem.save_to_memory(obs, action, reward, nobs, done, is_vectorised=True, priorities_from=X)
        if len(mem) >= 64:
            losses.append(L.learn_from(mem)['loss'])
            if len(losses) % 10 == 0:
                X.sync_from(L)
    return L, mem, losses


def test_captured_learn_from_loop_is_deterministic():
    L1, m1, l1 = _loop(5)
    L2, m2, l2 = _loop(5)
    assert len(l1) > 50 and len(L1._graphs) == 1 and all(math.isfinite(x) for x in l1)
    assert l1 == l2 and torch.equal(L1.flat_params, L2.flat_params)
    assert torch.equal(m1.sampler.trees()[0], m2.sampler.trees()[0])
    assert m1.sampler._L.srl_per_invalid_updates(m1.sampler._h, m1.sampler._stream()) == 0


@pytest.mark.parametrize('head', ['plain', 'dueling'])
def test_checkpoint_roundtrip_and_resume(tmp_path, head):
    B, A = 16, 6
    on, tg = _nets(A, head, seed=4)
    batches = [_batch(B, A, seed=40 + s, device='cuda') for s in range(6)]
    kw = dict(target_update_frequency=2, soft_update_tau=0.3)
    full = _learner(B, A, head, on, tg, seed=7, **kw)
    half = _learner(B, A, head, on, tg, seed=7, **kw)
    for b, w in batches[:3]:
        full.learn(b, weights=w)
        half.learn(b, weights=w)
    path = str(tmp_path / 'apex_noisy.pt')
    half.save_checkpoint(path)
    ck = torch.load(path, weights_only=False)
    assert set(ck) == {'actor_state_dict', 'actor_target_state_dict', 'optimizer_state_dict'}
    assert tuple(ck['actor_state_dict']) == tuple(half.names)
    net = AtariQNet(A, dueling=head == 'dueling', noisy=True)
    net.load_state_dict(ck['actor_state_dict'])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    opt.load_state_dict(ck['optimizer_state_dict'])
    assert all(float(s['step']) == 3 for s in opt.state.values()) and len(opt.state) == len(half.names)
    i = half.names.index('fc.weight_sigma')
    torch.testing.assert_close(opt.state[opt.param_groups[0]['params'][i]]['exp_avg'],
                               half.exp_avg[half._off[i]:half._off[i] + half._cnt[i]].view(512, 3136).cpu(), rtol=0, atol=0)
    resumed = _learner(B, A, head, on, on, seed=7, **kw)
    resumed.load_checkpoint(path)
    assert int(resumed.debug_buffer('step')[0]) == 3
    for b, w in batches[3:]:
        full.learn(b, weights=w)
        resumed.learn(b, weights=w)
    torch.cuda.synchronize()
    assert torch.equal(full.debug_buffer('noise_online'), resumed.debug_buffer('noise_online'))      # the noise continues
    assert torch.equal(full.flat_params, resumed.flat_params) and torch.equal(full.flat_target, resumed.flat_target)
    assert torch.equal(full.exp_avg, resumed.exp_avg) and torch.equal(full.exp_avg_sq, resumed.exp_avg_sq)


# ---------------------------------------------------------------------------------------------------------------- 6
def _plain_sd(sd):
    return {n.replace('_mu', ''): v for n, v in sd.items() if 'sigma' not in n}


@pytest.mark.parametrize('head', list(HEADS))
def test_learner_q_values_use_mu(head):
    B, A = 16, 6
    on, _ = _nets(A, head, seed=2)
    L = _learner(B, A, head, on, on)
    P = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, **HEADS[head]), init_state_dict=_plain_sd(on))
    obs = frames(37, 1)
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
    kw = HEADS[head]
    d, K = _dims(head)
    sd = default_q_state_dict(A, 4, d, K, noisy=True)
    X = B200ApexActor(E, A, seed=9, init_state_dict=sd, noisy_dqn=True, **kw)
    assert bool((X.epsilons == 0).all())
    obs = frames(E, 2)
    # a new actor keeps a first draw: q_values compose it
    n0 = X.debug_buffer('noise')
    q0 = X.q_values(obs)
    ref = NR.composed(sd, n0, A, d, K)
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
    obs = frames(E, 3)
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
