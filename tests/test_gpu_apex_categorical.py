"""The categorical (C51) head of the Ape-X learner and actors on the H100 (ApexHParams(categorical_dqn=True),
B200ApexActor(..., categorical_dqn=True)):
  1. fp32-accurate split operands against the categorical fp32 CPU oracle (tests/apex_categorical_ref.py): Q(s, a), m, CE, priorities
     and loss to 1e-5 (Q and the KL priorities normalised by the size of the terms they sum: Q = sum z p cancels on a support around
     0, KL = CE - H(m) cancels when m is close to p), the 10 gradients to rel-L2 1e-4 (2e-2 when a genuine ReLU tie flipped: test_gpu_apex.py's accounting), the
     weights after the step against the oracle's Adam on the device gradients to 2e-6;
  2. bf16: the categorical tail against fp64 on its own operands (core rows, fp32 head weights): logits, p, m, CE, KL, dlogits, the head
     gradients and dcore; the encoder gradients equal srl_encoder_backward on the tail's dcore, bit for bit;
  3. the actor's logits, Q values and ε = 0 actions are the learner's bit for bit (ties included), bf16 actor priorities are the
     learner's bit for bit, fp32-accurate actor priorities match the oracle's and the trees match PerOracle;
  4. eager, repeated and captured runs (and a captured learn_from loop with prioritized adds) are bit-identical; checkpoints load
     into AtariQNet(A, categorical=True) and torch.optim.Adam, and a resumed run equals an uninterrupted one; q_values against the CPU net.
The measured errors are written to $SRL_RESULTS_DIR/apex_categorical.json when SRL_RESULTS_DIR is set."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle.per_oracle import PerOracle
from tests import apex_categorical_ref as R
from tests.test_gpu_apex import _batch, _mask_flips, nmax, rel_l2
from scalerl_b200 import _lib
from scalerl_b200.algorithms.apex import (APEX_PARAM_NAMES as NAMES, ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner,
                                          default_q_state_dict)
from scalerl_b200.data.per_sampler import GpuPrioritizedSampler
from scalerl_b200.data.replay_memory import GpuPrioritizedReplayBuffer

pytestmark = pytest.mark.gpu
F64 = torch.float64


def _record(name, obj):
    d = os.environ.get('SRL_RESULTS_DIR')
    if not d:
        return
    os.makedirs(d, exist_ok=True)
    p = os.path.join(d, 'apex_categorical.json')
    cur = json.load(open(p)) if os.path.exists(p) else {}
    cur[name] = obj
    json.dump(cur, open(p, 'w'), indent=1)


def _nets(A, K, seed=0):
    return default_q_state_dict(A, 2 * seed, num_atoms=K), default_q_state_dict(A, 2 * seed + 1, num_atoms=K)


def _hp(B, A, K, support, **kw):
    return ApexHParams(batch_size=B, num_actions=A, categorical_dqn=True, num_atoms=K, v_min=support[0], v_max=support[1], **kw)


def _learner(B, A, K, support, on, tg, **kw):
    L = B200ApexLearner(_hp(B, A, K, support, **kw), init_state_dict=on)
    L.load_state_dict(tg, target=True)
    return L


def _actor(E, A, K, support, **kw):
    return B200ApexActor(E, A, categorical_dqn=True, num_atoms=K, v_min=support[0], v_max=support[1], **kw)


def frames(n, seed):
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).cuda()


SUPPORTS = [(0.0, 200.0), (-10.0, 10.0)]
GRID = [(32, 6, 51), (5, 4, 2), (512, 18, 51), (64, 31, 64)]


def _scaled(a, b, scale):
    """max |a - b| over the largest term size of the sums a and b are"""
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    return float((a - b).abs().max() / max(float(scale.abs().max()), 1e-300))


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('support', SUPPORTS)
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,K', GRID)
def test_split_against_categorical_oracle(B, A, K, double, clip, support):
    on, tg = _nets(A, K, seed=B)
    (obs, act, rew, nobs, done), w = _batch(B, A, seed=B + A)
    rew = rew * (support[1] - support[0]) / 20          # rewards on the scale of the support
    L = _learner(B, A, K, support, on, tg, precision='fp32_split', double_dqn=double, max_grad_norm=clip, priority_eps=0.0)
    L.learn(tuple(t.cuda() for t in (obs, act, rew, nobs, done)), weights=w.cuda(), use_graph=False)
    ref = R.learn_step(on, tg, obs, act, rew, nobs, done, K, *support, weights=w, gamma=0.99, double_dqn=double, max_grad_norm=clip)
    assert tuple(ref['grads']) == NAMES
    err = {'q': _scaled(L.debug_buffer('q'), ref['q'], ref['q_scale']), 'm': nmax(L.debug_buffer('m').view(B, K), ref['m']),
           'ce': nmax(L.debug_buffer('ce'), ref['ce']),
           'priorities': _scaled(L.debug_buffer('priorities'), ref['kl'].clamp(min=0), ref['kl_scale']),
           'loss': abs(float(L.debug_buffer('loss')[0]) - ref['loss']) / max(abs(ref['loss']), 1e-30)}
    flips, units, worst = _mask_flips(L, on, obs, B)
    gerr = {n: rel_l2(L.grads[n], ref['grads'][n]) for n in NAMES}
    post = R.adam_on_grads(on, {n: L.grads[n] for n in NAMES}, max_grad_norm=clip)
    perr = max(float((L.params[n].cpu() - post[n]).abs().max()) for n in NAMES)
    _record(f'split_B{B}_A{A}_K{K}_double{int(double)}_clip{clip}_support{support}',
            dict(err, grads=gerr, relu_mask_flips=flips, relu_units=units, worst_flipped_margin=worst, post_step_max_abs=perr))
    for k, v in err.items():
        assert v <= 1e-5, (k, v)
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)
    gtol = 1e-4 if flips == 0 else 2e-2
    for n, v in gerr.items():
        assert v <= gtol, (n, v, flips)
    assert perr <= 2e-6, perr


# ---------------------------------------------------------------------------------------------------------------- 2
def _tail64(h, W, b, z, A, K):
    """logits, p, log p [B, A, K] and Q [B, A] in fp64 from core rows h and the fp32 head weights"""
    logits = (h @ W.T + b).view(-1, A, K)
    logp = torch.log_softmax(logits, dim=2)
    p = logp.exp()
    return logits, p, logp, (p * z).sum(2)


@pytest.mark.parametrize('support', SUPPORTS)
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,K', [(32, 6, 51), (512, 18, 51), (64, 31, 64)])
def test_bf16_categorical_tail_against_fp64_and_encoder_backward(B, A, K, double, support):
    on, tg = _nets(A, K, seed=7)
    batch, w = _batch(B, A, seed=3, device='cuda')
    obs, act, rew, nobs, done = batch
    rew = rew * (support[1] - support[0]) / 20
    batch = (obs, act, rew, nobs, done)
    gamma = 0.97
    L = _learner(B, A, K, support, on, tg, double_dqn=double, gamma=gamma, priority_eps=0.0)
    pre = L.state_dict()
    L.learn(batch, weights=w, use_graph=False)
    z32, dz32 = R.support(K, *support)
    z, lo, hi = z32.to(F64).cuda(), float(np.float32(support[0])), float(np.float32(support[1]))
    core = lambda name: L.debug_buffer(name).view(B, 514)[:, :512].to(F64)
    h = core('core')
    Wo, bo = pre['q.weight'].cuda().to(F64), pre['q.bias'].cuda().to(F64)
    logits, p, logp, _ = _tail64(h, Wo, bo, z, A, K)
    _, pt, _, qt = _tail64(core('core_next_target'), tg['q.weight'].cuda().to(F64), tg['q.bias'].cuda().to(F64), z, A, K)
    astar = (_tail64(core('core_next'), Wo, bo, z, A, K)[3] if double else qt).argmax(1)
    rows, a = torch.arange(B, device='cuda'), act.long()
    g = float(np.float32(gamma)) * (1 - done.to(F64))
    tz = (rew.to(F64)[:, None] + g[:, None] * z[None]).clamp(lo, hi)
    bj = (tz - lo) / float(dz32)
    lower, upper = bj.floor().long().clamp(0, K - 1), bj.ceil().long().clamp(0, K - 1)
    pj = pt[rows, astar]
    m = torch.zeros(B, K, dtype=F64, device='cuda')
    eq = lower == upper
    m.scatter_add_(1, lower, torch.where(eq, pj, pj * (upper.to(F64) - bj)))
    m.scatter_add_(1, upper, torch.where(eq, torch.zeros_like(pj), pj * (bj - lower.to(F64))))
    lp = logp[rows, a]
    ce = -(m * lp).sum(1)
    kl = (torch.xlogy(m, m) - m * lp).sum(1)
    dl = torch.zeros(B, A, K, dtype=F64, device='cuda')
    dl[rows, a] = (w.to(F64) / B)[:, None] * (p[rows, a] * m.sum(1, keepdim=True) - m)
    dl = dl.view(B, A * K)
    hb = torch.cat([h, torch.ones(B, 1, dtype=F64, device='cuda')], 1)
    gWb = dl.T @ hb
    dcore = dl @ Wo
    dev_dcore = L.debug_buffer('dcore').view(B, 514)
    pairs = {'logits': (L.debug_buffer('logits').view(B, A, K), logits), 'm': (L.debug_buffer('m').view(B, K), m),
             'ce': (L.debug_buffer('ce'), ce), 'kl': (L.debug_buffer('priorities'), kl.clamp(min=0)),
             'dlogits': (L.debug_buffer('dlogits').view(B, A * K), dl), 'q.weight': (L.grads['q.weight'], gWb[:, :512]),
             'q.bias': (L.grads['q.bias'], gWb[:, 512]), 'dcore': (dev_dcore[:, :512], dcore),
             'q': (L.debug_buffer('q'), (p[rows, a] * z).sum(1)), 'y': (L.debug_buffer('y'), (m * z).sum(1))}
    err = {k: (rel_l2(u, v), nmax(u, v)) for k, (u, v) in pairs.items()}
    err['loss'] = (abs(float(L.debug_buffer('loss')[0]) - float((w.to(F64) * ce).mean())) / float((w.to(F64) * ce).mean()),) * 2
    # p: the softmax of the kernel's own logits against that of the fp64 logits
    pk = torch.softmax(L.debug_buffer('logits').view(B, A, K).to(F64), dim=2)
    err['p'] = (rel_l2(pk, p), nmax(pk, p))
    _record(f'bf16_tail_B{B}_A{A}_K{K}_double{int(double)}_support{support}', err)
    for k, (r_, m_) in err.items():
        assert r_ <= 2e-5 and m_ <= 1e-4, (k, r_, m_)
    assert not bool(dev_dcore[:, 512:].any())

    # the encoder gradients of the step are srl_encoder_backward on the tail's dcore, bit for bit
    lib = _lib.lib()
    E = C.c_void_p()
    _lib.check(lib.srl_encoder_create(0, C.byref(E)), 'encoder_create')
    try:
        sb, kb = C.c_int64(), C.c_int64()
        _lib.check(lib.srl_encoder_sizes(B, 0, C.byref(sb), C.byref(kb)), 'encoder_sizes')
        saved = torch.empty(sb.value, dtype=torch.uint8, device='cuda')
        scratch = torch.empty(kb.value, dtype=torch.uint8, device='cuda')
        ws = [pre[n].cuda().contiguous() for n in NAMES[:8]]
        gs = [torch.empty_like(t) for t in ws]
        core_out = torch.empty(B, 514, device='cuda')
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(lib.srl_encoder_forward(E, obs.data_ptr(), rew.data_ptr(), act.data_ptr(), B, 1, (C.c_void_p * 8)(*[t.data_ptr() for t in ws]),
                                           saved.data_ptr(), scratch.data_ptr(), core_out.data_ptr(), st), 'encoder_forward')
        dc = dev_dcore.contiguous()
        _lib.check(lib.srl_encoder_backward(E, dc.data_ptr(), B, 1, saved.data_ptr(), scratch.data_ptr(),
                                            (C.c_void_p * 8)(*[t.data_ptr() for t in gs]), st), 'encoder_backward')
        torch.cuda.synchronize()
    finally:
        lib.srl_encoder_destroy(E)
    assert torch.equal(core_out, L.debug_buffer('core').view(B, 514))
    for n, g_ in zip(NAMES[:8], gs):
        assert torch.equal(g_, L.grads[n]), n


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('E', [1, 13, 256, 1500])
def test_actor_logits_q_values_and_greedy_act_are_the_learners(E):
    A, K, support = 6, 51, (-10.0, 10.0)
    L = B200ApexLearner(_hp(E, A, K, support), seed=3)
    X = _actor(E, A, K, support, epsilons=np.zeros(E), seed=1)
    X.sync_from(L)
    obs = frames(E, E)
    q = X.q_values(obs)
    assert torch.equal(q, L.q_values(obs))
    assert torch.equal(X.act(obs), torch.argmax(q, dim=1))
    # the logits of the learner's step over s are the actor's over the same frames
    batch, _ = _batch(E, A, seed=E, device='cuda')
    batch = (obs,) + batch[1:]
    L.learn(batch, use_graph=False)
    X.act(obs)
    assert torch.equal(X.debug_buffer('logits')[:E * A * K], L.debug_buffer('logits'))
    # ties of Q: actions 1 and 4 share their logit rows, and their top atom dominates; the first index wins
    X.sync_from(L)
    sd = X.state_dict()
    sd['q.weight'][4 * K:5 * K] = sd['q.weight'][K:2 * K]
    sd['q.bias'][4 * K:5 * K] = sd['q.bias'][K:2 * K]
    sd['q.bias'][2 * K - 1] += 30.0
    sd['q.bias'][5 * K - 1] += 30.0
    X.load_state_dict(sd)
    L.load_state_dict(sd)
    q = X.q_values(obs)
    assert torch.equal(q[:, 1], q[:, 4]) and bool((torch.argmax(q, dim=1) == 1).all())
    assert bool((X.act(obs) == 1).all())
    assert torch.equal(q, L.q_values(obs))


def test_fp32_actor_priorities_against_oracle_and_trees():
    E, A, K, gamma, M, support = 300, 6, 51, 0.99, 1024, (0.0, 200.0)
    sd = default_q_state_dict(A, 4, num_atoms=K)
    X = _actor(E, A, K, support, precision='fp32_split', priority_eps=1e-6, init_state_dict=sd)
    mem = GpuPrioritizedReplayBuffer(M, E, alpha=1.0, n_step=1, gamma=gamma)       # n = 1, alpha = 1: leaf e is transition e's priority
    g = torch.Generator().manual_seed(8)
    s, ns = frames(E, 1), frames(E, 2)
    a, r, d = torch.randint(0, A, (E,), generator=g), 10 * torch.randn(E, generator=g), torch.rand(E, generator=g) < 0.3
    mem.save_to_memory(s, a.cuda(), r.cuda(), ns, d.cuda(), is_vectorised=True, priorities_from=X)
    sum_t, min_t, mp = mem.sampler.trees()
    cap = mem.sampler.capacity
    leaves = sum_t[cap:cap + E]
    want = R.initial_priorities(sd, s.cpu(), a, r, ns.cpu(), d, float(np.float32(gamma)), 1e-6, K, *support)
    err = nmax(leaves, want)
    _record('fp32_split_actor_priorities', {'nmax': err})
    assert err <= 1e-5, err
    po = PerOracle(M, 1.0)
    po.update_priorities(list(range(E)), leaves.cpu().numpy())
    po.tree_ptr, po.size = E % M, E
    assert np.array_equal(sum_t.cpu().numpy(), po.sum_tree.tree) and np.array_equal(min_t.cpu().numpy(), po.min_tree.tree)
    assert mp == po.max_priority


def test_bf16_actor_priorities_are_the_learners():
    E, A, K, n, gamma, support = 32, 6, 51, 3, 0.99, (-10.0, 10.0)
    L = B200ApexLearner(_hp(E, A, K, support, gamma=gamma ** n, double_dqn=False, priority_eps=1e-6), seed=2)
    X = _actor(E, A, K, support, priority_eps=1e-6)
    X.sync_from(L)
    mem = GpuPrioritizedReplayBuffer(256, E, alpha=1.0, n_step=n, gamma=gamma)
    S = GpuPrioritizedSampler(256, alpha=1.0)
    S.add(256)
    g = torch.Generator().manual_seed(6)
    compared = 0
    for t in range(5):
        args = (torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(), torch.randint(0, A, (E,), generator=g).cuda(),
                (3 * torch.randn(E, generator=g)).cuda(), torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(),
                (torch.rand(E, generator=g) < 0.3).cuda())
        ptr = (t - n + 1) * E % 256
        mem.save_to_memory(*args, is_vectorised=True, priorities_from=X)
        if t + 1 < n:
            continue
        idxs = (torch.arange(E) + ptr) % 256
        cap = mem.sampler.capacity
        leaves = mem.sampler.trees()[0][cap + idxs.cuda()]
        L.learn(mem.gather(idxs), idxs=idxs.cuda(), sampler=S, use_graph=False)
        assert torch.equal(S.trees()[0][S.capacity + idxs.cuda()], leaves), t
        X.sync_from(L)
        L.update_target(1.0)
        compared += 1
    assert compared == 3


# ---------------------------------------------------------------------------------------------------------------- 4
def _run(A, K, on, tg, batches, use_graph, mem=64, **kw):
    B = batches[0][0][0].shape[0]
    L = _learner(B, A, K, (-10.0, 10.0), on, tg, **kw)
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


def test_determinism_and_graph_replay():
    B, A, K = 32, 6, 51
    on, tg = _nets(A, K, seed=1)
    batches = [_batch(B, A, seed=s, device='cuda') for s in range(5)]
    kw = dict(double_dqn=True, max_grad_norm=10.0, target_update_frequency=2, soft_update_tau=0.5)
    (e1, s1), (e2, s2), (g, sg) = (_run(A, K, on, tg, batches, False, **kw), _run(A, K, on, tg, batches, False, **kw),
                                   _run(A, K, on, tg, batches, True, **kw))
    assert len(g._graphs) == 1
    for t1, t2, tg_ in zip(s1.trees(), s2.trees(), sg.trees()):
        assert (t1 == t2 == tg_) if isinstance(t1, float) else (torch.equal(t1, t2) and torch.equal(t1, tg_))
    for n in NAMES:
        assert torch.equal(e1.params[n], e2.params[n]) and torch.equal(e1.params[n], g.params[n]), n
        assert torch.equal(e1.target_params[n], g.target_params[n]), n
    assert torch.equal(e1.exp_avg, g.exp_avg) and torch.equal(e1.exp_avg_sq, g.exp_avg_sq)
    assert not torch.equal(e1.params['q.weight'], on['q.weight'].cuda())
    assert int(g.debug_buffer('step')[0]) == 5


def _loop(seed, steps=60):
    E, A, K, n, support = 16, 4, 51, 3, (-10.0, 10.0)
    L = B200ApexLearner(_hp(32, A, K, support, gamma=0.99 ** n, target_update_frequency=20), seed=seed)
    X = _actor(E, A, K, support, seed=seed)
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


def test_checkpoint_roundtrip_and_resume(tmp_path):
    B, A, K, support = 16, 6, 51, (-10.0, 10.0)
    on, tg = _nets(A, K, seed=4)
    batches = [_batch(B, A, seed=40 + s, device='cuda') for s in range(6)]
    kw = dict(target_update_frequency=2, soft_update_tau=0.3)
    full = _learner(B, A, K, support, on, tg, **kw)
    half = _learner(B, A, K, support, on, tg, **kw)
    for b, w in batches[:3]:
        full.learn(b, weights=w)
        half.learn(b, weights=w)
    path = str(tmp_path / 'apex_categorical.pt')
    half.save_checkpoint(path)
    ck = torch.load(path, weights_only=False)
    assert set(ck) == {'actor_state_dict', 'actor_target_state_dict', 'optimizer_state_dict'}
    assert tuple(ck['actor_state_dict']) == NAMES
    net = AtariQNet(A, categorical=True, num_atoms=K, v_min=support[0], v_max=support[1])
    net.load_state_dict(ck['actor_state_dict'])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    opt.load_state_dict(ck['optimizer_state_dict'])
    assert all(float(s['step']) == 3 for s in opt.state.values()) and len(opt.state) == 10
    i = NAMES.index('q.weight')
    torch.testing.assert_close(opt.state[opt.param_groups[0]['params'][i]]['exp_avg'],
                               half.exp_avg[half._off[i]:half._off[i] + half._cnt[i]].view(A * K, 512).cpu(), rtol=0, atol=0)
    resumed = _learner(B, A, K, support, on, on, **kw)
    resumed.load_checkpoint(path)
    assert int(resumed.debug_buffer('step')[0]) == 3
    for b, w in batches[3:]:
        full.learn(b, weights=w)
        resumed.learn(b, weights=w)
    torch.cuda.synchronize()
    for n in NAMES:
        assert torch.equal(full.params[n], resumed.params[n]), n
        assert torch.equal(full.target_params[n], resumed.target_params[n]), n
    assert torch.equal(full.exp_avg, resumed.exp_avg) and torch.equal(full.exp_avg_sq, resumed.exp_avg_sq)


@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
def test_q_values_against_cpu_network(precision, tol):
    B, A, K, n, support = 16, 18, 51, 37, (0.0, 200.0)      # Q near 100: a relative error is meaningful
    torch.manual_seed(9)
    net = AtariQNet(A, categorical=True, num_atoms=K, v_min=support[0], v_max=support[1])
    L = B200ApexLearner(_hp(B, A, K, support, precision=precision), init_state_dict=net.state_dict())
    obs = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8)
    q = L.q_values(obs)
    ref = net(obs).detach()
    err = rel_l2(q, ref)
    _record(f'q_values_{precision}', err)
    assert err <= tol, err
    assert torch.equal(L.predict(obs), q.argmax(-1))
    with pytest.raises(ValueError, match='categorical_dqn'):
        B200ApexActor(4, A).sync_from(L)
