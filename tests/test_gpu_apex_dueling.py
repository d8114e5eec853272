"""The dueling head of the Ape-X learner and actors on the H100 (ApexHParams(dueling_dqn=True), B200ApexActor(..., dueling_dqn=True)):
  1. fp32-accurate split operands against the dueling fp32 CPU oracle (tests/apex_dueling_ref.py): q, y, priorities and loss to 1e-5,
     the 12 gradients to rel-L2 1e-4 (2e-2 when a genuine ReLU tie flipped: test_gpu_apex.py's accounting), the weights after
     the step against the oracle's Adam on the device gradients to 2e-6;
  2. bf16: the dueling tail against fp64 on its own operands (core rows, fp32 head weights); the encoder gradients equal
     srl_encoder_backward on the tail's dcore, bit for bit;
  3. the actor's Q values are the learner's bit for bit, act with epsilon 0 is their first argmax, fp32-accurate initial priorities
     match compute_prior on the dueling net, and bf16 actor priorities are the learner's bit for bit;
  4. eager, repeated and captured runs (and a captured learn_from loop with prioritized adds) are bit-identical; checkpoints load
     into AtariQNet(A, dueling=True) and torch.optim.Adam, and a resumed run equals an uninterrupted one; q_values against the CPU net.
The measured errors are written to $SRL_RESULTS_DIR/apex_dueling.json when SRL_RESULTS_DIR is set."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from tests import apex_dueling_ref as D
from tests.test_gpu_apex import _batch, _mask_flips, nmax, rel_l2
from scalerl_b200 import _lib
from scalerl_b200.algorithms.apex import (APEX_DUELING_PARAM_NAMES as NAMES, ApexHParams, AtariQNet, B200ApexActor, B200ApexLearner,
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
    p = os.path.join(d, 'apex_dueling.json')
    cur = json.load(open(p)) if os.path.exists(p) else {}
    cur[name] = obj
    json.dump(cur, open(p, 'w'), indent=1)


def _nets(A, seed=0):
    return default_q_state_dict(A, 2 * seed, dueling=True), default_q_state_dict(A, 2 * seed + 1, dueling=True)


def _learner(B, A, on, tg, **kw):
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, dueling_dqn=True, **kw), init_state_dict=on)
    L.load_state_dict(tg, target=True)
    return L


def frames(n, seed):
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).cuda()


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (5, 4), (512, 18)])
def test_split_against_dueling_oracle(B, A, double, clip):
    on, tg = _nets(A, seed=B)
    (obs, act, rew, nobs, done), w = _batch(B, A, seed=B + A)
    L = _learner(B, A, on, tg, precision='fp32_split', double_dqn=double, max_grad_norm=clip, priority_eps=0.0)
    L.learn(tuple(t.cuda() for t in (obs, act, rew, nobs, done)), weights=w.cuda(), use_graph=False)
    ref = D.learn_step(on, tg, obs, act, rew, nobs, done, weights=w, gamma=0.99, double_dqn=double, max_grad_norm=clip)
    assert tuple(ref['grads']) == NAMES
    q, y, prio, loss = L.debug_buffer('q'), L.debug_buffer('y'), L.debug_buffer('priorities'), float(L.debug_buffer('loss')[0])
    err = {'q': nmax(q, ref['q']), 'y': nmax(y, ref['y']), 'priorities': nmax(prio, ref['td']),
           'loss': abs(loss - ref['loss']) / max(abs(ref['loss']), 1e-30)}
    flips, units, worst = _mask_flips(L, on, obs, B)
    gerr = {n: rel_l2(L.grads[n], ref['grads'][n]) for n in NAMES}
    post = D.adam_on_grads(on, {n: L.grads[n] for n in NAMES}, max_grad_norm=clip)
    perr = max(float((L.params[n].cpu() - post[n]).abs().max()) for n in NAMES)
    _record(f'split_B{B}_A{A}_double{int(double)}_clip{clip}', dict(err, grads=gerr, relu_mask_flips=flips, relu_units=units,
                                                                         worst_flipped_margin=worst, post_step_max_abs=perr))
    for k, v in err.items():
        assert v <= 1e-5, (k, v)
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)
    gtol = 1e-4 if flips == 0 else 2e-2
    for n, v in gerr.items():
        assert v <= gtol, (n, v, flips)
    assert perr <= 2e-6, perr


# ---------------------------------------------------------------------------------------------------------------- 2
def _q64(h, sd):
    """the dueling Q rows [B, A] in fp64"""
    Wv, bv = sd['value.weight'].cuda().to(F64), sd['value.bias'].cuda().to(F64)
    Wa, ba = sd['advantage.weight'].cuda().to(F64), sd['advantage.bias'].cuda().to(F64)
    adv = h @ Wa.T + ba
    return (h @ Wv.T + bv) + adv - adv.mean(1, keepdim=True)


@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A', [(32, 6), (512, 18)])
def test_bf16_dueling_tail_against_fp64_and_encoder_backward(B, A, double):
    on, tg = _nets(A, seed=7)
    batch, w = _batch(B, A, seed=3, device='cuda')
    obs, act, rew, nobs, done = batch
    gamma = 0.97
    L = _learner(B, A, on, tg, double_dqn=double, gamma=gamma, priority_eps=0.0)
    pre = L.state_dict()
    L.learn(batch, weights=w, use_graph=False)
    h = L.debug_buffer('core').view(B, 514)[:, :512].to(F64)
    hnt = L.debug_buffer('core_next_target').view(B, 514)[:, :512].to(F64)
    a = act.long()
    q = _q64(h, pre).gather(1, a[:, None]).squeeze(1)
    qt = _q64(hnt, tg)
    if double:
        astar = _q64(L.debug_buffer('core_next').view(B, 514)[:, :512].to(F64), pre).argmax(1)
    else:
        astar = qt.argmax(1)
    y = rew.to(F64) + gamma * qt.gather(1, astar[:, None]).squeeze(1) * (1 - done.to(F64))
    delta = q - y
    loss = (w.to(F64) * delta ** 2).mean()
    dq = 2 * w.to(F64) * delta / B
    coef = dq[:, None] * (torch.nn.functional.one_hot(a, A).to(F64) - 1.0 / A)      # dL/dAdv
    Wv, Wa = pre['value.weight'].to(F64), pre['advantage.weight'].to(F64)
    dcore = dq[:, None] * (Wv + Wa[a] - Wa.mean(0, keepdim=True))
    dev_dcore = L.debug_buffer('dcore').view(B, 514)
    pairs = {'q': (L.debug_buffer('q'), q), 'y': (L.debug_buffer('y'), y), 'delta': (L.debug_buffer('priorities'), delta.abs()),
             'value.weight': (L.grads['value.weight'], (dq[:, None] * h).sum(0, keepdim=True)),
             'value.bias': (L.grads['value.bias'], dq.sum().view(1)),
             'advantage.weight': (L.grads['advantage.weight'], coef.T @ h), 'advantage.bias': (L.grads['advantage.bias'], coef.sum(0)),
             'dcore': (dev_dcore[:, :512], dcore)}
    err = {k: (rel_l2(u, v), nmax(u, v)) for k, (u, v) in pairs.items()}
    err['loss'] = (abs(float(L.debug_buffer('loss')[0]) - float(loss)) / float(loss),) * 2
    _record(f'bf16_tail_B{B}_A{A}_double{int(double)}', err)
    for k, (r, m) in err.items():
        assert r <= 2e-5 and m <= 1e-4, (k, r, m)
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
    for n, g in zip(NAMES[:8], gs):
        assert torch.equal(g, L.grads[n]), n


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('E', [1, 13, 256, 1500])
def test_actor_q_values_are_the_learners_and_greedy_act(E):
    A = 6
    L = B200ApexLearner(ApexHParams(batch_size=32, num_actions=A, dueling_dqn=True), seed=3)
    X = B200ApexActor(E, A, epsilons=np.zeros(E), seed=1, dueling_dqn=True)
    X.sync_from(L)
    obs = frames(E, E)
    q = X.q_values(obs)
    assert torch.equal(q, L.q_values(obs))
    assert torch.equal(X.act(obs), torch.argmax(q, dim=1))
    # ties of Q (not of Adv alone): actions 1 and 4 share their advantage row and the largest bias; the first index wins
    sd = L.state_dict()
    sd['advantage.weight'][4] = sd['advantage.weight'][1]
    sd['advantage.bias'][1] = sd['advantage.bias'][4] = 30.0
    X.load_state_dict(sd)
    q = X.q_values(obs)
    assert torch.equal(q[:, 1], q[:, 4]) and bool((torch.argmax(q, dim=1) == 1).all())
    assert bool((X.act(obs) == 1).all())


def test_fp32_actor_priorities_against_compute_prior():
    E, A, gamma, M = 300, 6, 0.99, 1024
    sd = default_q_state_dict(A, 4, dueling=True)
    X = B200ApexActor(E, A, precision='fp32_split', priority_eps=1e-6, init_state_dict=sd, dueling_dqn=True)
    mem = GpuPrioritizedReplayBuffer(M, E, alpha=1.0, n_step=1, gamma=gamma)       # n = 1, alpha = 1: leaf e is transition e's priority
    g = torch.Generator().manual_seed(8)
    s, ns = frames(E, 1), frames(E, 2)
    a, r, d = torch.randint(0, A, (E,), generator=g), torch.randn(E, generator=g), torch.rand(E, generator=g) < 0.3
    mem.save_to_memory(s, a.cuda(), r.cuda(), ns, d.cuda(), is_vectorised=True, priorities_from=X)
    cap = mem.sampler.capacity
    leaves = mem.sampler.trees()[0][cap:cap + E]
    want = D.initial_priorities(sd, s.cpu(), a, r, ns.cpu(), d, float(np.float32(gamma)), 1e-6)
    err = nmax(leaves, want)
    _record('fp32_split_actor_priorities', {'nmax': err})
    assert err <= 1e-5, err


def test_bf16_actor_priorities_are_the_learners():
    E, A, n, gamma = 32, 6, 3, 0.99
    L = B200ApexLearner(ApexHParams(batch_size=E, num_actions=A, gamma=gamma ** n, double_dqn=False, priority_eps=1e-6, dueling_dqn=True), seed=2)
    X = B200ApexActor(E, A, priority_eps=1e-6, dueling_dqn=True)
    X.sync_from(L)
    mem = GpuPrioritizedReplayBuffer(256, E, alpha=1.0, n_step=n, gamma=gamma)
    # the learner writes its priorities into trees of its own through the same leaf update (p^alpha in double: pow(p, 1) need not
    # return p exactly), so equal leaves mean equal priorities
    S = GpuPrioritizedSampler(256, alpha=1.0)
    S.add(256)
    g = torch.Generator().manual_seed(6)
    compared = 0
    for t in range(5):
        args = (torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(), torch.randint(0, A, (E,), generator=g).cuda(),
                torch.randn(E, generator=g).cuda(), torch.randint(0, 256, (E, 4, 84, 84), dtype=torch.uint8, generator=g).cuda(),
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
def _run(A, on, tg, batches, use_graph, mem=64, **kw):
    B = batches[0][0][0].shape[0]
    L = _learner(B, A, on, tg, **kw)
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
    B, A = 32, 6
    on, tg = _nets(A, seed=1)
    batches = [_batch(B, A, seed=s, device='cuda') for s in range(5)]
    kw = dict(double_dqn=True, max_grad_norm=10.0, target_update_frequency=2, soft_update_tau=0.5)
    (e1, s1), (e2, s2), (g, sg) = _run(A, on, tg, batches, False, **kw), _run(A, on, tg, batches, False, **kw), _run(A, on, tg, batches, True, **kw)
    assert len(g._graphs) == 1
    for t1, t2, tg_ in zip(s1.trees(), s2.trees(), sg.trees()):
        assert (t1 == t2 == tg_) if isinstance(t1, float) else (torch.equal(t1, t2) and torch.equal(t1, tg_))
    for n in NAMES:
        assert torch.equal(e1.params[n], e2.params[n]) and torch.equal(e1.params[n], g.params[n]), n
        assert torch.equal(e1.target_params[n], g.target_params[n]), n
    assert torch.equal(e1.exp_avg, g.exp_avg) and torch.equal(e1.exp_avg_sq, g.exp_avg_sq)
    assert not torch.equal(e1.params['advantage.weight'], on['advantage.weight'].cuda())      # the advantage stream trains
    assert int(g.debug_buffer('step')[0]) == 5


def _loop(seed, steps=60):
    E, A, n = 16, 4, 3
    L = B200ApexLearner(ApexHParams(batch_size=32, num_actions=A, gamma=0.99 ** n, target_update_frequency=20, dueling_dqn=True), seed=seed)
    X = B200ApexActor(E, A, seed=seed, dueling_dqn=True)
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
    B, A = 16, 6
    on, tg = _nets(A, seed=4)
    batches = [_batch(B, A, seed=40 + s, device='cuda') for s in range(6)]
    kw = dict(target_update_frequency=2, soft_update_tau=0.3)
    full = _learner(B, A, on, tg, **kw)
    half = _learner(B, A, on, tg, **kw)
    for b, w in batches[:3]:
        full.learn(b, weights=w)
        half.learn(b, weights=w)
    path = str(tmp_path / 'apex_dueling.pt')
    half.save_checkpoint(path)
    ck = torch.load(path, weights_only=False)
    assert set(ck) == {'actor_state_dict', 'actor_target_state_dict', 'optimizer_state_dict'}
    assert tuple(ck['actor_state_dict']) == NAMES
    net = AtariQNet(A, dueling=True)
    net.load_state_dict(ck['actor_state_dict'])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    opt.load_state_dict(ck['optimizer_state_dict'])
    assert all(float(s['step']) == 3 for s in opt.state.values()) and len(opt.state) == 12
    i = NAMES.index('advantage.weight')
    torch.testing.assert_close(opt.state[opt.param_groups[0]['params'][i]]['exp_avg'],
                               half.exp_avg[half._off[i]:half._off[i] + half._cnt[i]].view(A, 512).cpu(), rtol=0, atol=0)
    resumed = _learner(B, A, on, on, **kw)
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
    B, A, n = 16, 18, 37
    torch.manual_seed(9)
    net = AtariQNet(A, dueling=True)
    L = B200ApexLearner(ApexHParams(batch_size=B, num_actions=A, precision=precision, dueling_dqn=True), init_state_dict=net.state_dict())
    obs = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8)
    q = L.q_values(obs)
    ref = net(obs).detach()
    err = rel_l2(q, ref)
    _record(f'q_values_{precision}', err)
    assert err <= tol, err
    assert torch.equal(L.predict(obs), q.argmax(-1))
    with pytest.raises(ValueError, match='dueling_dqn'):
        B200ApexActor(4, A).sync_from(L)
