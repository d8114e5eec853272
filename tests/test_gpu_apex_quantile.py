"""The quantile (QR-DQN) head of the Ape-X learner and actors on the H100 (ApexHParams(quantile_dqn=True),
B200ApexActor(..., quantile_dqn=True)):
  1. fp32-accurate split operands against the quantile fp32 CPU oracle (tests/apex_quantile_ref.py): Q(s, a) and y normalised by the
     size of the terms they sum, the target quantiles, the per-transition loss, priorities and loss to 1e-5, the 10 gradients to
     rel-L2 1e-4 (2e-2 when a genuine ReLU tie flipped: test_gpu_apex.py's accounting), the weights after the step against the
     oracle's Adam on the device gradients to 2e-6;
  2. bf16: the quantile tail against fp64 on its own operands (core rows, fp32 head weights): theta, the target quantiles, the loss,
     dtheta, the head gradients and dcore; the encoder gradients equal srl_encoder_backward on the tail's dcore, bit for bit;
  3. the actor's quantiles, Q values and eps = 0 actions are the learner's bit for bit (ties included), bf16 actor priorities are the
     learner's bit for bit, fp32-accurate actor priorities match the oracle's and the trees match PerOracle;
  4. noisy: with sigma = 0 a step is the plain quantile learner's on mu, bit for bit, and the composed head weights are torch's;
  5. eager, repeated and captured runs (and a captured learn_from loop with prioritized adds) are bit-identical; checkpoints load into
     AtariQNet(A, quantile=True) and torch.optim.Adam, and a resumed run equals an uninterrupted one;
  6. q_values against the CPU network.
The measured errors are written to $SRL_RESULTS_DIR/apex_quantile.json when SRL_RESULTS_DIR is set."""
import ctypes as C
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle.per_oracle import PerOracle
from tests import apex_noisy_ref as NR
from tests import apex_quantile_ref as R
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
    p = os.path.join(d, 'apex_quantile.json')
    cur = json.load(open(p)) if os.path.exists(p) else {}
    cur[name] = obj
    json.dump(cur, open(p, 'w'), indent=1)


def _nets(A, N, seed=0):
    return default_q_state_dict(A, 2 * seed, num_quantiles=N), default_q_state_dict(A, 2 * seed + 1, num_quantiles=N)


def _hp(B, A, N, kappa=1.0, **kw):
    return ApexHParams(batch_size=B, num_actions=A, quantile_dqn=True, num_quantiles=N, quantile_kappa=kappa, **kw)


def _learner(B, A, N, on, tg, kappa=1.0, **kw):
    L = B200ApexLearner(_hp(B, A, N, kappa, **kw), init_state_dict=on)
    L.load_state_dict(tg, target=True)
    return L


def _actor(E, A, N, kappa=1.0, **kw):
    return B200ApexActor(E, A, quantile_dqn=True, num_quantiles=N, quantile_kappa=kappa, **kw)


def frames(n, seed):
    return torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8, generator=torch.Generator().manual_seed(seed)).cuda()


def _scaled(a, b, scale):
    """max |a - b| over the largest term size of the sums a and b are"""
    a, b = a.detach().cpu().to(F64), b.detach().cpu().to(F64)
    return float((a - b).abs().max() / max(float(scale.abs().max()), 1e-300))


GRID = [(32, 6, 200), (5, 4, 2), (512, 18, 51)]


# ---------------------------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize('kappa', [1.0, 0.5])
@pytest.mark.parametrize('clip', [None, 40.0])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,N', GRID)
def test_split_against_quantile_oracle(B, A, N, double, clip, kappa):
    on, tg = _nets(A, N, seed=B)
    (obs, act, rew, nobs, done), w = _batch(B, A, seed=B + A)
    L = _learner(B, A, N, on, tg, kappa, precision='fp32_split', double_dqn=double, max_grad_norm=clip, priority_eps=0.0)
    L.learn(tuple(t.cuda() for t in (obs, act, rew, nobs, done)), weights=w.cuda(), use_graph=False)
    ref = R.learn_step(on, tg, obs, act, rew, nobs, done, N, kappa, weights=w, gamma=0.99, double_dqn=double, max_grad_norm=clip)
    assert tuple(ref['grads']) == NAMES
    err = {'q': _scaled(L.debug_buffer('q'), ref['q'], ref['q_scale']), 'y': _scaled(L.debug_buffer('y'), ref['y'], ref['y_scale']),
           'target_quantiles': nmax(L.debug_buffer('target_quantiles').view(B, N), ref['T']),
           'qr_loss': nmax(L.debug_buffer('qr_loss'), ref['loss_n']),
           'priorities': nmax(L.debug_buffer('priorities'), ref['loss_n']),
           'loss': abs(float(L.debug_buffer('loss')[0]) - ref['loss']) / max(abs(ref['loss']), 1e-30)}
    flips, units, worst = _mask_flips(L, on, obs, B)
    gerr = {n: rel_l2(L.grads[n], ref['grads'][n]) for n in NAMES}
    post = R.adam_on_grads(on, {n: L.grads[n] for n in NAMES}, max_grad_norm=clip)
    perr = max(float((L.params[n].cpu() - post[n]).abs().max()) for n in NAMES)
    _record(f'split_B{B}_A{A}_N{N}_double{int(double)}_clip{clip}_kappa{kappa}',
            dict(err, grads=gerr, relu_mask_flips=flips, relu_units=units, worst_flipped_margin=worst, post_step_max_abs=perr))
    for k, v in err.items():
        assert v <= 1e-5, (k, v)
    assert flips <= 2 + units * 2e-5 and worst < 1e-4, (flips, units, worst)
    gtol = 1e-4 if flips == 0 else 2e-2
    for n, v in gerr.items():
        assert v <= gtol, (n, v, flips)
    assert perr <= 2e-6, perr


# ---------------------------------------------------------------------------------------------------------------- 2
@pytest.mark.parametrize('kappa', [1.0, 0.5])
@pytest.mark.parametrize('double', [False, True])
@pytest.mark.parametrize('B,A,N', [(32, 6, 200), (512, 18, 51)])
def test_bf16_quantile_tail_against_fp64_and_encoder_backward(B, A, N, double, kappa):
    on, tg = _nets(A, N, seed=7)
    batch, w = _batch(B, A, seed=3, device='cuda')
    obs, act, rew, nobs, done = batch
    gamma = 0.97
    L = _learner(B, A, N, on, tg, kappa, double_dqn=double, gamma=gamma, priority_eps=0.0)
    pre = L.state_dict()
    L.learn(batch, weights=w, use_graph=False)
    core = lambda name: L.debug_buffer(name).view(B, 514)[:, :512].to(F64)
    h = core('core')
    Wo, bo = pre['q.weight'].cuda().to(F64), pre['q.bias'].cuda().to(F64)
    theta = (h @ Wo.T + bo).view(B, A, N)
    tn = (core('core_next_target') @ tg['q.weight'].cuda().to(F64).T + tg['q.bias'].cuda().to(F64)).view(B, A, N)
    tno = (core('core_next') @ Wo.T + bo).view(B, A, N) if double else None
    T = R.targets(tn, rew.to(F64), done, float(np.float32(gamma)), tno)
    rows, a = torch.arange(B, device='cuda'), act.long()
    ta = theta[rows, a]
    loss_n = R.quantile_loss(ta, T, kappa)
    dl = torch.zeros(B, A, N, dtype=F64, device='cuda')
    dl[rows, a] = R.dtheta_written(ta, T, kappa, w.to(F64))
    dl = dl.view(B, A * N)
    hb = torch.cat([h, torch.ones(B, 1, dtype=F64, device='cuda')], 1)
    gWb = dl.T @ hb
    dcore = dl @ Wo
    dev_dcore = L.debug_buffer('dcore').view(B, 514)
    pairs = {'theta': (L.debug_buffer('theta').view(B, A, N), theta), 'target_quantiles': (L.debug_buffer('target_quantiles').view(B, N), T),
             'qr_loss': (L.debug_buffer('qr_loss'), loss_n), 'priorities': (L.debug_buffer('priorities'), loss_n),
             'dtheta': (L.debug_buffer('dtheta').view(B, A * N), dl), 'q.weight': (L.grads['q.weight'], gWb[:, :512]),
             'q.bias': (L.grads['q.bias'], gWb[:, 512]), 'dcore': (dev_dcore[:, :512], dcore),
             'q': (L.debug_buffer('q'), ta.sum(1) / N), 'y': (L.debug_buffer('y'), T.sum(1) / N)}
    err = {k: (rel_l2(u, v), nmax(u, v)) for k, (u, v) in pairs.items()}
    want_loss = float((w.to(F64) * loss_n).mean())
    err['loss'] = (abs(float(L.debug_buffer('loss')[0]) - want_loss) / want_loss,) * 2
    _record(f'bf16_tail_B{B}_A{A}_N{N}_double{int(double)}_kappa{kappa}', err)
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


def test_done_transitions_do_not_read_s_prime():
    """every transition done: the targets are the rewards, whatever the target network says of s' (here: inf quantiles)"""
    B, A, N = 16, 4, 32
    on, tg = _nets(A, N, seed=5)
    tg['q.bias'] = torch.full_like(tg['q.bias'], math.inf)
    (obs, act, rew, nobs, done), w = _batch(B, A, seed=9, device='cuda')
    L = _learner(B, A, N, on, tg, priority_eps=0.0)
    L.learn((obs, act, rew, nobs, torch.ones_like(done)), weights=w, use_graph=False)
    assert torch.equal(L.debug_buffer('target_quantiles').view(B, N), rew[:, None].expand(B, N))
    assert bool(torch.isfinite(L.debug_buffer('priorities')).all()) and math.isfinite(float(L.debug_buffer('loss')[0]))


# ---------------------------------------------------------------------------------------------------------------- 3
@pytest.mark.parametrize('E', [1, 13, 256])
def test_actor_quantiles_q_values_and_greedy_act_are_the_learners(E):
    A, N = 6, 200
    L = B200ApexLearner(_hp(E, A, N), seed=3)
    X = _actor(E, A, N, epsilons=np.zeros(E), seed=1)
    X.sync_from(L)
    obs = frames(E, E)
    q = X.q_values(obs)
    assert torch.equal(q, L.q_values(obs))
    assert torch.equal(X.act(obs), torch.argmax(q, dim=1))
    # the quantiles of the learner's step over s are the actor's over the same frames
    batch, _ = _batch(E, A, seed=E, device='cuda')
    batch = (obs,) + batch[1:]
    L.learn(batch, use_graph=False)
    X.act(obs)
    assert torch.equal(X.debug_buffer('theta')[:E * A * N], L.debug_buffer('theta'))
    # ties of Q: actions 1 and 4 share their quantile rows, which dominate; the first index wins
    X.sync_from(L)
    sd = X.state_dict()
    sd['q.weight'][4 * N:5 * N] = sd['q.weight'][N:2 * N]
    sd['q.bias'][N:2 * N] += 30.0
    sd['q.bias'][4 * N:5 * N] = sd['q.bias'][N:2 * N]
    X.load_state_dict(sd)
    L.load_state_dict(sd)
    q = X.q_values(obs)
    assert torch.equal(q[:, 1], q[:, 4]) and bool((torch.argmax(q, dim=1) == 1).all())
    assert bool((X.act(obs) == 1).all())
    assert torch.equal(q, L.q_values(obs))


def test_fp32_actor_priorities_against_oracle_and_trees():
    E, A, N, gamma, M, kappa = 300, 6, 51, 0.99, 1024, 0.5
    sd = default_q_state_dict(A, 4, num_quantiles=N)
    X = _actor(E, A, N, kappa, precision='fp32_split', priority_eps=1e-6, init_state_dict=sd)
    mem = GpuPrioritizedReplayBuffer(M, E, alpha=1.0, n_step=1, gamma=gamma)       # n = 1, alpha = 1: leaf e is transition e's priority
    g = torch.Generator().manual_seed(8)
    s, ns = frames(E, 1), frames(E, 2)
    a, r, d = torch.randint(0, A, (E,), generator=g), torch.randn(E, generator=g), torch.rand(E, generator=g) < 0.3
    mem.save_to_memory(s, a.cuda(), r.cuda(), ns, d.cuda(), is_vectorised=True, priorities_from=X)
    sum_t, min_t, mp = mem.sampler.trees()
    cap = mem.sampler.capacity
    leaves = sum_t[cap:cap + E]
    want = R.initial_priorities(sd, s.cpu(), a, r, ns.cpu(), d, float(np.float32(gamma)), 1e-6, N, kappa)
    err = nmax(leaves, want)
    _record('fp32_split_actor_priorities', {'nmax': err})
    assert err <= 1e-5, err
    po = PerOracle(M, 1.0)
    po.update_priorities(list(range(E)), leaves.cpu().numpy())
    po.tree_ptr, po.size = E % M, E
    assert np.array_equal(sum_t.cpu().numpy(), po.sum_tree.tree) and np.array_equal(min_t.cpu().numpy(), po.min_tree.tree)
    assert mp == po.max_priority


def test_bf16_actor_priorities_are_the_learners():
    E, A, N, n, gamma = 32, 6, 200, 3, 0.99
    L = B200ApexLearner(_hp(E, A, N, gamma=gamma ** n, double_dqn=False, priority_eps=1e-6), seed=2)
    X = _actor(E, A, N, priority_eps=1e-6)
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
@pytest.mark.parametrize('double', [False, True])
def test_noisy_sigma_zero_is_the_plain_quantile_learner(double):
    B, A, N = 32, 6, 51
    on, tg = (default_q_state_dict(A, s, noisy=True, noisy_std=0.0, num_quantiles=N) for s in (6, 7))
    strip = lambda sd: {n.replace('_mu', ''): v for n, v in sd.items() if 'sigma' not in n}
    batch, w = _batch(B, A, seed=4, device='cuda')
    Nz = _learner(B, A, N, on, tg, noisy_dqn=True, double_dqn=double)
    P = _learner(B, A, N, strip(on), strip(tg), double_dqn=double)
    Nz.learn(batch, weights=w, use_graph=False)
    P.learn(batch, weights=w, use_graph=False)
    for k in ('q', 'y', 'priorities', 'loss', 'dcore', 'theta', 'target_quantiles', 'qr_loss', 'dtheta'):
        assert torch.equal(Nz.debug_buffer(k), P.debug_buffer(k)), k
    for n, g in P.grads.items():
        m = n.replace('weight', 'weight_mu').replace('bias', 'bias_mu') if not n.startswith('conv') else n
        assert torch.equal(Nz.grads[m], g), n
        assert torch.equal(Nz.params[m], P.params[n]), n
    assert bool(Nz.grads['q.weight_sigma'].any())          # sigma learns even from 0


def test_noisy_quantile_composition_is_torchs():
    B, A, N = 16, 4, 64
    on, tg = (default_q_state_dict(A, s, noisy=True, num_quantiles=N) for s in (8, 9))
    batch, w = _batch(B, A, seed=5, device='cuda')
    L = _learner(B, A, N, on, tg, noisy_dqn=True, double_dqn=True)
    L.learn(batch, weights=w, use_graph=False)
    for net, sd in (('online', on), ('target', tg)):
        noise = L.debug_buffer(f'noise_{net}').cpu()
        want = NR.composed(sd, noise, A, False, N)
        assert torch.equal(L.debug_buffer(f'head_weight_{net}').view(-1, 512).cpu(), want['q'][0]), net
        assert torch.equal(L.debug_buffer(f'head_bias_{net}').cpu(), want['q'][1]), net
    ei, eo = NR.split_noise(L.debug_buffer('noise_online'), A, False, N)['q']
    assert torch.equal(L.grads['q.weight_sigma'].cpu(), L.grads['q.weight_mu'].cpu() * torch.outer(eo, ei))


# ---------------------------------------------------------------------------------------------------------------- 5
def _run(A, N, on, tg, batches, use_graph, mem=64, **kw):
    B = batches[0][0][0].shape[0]
    L = _learner(B, A, N, on, tg, **kw)
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
    B, A, N = 32, 6, 200
    on, tg = _nets(A, N, seed=1)
    batches = [_batch(B, A, seed=s, device='cuda') for s in range(5)]
    kw = dict(double_dqn=True, max_grad_norm=10.0, target_update_frequency=2, soft_update_tau=0.5)
    (e1, s1), (e2, s2), (g, sg) = (_run(A, N, on, tg, batches, False, **kw), _run(A, N, on, tg, batches, False, **kw),
                                   _run(A, N, on, tg, batches, True, **kw))
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
    E, A, N, n = 16, 4, 51, 3
    L = B200ApexLearner(_hp(32, A, N, gamma=0.99 ** n, target_update_frequency=20), seed=seed)
    X = _actor(E, A, N, seed=seed)
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
    B, A, N = 16, 6, 200
    on, tg = _nets(A, N, seed=4)
    batches = [_batch(B, A, seed=40 + s, device='cuda') for s in range(6)]
    kw = dict(target_update_frequency=2, soft_update_tau=0.3)
    full = _learner(B, A, N, on, tg, **kw)
    half = _learner(B, A, N, on, tg, **kw)
    for b, w in batches[:3]:
        full.learn(b, weights=w)
        half.learn(b, weights=w)
    path = str(tmp_path / 'apex_quantile.pt')
    half.save_checkpoint(path)
    ck = torch.load(path, weights_only=False)
    assert set(ck) == {'actor_state_dict', 'actor_target_state_dict', 'optimizer_state_dict'}
    assert tuple(ck['actor_state_dict']) == NAMES
    net = AtariQNet(A, quantile=True, num_quantiles=N)
    net.load_state_dict(ck['actor_state_dict'])
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    opt.load_state_dict(ck['optimizer_state_dict'])
    assert all(float(s['step']) == 3 for s in opt.state.values()) and len(opt.state) == 10
    i = NAMES.index('q.weight')
    torch.testing.assert_close(opt.state[opt.param_groups[0]['params'][i]]['exp_avg'],
                               half.exp_avg[half._off[i]:half._off[i] + half._cnt[i]].view(A * N, 512).cpu(), rtol=0, atol=0)
    resumed = _learner(B, A, N, on, on, **kw)
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


# ---------------------------------------------------------------------------------------------------------------- 6
@pytest.mark.parametrize('precision,tol', [('bf16', 2e-2), ('fp32_split', 1e-5)])
def test_q_values_against_cpu_network(precision, tol):
    B, A, N, n = 16, 18, 200, 37
    torch.manual_seed(9)
    net = AtariQNet(A, quantile=True, num_quantiles=N)
    with torch.no_grad():
        net.q.bias.add_(5.0)                   # Q away from 0: a relative error is meaningful
    L = B200ApexLearner(_hp(B, A, N, precision=precision), init_state_dict=net.state_dict())
    obs = torch.randint(0, 256, (n, 4, 84, 84), dtype=torch.uint8)
    q = L.q_values(obs)
    ref = net(obs).detach()
    err = rel_l2(q, ref)
    _record(f'q_values_{precision}', err)
    assert err <= tol, err
    assert torch.equal(L.predict(obs), q.argmax(-1))
    with pytest.raises(ValueError, match='quantile_dqn'):
        B200ApexActor(4, A).sync_from(L)
